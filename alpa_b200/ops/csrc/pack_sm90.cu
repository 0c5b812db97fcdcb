// Cross-mesh resharding pack / unpack: gather the strided tiles one device sends to a peer into ONE contiguous
// staging buffer (and scatter a received buffer into the destination slices) in a single launch.
//
// The cross-mesh path of a pipeline moves, per resharding task and per peer, a handful of tiles that are slices of a
// stage output (reference: the per-tile ncclSend / ncclRecv + the dynamic-update-slice of
// alpa/pipeline_parallel/cross_mesh_resharding.py:60-230 and the "pack kernel" of SURVEY.md K14).  Packing them first
// turns N slice-copy launches + N messages into one launch + one message per peer, and the receive side needs no
// temporary per tile: one buffer lands, one launch writes every destination slice.
//
// Tiles are described as <= 4-D boxes with byte strides and a contiguous innermost dimension; 16-byte vector copies
// when the box and both addresses allow it, byte copies otherwise.  Up to 32 tiles per launch ride in the kernel
// parameters (no descriptor upload, graph-capturable).
#include <cuda_runtime.h>
#include <stdint.h>

#include "kernels.h"

namespace ab {
namespace {

template <bool kUnpack>
__global__ void __launch_bounds__(256) pack_tiles_kernel(const __grid_constant__ PackArgs args) {
  const PackTile& t = args.tiles[blockIdx.y];
  const long long rows = t.shape[0] * t.shape[1] * t.shape[2];
  const long long inner = t.shape[3];                        // bytes of the contiguous innermost run
  for (long long row = blockIdx.x; row < rows; row += gridDim.x) {
    const long long i2 = row % t.shape[2];
    const long long r1 = row / t.shape[2];
    const long long i1 = r1 % t.shape[1];
    const long long i0 = r1 / t.shape[1];
    char* strided = t.strided + i0 * t.stride[0] + i1 * t.stride[1] + i2 * t.stride[2];
    char* packed = t.packed + row * inner;
    if (t.vec16) {
      const int4* s = reinterpret_cast<const int4*>(kUnpack ? packed : strided);
      int4* d = reinterpret_cast<int4*>(kUnpack ? strided : packed);
      for (long long i = threadIdx.x; i < (inner >> 4); i += blockDim.x) d[i] = s[i];
    } else {
      const char* s = kUnpack ? packed : strided;
      char* d = kUnpack ? strided : packed;
      for (long long i = threadIdx.x; i < inner; i += blockDim.x) d[i] = s[i];
    }
  }
}

}  // namespace
}  // namespace ab

extern "C" int ab_pack_tiles(const ab::PackArgs* args, int unpack, cudaStream_t st) {
  if (args->num_tiles <= 0 || args->num_tiles > ab::kMaxPackTiles) return 1;
  long long max_rows = 1;
  for (int i = 0; i < args->num_tiles; ++i) {
    const ab::PackTile& t = args->tiles[i];
    const long long rows = t.shape[0] * t.shape[1] * t.shape[2];
    max_rows = rows > max_rows ? rows : max_rows;
  }
  // enough CTAs per tile to cover the machine a few times over without exceeding the row count
  const int cap = ab::num_sms() * 8;   // 8 resident 256-thread CTAs per SM
  const int per_tile = (int)(max_rows < cap ? max_rows : cap);
  dim3 grid((unsigned)per_tile, (unsigned)args->num_tiles);
  if (unpack)
    ab::pack_tiles_kernel<true><<<grid, 256, 0, st>>>(*args);
  else
    ab::pack_tiles_kernel<false><<<grid, 256, 0, st>>>(*args);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

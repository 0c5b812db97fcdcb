// Peer-memory (NVLink 4 / NVSwitch) building blocks of the fused compute+collective ops.
//
//  * GEMM -> reduce-scatter : the GEMM epilogue (gemm_sm90.cu, `scatter_*` fields) stores each
//    partial tile straight into the *owner GPU's* staging slot over NVLink and bumps a per-32-row arrival
//    counter there; `rs_reduce_kernel` (below, on the owner) waits per row block and sums the slots, with
//    bias / residual fused.  Transfers therefore overlap the math tile by tile; no NCCL call.
//  * all-gather -> GEMM      : `ag_push_kernel` writes this rank's activation shard into every peer's
//    gather buffer (peer stores, or one NVLS multicast store) and publishes a per-128-row epoch flag; the
//    consumer GEMM's TMA producer waits on the flag of the M-block it is about to load
//    (`a_ready` in GemmArgs) and starts with its own shard, so math overlaps the gather.
//  * `allreduce_multimem_kernel`: NVLS in-switch all-reduce (multimem.ld_reduce + multimem.st) for
//    replicated results.
//
// Replaces: NCCL thunks after cuBLAS GEMMs in the reference (K3/K5/K10 of SURVEY.md §2.5,
// XLA/service/gpu/nccl_all_reduce_thunk.cc:103-121, :434-458, nccl_all_gather_thunk.cc:73-91).
#include <stdio.h>

#include "kernels.h"
#include "pdl.h"
#include "ptx.cuh"

namespace ab {

__device__ __forceinline__ void spin_until_ge(const uint32_t* flag, uint32_t expected) {
  uint32_t spins = 0;
  while (ld_acquire_sys(flag) < expected) {
    __nanosleep(64);
    if (++spins > (1u << 24)) {
      printf("alpa_b200: peer-flag watchdog (block %d, flag %p, have %u want %u)\n", blockIdx.x, flag,
             ld_relaxed_sys(flag), expected);
      __trap();
    }
  }
}

// out[r, :] = sum_s staging[s][r, :] (+ bias) (+ residual[r, :]);  one CTA per 32-row block x column slab.
__global__ void __launch_bounds__(256)
rs_reduce_kernel(const __nv_bfloat16* __restrict__ staging, const uint32_t* __restrict__ flags,
                 uint32_t expected, __nv_bfloat16* __restrict__ out, const __nv_bfloat16* __restrict__ bias,
                 const __nv_bfloat16* __restrict__ residual, int rows, int N, int tp, long long slot_stride) {
  const int blk = blockIdx.x;          // 32-row block
  const int r0 = blk * 32;
  if (r0 >= rows) return;
  if (threadIdx.x == 0) spin_until_ge(flags + blk, expected);
  __syncthreads();
  const int nvec = N / 8;
  const int rmax = min(32, rows - r0);
  for (int idx = blockIdx.y * blockDim.x + threadIdx.x; idx < rmax * nvec; idx += gridDim.y * blockDim.x) {
    const int r = r0 + idx / nvec;
    const int c = (idx % nvec) * 8;
    float acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.f;
    for (int s = 0; s < tp; ++s) {
      const int4 v = ld_volatile_v4(staging + (size_t)s * slot_stride + (size_t)r * N + c);
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    if (bias != nullptr) {
      const int4 v = *reinterpret_cast<const int4*>(bias + c);
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    if (residual != nullptr) {
      const int4 v = *reinterpret_cast<const int4*>(residual + (size_t)r * N + c);
      const uint32_t* u = reinterpret_cast<const uint32_t*>(&v);
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float2 f = unpack_bf16x2(u[j]);
        acc[2 * j] += f.x;
        acc[2 * j + 1] += f.y;
      }
    }
    int4 o;
    o.x = pack_bf16x2(acc[0], acc[1]);
    o.y = pack_bf16x2(acc[2], acc[3]);
    o.z = pack_bf16x2(acc[4], acc[5]);
    o.w = pack_bf16x2(acc[6], acc[7]);
    *reinterpret_cast<int4*>(out + (size_t)r * N + c) = o;
  }
}

struct PeerPtrs {
  void* data[kMaxPeersComm];
  uint32_t* flags[kMaxPeersComm];
};

// Push rows [0, rows) of `src` into slot `rank` of every peer's gather buffer ([tp*rows, K] on each
// peer).  One CTA per (128-row block, peer); flag = epoch once the block has landed.
__global__ void __launch_bounds__(256)
ag_push_kernel(const __nv_bfloat16* __restrict__ src, PeerPtrs peers, int rows, int K, int rank, int tp,
               uint32_t epoch, int include_self) {
  const int blk = blockIdx.x;  // 128-row block within my shard
  const int p = blockIdx.y;    // destination peer
  if (p >= tp || (!include_self && p == rank)) return;
  const int r0 = blk * 128;
  const int rmax = min(128, rows - r0);
  if (rmax <= 0) return;
  const int nvec = K / 8;
  __nv_bfloat16* dst = reinterpret_cast<__nv_bfloat16*>(peers.data[p]) + ((size_t)rank * rows + r0) * K;
  const __nv_bfloat16* s = src + (size_t)r0 * K;
  for (int idx = threadIdx.x; idx < rmax * nvec; idx += blockDim.x) {
    const int4 v = ld_nc_v4(s + (size_t)idx * 8);
    st_v4(dst + (size_t)idx * 8, v);
  }
  __threadfence_system();
  __syncthreads();
  if (threadIdx.x == 0) {
    const int blocks_per_rank = (rows + 127) / 128;
    st_release_sys(peers.flags[p] + rank * blocks_per_rank + blk, epoch);
  }
}

// NVLS all-reduce over a symmetric buffer: every rank reduces 1/tp of the elements in the switch
// (multimem.ld_reduce) and broadcasts the result (multimem.st).  `mc` is the multicast address of the
// buffer; barriers before/after are the caller's (symmetric-memory signal pads).
__global__ void __launch_bounds__(512)
allreduce_multimem_kernel(__nv_bfloat16* mc, long long numel, int rank, int tp) {
  const long long nvec = numel / 8;
  const long long per = (nvec + tp - 1) / tp;
  const long long lo = per * rank, hi = min(nvec, per * (rank + 1));
  const long long stride = (long long)gridDim.x * blockDim.x;
  long long i = lo + blockIdx.x * (long long)blockDim.x + threadIdx.x;
  // four independent in-switch reductions in flight per thread: a gradient bucket is reduced by a handful of CTAs
  // (the rest of the GPU keeps running backward), so the bandwidth has to come from memory-level parallelism
  for (; i + 3 * stride < hi; i += 4 * stride) {
    const int4 v0 = multimem_ld_reduce_bf16x8(mc + i * 8);
    const int4 v1 = multimem_ld_reduce_bf16x8(mc + (i + stride) * 8);
    const int4 v2 = multimem_ld_reduce_bf16x8(mc + (i + 2 * stride) * 8);
    const int4 v3 = multimem_ld_reduce_bf16x8(mc + (i + 3 * stride) * 8);
    multimem_st_v4(mc + i * 8, v0);
    multimem_st_v4(mc + (i + stride) * 8, v1);
    multimem_st_v4(mc + (i + 2 * stride) * 8, v2);
    multimem_st_v4(mc + (i + 3 * stride) * 8, v3);
  }
  for (; i < hi; i += stride) {
    const int4 v = multimem_ld_reduce_bf16x8(mc + i * 8);
    multimem_st_v4(mc + i * 8, v);
  }
}

// Cross-GPU barrier on symmetric signal pads: each rank bumps slot[rank] on every peer, then waits
// until all of its own slots reach `epoch`.
__global__ void peer_barrier_kernel(PeerPtrs peers, int rank, int tp, uint32_t epoch) {
  const int p = threadIdx.x;
  if (p < tp) {
    __threadfence_system();
    st_release_sys(peers.flags[p] + rank, epoch);
    spin_until_ge(peers.flags[rank] + p, epoch);
  }
}

// The same barrier with the epoch kept on the device: `counter` (local memory) is bumped by the kernel itself, so the
// launch has no per-call arguments and can be replayed from a CUDA graph (every rank runs the same sequence of
// barriers, so the epochs agree).  The watchdog is wall-clock based and generous: ranks may be seconds apart during
// warm-up (compilation, graph capture).
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

__global__ void peer_barrier_auto_kernel(PeerPtrs peers, uint32_t* counter, int rank, int tp) {
  const int p = threadIdx.x;
  const uint32_t epoch = *reinterpret_cast<volatile uint32_t*>(counter) + 1;
  __syncwarp();
  if (p == 0) *reinterpret_cast<volatile uint32_t*>(counter) = epoch;
  if (p < tp) {
    __threadfence_system();
    st_release_sys(peers.flags[p] + rank, epoch);
    const uint32_t* mine = peers.flags[rank] + p;
    const unsigned long long t0 = globaltimer_ns();
    uint32_t spins = 0;
    while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
      __nanosleep(100);
      if ((++spins & 0xfffffu) == 0 && globaltimer_ns() - t0 > 600ull * 1000000000ull) {
        printf("alpa_b200: peer barrier timed out (rank %d waiting for %d, have %u want %u)\n", rank, p,
               ld_relaxed_sys(mine), epoch);
        __trap();
      }
    }
  }
}

// One-shot all-reduce of a small vector (tensor-parallel decode: [batch, hidden] activations, a few KB) in ONE kernel:
//   copy x into my symmetric staging buffer -> cross-GPU barrier (every partial result is in place) -> in-switch
//   reduction of the WHOLE vector by every rank (multimem.ld_reduce; nothing is written back, so no second barrier)
//   -> result stored to `out` (may alias x).
// Two staging halves alternate by the parity of the device-side epoch: a rank re-writes half h for call k+2 only after
// it passed the barrier of call k+1, which every peer signals after finishing its reads of call k.  Epoch and buffer
// choice live on the device: the launch has no per-call arguments and is replayable from a CUDA graph.
__global__ void __launch_bounds__(1024)
allreduce_oneshot_kernel(const __nv_bfloat16* __restrict__ x, __nv_bfloat16* sym_local, const __nv_bfloat16* mc,
                         long long half_stride, __nv_bfloat16* out, const __nv_bfloat16* __restrict__ residual,
                         int nvec, PeerPtrs peers, uint32_t* counter, int rank, int tp) {
  __shared__ uint32_t s_epoch;
  griddep_launch_dependents();      // the next kernel's weight prefetch may start now
  griddep_wait();                   // x is produced by the previous kernel
  if (threadIdx.x == 0) {
    const uint32_t e = *reinterpret_cast<volatile uint32_t*>(counter) + 1;
    *reinterpret_cast<volatile uint32_t*>(counter) = e;
    s_epoch = e;
  }
  __syncthreads();
  const uint32_t epoch = s_epoch;
  const long long off = (epoch & 1u) ? half_stride : 0;
  for (int i = threadIdx.x; i < nvec; i += blockDim.x)
    st_v4(sym_local + off + (size_t)i * 8, ld_nc_v4(x + (size_t)i * 8));
  __threadfence_system();
  __syncthreads();
  if ((int)threadIdx.x < tp) {
    const int p = threadIdx.x;
    __threadfence_system();
    st_release_sys(peers.flags[p] + rank, epoch);
    const uint32_t* mine = peers.flags[rank] + p;
    const unsigned long long t0 = globaltimer_ns();
    uint32_t spins = 0;
    while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
      if ((++spins & 0xfffffu) == 0 && globaltimer_ns() - t0 > 600ull * 1000000000ull) {
        printf("alpa_b200: one-shot all-reduce timed out (rank %d waiting for %d)\n", rank, p);
        __trap();
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < nvec; i += blockDim.x) {
    int4 v = multimem_ld_reduce_bf16x8(mc + off + (size_t)i * 8);
    if (residual != nullptr) {      // fused residual add (fp32, rounded once)
      const int4 r = *reinterpret_cast<const int4*>(residual + (size_t)i * 8);
      uint32_t* vu = reinterpret_cast<uint32_t*>(&v);
      const uint32_t* ru = reinterpret_cast<const uint32_t*>(&r);
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float2 a = unpack_bf16x2(vu[q]), b = unpack_bf16x2(ru[q]);
        vu[q] = pack_bf16x2(a.x + b.x, a.y + b.y);
      }
    }
    *reinterpret_cast<int4*>(out + (size_t)i * 8) = v;
  }
}

}  // namespace ab

using namespace ab;

extern "C" int ab_allreduce_oneshot(const __nv_bfloat16* x, __nv_bfloat16* sym_local, const __nv_bfloat16* mc,
                                    long long half_stride, __nv_bfloat16* out, const __nv_bfloat16* residual,
                                    long long numel, uint32_t* const* peer_flags, uint32_t* counter, int rank, int tp,
                                    cudaStream_t st) {
  if (numel % 8 != 0 || tp > kMaxPeersComm || numel > half_stride) return 1;
  PeerPtrs p;
  for (int i = 0; i < tp; ++i) {
    p.data[i] = nullptr;
    p.flags[i] = peer_flags[i];
  }
  const int nvec = (int)(numel / 8);
  int threads = (nvec + 31) / 32 * 32;
  if (threads < 32) threads = 32;
  if (threads > 1024) threads = 1024;
  const cudaError_t e = launch_pdl(allreduce_oneshot_kernel, dim3(1), dim3(threads), 0, st, x, sym_local, mc, half_stride,
                                   out, residual, nvec, p, counter, rank, tp);
  return e == cudaSuccess ? 0 : 2;
}

extern "C" int ab_peer_barrier_auto(uint32_t* const* peer_flags, uint32_t* counter, int rank, int tp, cudaStream_t st) {
  if (tp > kMaxPeersComm) return 1;
  PeerPtrs p;
  for (int i = 0; i < tp; ++i) {
    p.data[i] = nullptr;
    p.flags[i] = peer_flags[i];
  }
  peer_barrier_auto_kernel<<<1, 32, 0, st>>>(p, counter, rank, tp);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_rs_reduce(const __nv_bfloat16* staging, const uint32_t* flags, uint32_t expected,
                            __nv_bfloat16* out, const __nv_bfloat16* bias, const __nv_bfloat16* residual, int rows,
                            int N, int tp, long long slot_stride, cudaStream_t st) {
  if (N % 8 != 0) return 1;
  const int blocks = (rows + 31) / 32;
  int gy = (ab::num_sms() * 4 + blocks - 1) / blocks;
  if (gy < 1) gy = 1;
  if (gy > 16) gy = 16;
  rs_reduce_kernel<<<dim3(blocks, gy), 256, 0, st>>>(staging, flags, expected, out, bias, residual, rows, N, tp,
                                                    slot_stride);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_ag_push(const __nv_bfloat16* src, void* const* peer_data, uint32_t* const* peer_flags, int rows,
                          int K, int rank, int tp, uint32_t epoch, int include_self, cudaStream_t st) {
  if (K % 8 != 0 || tp > kMaxPeersComm) return 1;
  PeerPtrs p;
  for (int i = 0; i < tp; ++i) {
    p.data[i] = peer_data[i];
    p.flags[i] = peer_flags[i];
  }
  ag_push_kernel<<<dim3((rows + 127) / 128, tp), 256, 0, st>>>(src, p, rows, K, rank, tp, epoch, include_self);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_allreduce_multimem(__nv_bfloat16* mc, long long numel, int rank, int tp, int ctas, cudaStream_t st) {
  if (numel % 8 != 0) return 1;
  if (ctas <= 0 || ctas > ab::num_sms()) ctas = ab::num_sms();
  allreduce_multimem_kernel<<<ctas, 512, 0, st>>>(mc, numel, rank, tp);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

extern "C" int ab_peer_barrier(uint32_t* const* peer_flags, int rank, int tp, uint32_t epoch, cudaStream_t st) {
  if (tp > kMaxPeersComm) return 1;
  PeerPtrs p;
  for (int i = 0; i < tp; ++i) {
    p.data[i] = nullptr;
    p.flags[i] = peer_flags[i];
  }
  peer_barrier_kernel<<<1, 32, 0, st>>>(p, rank, tp, epoch);
  return cudaGetLastError() == cudaSuccess ? 0 : 2;
}

"""`ops.pack_tiles` / `ops.unpack_tiles`: the tiles of a resharding task for one peer as one 16-byte-aligned staging
buffer (reference of pack_sm90.cu; the kernel itself is checked by scripts/gpu_check_pack.py)."""
import torch

from alpa_b200 import ops


def test_pack_unpack_round_trip_and_layout():
    torch.manual_seed(0)
    x = torch.randn(6, 10, 12)
    h = torch.randn(5, 7).to(torch.bfloat16)
    views = [x[1:3, :, 4:8], x[0], x[:, 2:5, :], x[5, 9, 1:2], h[:, 2:5], h[4]]
    flat = ops.pack_tiles(views)
    assert flat.dtype == torch.uint8 and flat.numel() == ops.packed_nbytes(views)
    off = 0
    for v in views:                                          # every tile starts on a 16-byte boundary, row-major inside
        n = v.numel() * v.element_size()
        assert off % 16 == 0
        assert torch.equal(flat[off:off + n].view(v.dtype).view(v.shape), v)
        off += (n + 15) // 16 * 16
    y, g = torch.zeros_like(x), torch.zeros_like(h)
    dst = [y[1:3, :, 4:8], y[0], y[:, 2:5, :], y[5, 9, 1:2], g[:, 2:5], g[4]]
    ops.unpack_tiles(flat, dst)
    for a, b in zip(views, dst):
        assert torch.equal(a, b)
    assert float(y[3, 0, 0]) == 0.0                          # nothing outside the slices was written (row 3: only cols 2:5)

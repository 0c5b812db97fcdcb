"""Block-scaled MXFP8 (OCP microscaling) maths shared by the sm_90a kernel and its CPU reference: exponent choice,
the scale-factor atom layout the MXFP8 GEMM reads, and the reference linear."""
import torch

from alpa_b200 import ops


def test_block_exponents_are_tight_and_saturation_free():
    torch.manual_seed(0)
    x = torch.randn(200, 160) * torch.logspace(-3, 3, 160)[None]
    x[5, 32:64] = 0                                           # all-zero block
    x[7, 0] = 448.0 * 2.0 ** 5                                # block maximum exactly on the e4m3 maximum
    q, sf = ops.quantize_mxfp8(x)
    assert q.dtype == torch.float8_e4m3fn and sf.shape == (2, 2, 512) and sf.dtype == torch.uint8
    e = ops.mx_unpack_scale_atoms(sf, 200, 160).float() - 127
    amax = x.view(200, 5, 32).abs().amax(-1)
    scaled = amax * torch.exp2(-e)
    nz = amax > 0
    assert float(scaled.max()) <= 448.0 and float(scaled[nz].min()) > 224.0      # smallest power of two that fits
    assert int(e[5, 1]) == -127 and int(e[7, 0]) == 5
    d = ops.dequantize_mxfp8(q, sf)
    assert float(((d - x).abs() / amax.clamp(min=1e-30).repeat_interleave(32, 1)).max()) <= 2.0 ** -4 + 1e-6
    assert float(d[5, 32:64].abs().max()) == 0.0


def test_scale_atom_layout():
    e = torch.arange(300 * 9, dtype=torch.int64).remainder(251).to(torch.uint8).view(300, 9)   # 300 rows, K = 288
    sf = ops.mx_pack_scale_atoms(e)
    assert sf.shape == (3, 3, 512)
    for r, kb in ((0, 0), (31, 3), (32, 0), (150, 4), (299, 8), (127, 7)):
        rr = r % 128
        assert int(sf[r // 128, kb // 4, (rr % 32) * 16 + (rr // 32) * 4 + kb % 4]) == int(e[r, kb])
    assert int(sf[2, 0, (50 % 32) * 16 + (50 // 32) * 4]) == 127              # row 306: padding = scale 1.0
    assert int(sf[0, 2, 0 * 16 + 0 * 4 + 1]) == 127                          # K block 9: padding
    assert torch.equal(ops.mx_unpack_scale_atoms(sf, 300, 288), e)


def test_linear_mxfp8_reference_tracks_fp32_linear():
    torch.manual_seed(1)
    x = torch.randn(4, 70, 256) * 3
    x[..., 17] *= 200.0                                       # an outlier channel
    w, b = torch.randn(96, 256) * 0.05, torch.randn(96)
    wq, wsf = ops.quantize_mxfp8(w)
    y = ops.linear_mxfp8(x, wq, wsf, b, "gelu")
    ref = torch.nn.functional.gelu(torch.nn.functional.linear(x, w, b))
    assert y.shape == ref.shape
    rel = float((y - ref).norm() / ref.norm())
    assert rel < 0.06, rel


def test_serving_decoder_with_block_scaled_weights():
    """`weight_dtype="mxfp8"`: every linear of the serving decoder holds e4m3 weights + scale atoms; logits stay
    close to the full-precision model and generation (prefill + decode steps with the KV cache) runs."""
    from alpa_b200.model.opt_model import DecoderLM, get_config
    from alpa_b200.serve.generator import Generator
    torch.manual_seed(0)

    def build(wd):
        cfg = get_config("opt-125m", dtype=torch.float32)
        cfg.num_hidden_layers, cfg.hidden_size, cfg.num_attention_heads, cfg.ffn_dim, cfg.vocab_size = 2, 64, 4, 128, 128
        cfg.weight_dtype = wd
        return DecoderLM(cfg, device="cpu", seed=3)
    ref, mx = build("bf16"), build("mxfp8")
    lin = mx.layers[0]["fc1"]
    assert lin.mx and lin.w.dtype == torch.float8_e4m3fn and lin.scale.shape == (1, 1, 512)
    ids = torch.randint(4, 128, (2, 12))
    pos = torch.arange(12).repeat(2, 1)
    a = ref.forward(ids, pos, ref.init_cache(2, 16), 0, last_only=False).float()
    b = mx.forward(ids, pos, mx.init_cache(2, 16), 0, last_only=False).float()
    assert float((a - b).norm() / a.norm()) < 0.08
    out = Generator(mx, 2, 32).generate(ids, max_new_tokens=4).sequences
    assert out.shape == (2, 16) and torch.equal(out[:, :12], ids)

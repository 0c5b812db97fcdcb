"""GPU checks of the iteration-level batching path (new this round; runs after the other GPU tests)."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_gpu_kernels import check  # noqa: E402

pytestmark = pytest.mark.gpu


def test_ragged_attention_numerics():
    """Ragged 1-D attention over a slot-addressed KV cache (OPT-2.7B/TP1 head shapes), with and without ALiBi, against
    the fp32 PyTorch path of the same op."""
    from alpa_b200 import ops
    from alpa_b200.ops import primitives as P
    torch.manual_seed(0)
    dev = "cuda"
    fails = []
    for (h, D, lens, new) in [(4, 64, [37, 1, 300, 129], [5, 1, 1, 129]), (32, 80, [512, 77, 2048, 1000], [1, 1, 1, 64]),
                              (8, 128, [16, 4000], [16, 1])]:
        slots = sum(lens) + 64
        kc = torch.randn(slots + 1, h, D, device=dev, dtype=torch.bfloat16)
        vc = torch.randn(slots + 1, h, D, device=dev, dtype=torch.bfloat16)
        starts, s = [], 7
        for n in lens:
            starts.append(s)
            s += n + 3
        seq_start, ctx_len = [], []
        for st, n, k in zip(starts, lens, new):            # the last `k` tokens of each sequence are queries
            for j in range(n - k, n):
                seq_start.append(st)
                ctx_len.append(j + 1)
        seq_start += [0, 0]
        ctx_len += [0, 0]                                   # padding tokens
        T = len(seq_start)
        q = torch.randn(T, h, 3, D, device=dev, dtype=torch.bfloat16)[:, :, 0]          # strided view like qkv
        ss = torch.tensor(seq_start, dtype=torch.int32, device=dev)
        cl = torch.tensor(ctx_len, dtype=torch.int32, device=dev)
        mc = max(lens)
        for alibi in (None, torch.linspace(0.01, 0.2, h, device=dev)):
            got = ops.ragged_attention(q, kc, vc, ss, cl, D ** -0.5, mc, alibi)
            old = P.global_config.use_native_kernels
            P.global_config.use_native_kernels = False
            try:
                ref = ops.ragged_attention(q.float(), kc.float(), vc.float(), ss, cl, D ** -0.5, mc, alibi)
            finally:
                P.global_config.use_native_kernels = old
            check(fails, f"ragged_attention h{h} D{D} T{T} alibi={alibi is not None}", got, ref, 2e-2, 2e-2)
    assert not fails, "\n".join(fails)


def test_forward_1d_on_gpu_matches_padded_forward():
    """A mixed iteration (new prompt + running decode) through the ragged kernel and the native cache manager gives
    the logits of the padded per-sequence forward (flash-attention kernel) up to bf16 rounding."""
    from alpa_b200 import _planner
    from alpa_b200.model.opt_model import DecoderLM, OPTConfig
    torch.manual_seed(0)
    cfg = OPTConfig(vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=4, ffn_dim=1024,
                    max_position_embeddings=256, dtype=torch.bfloat16)
    m = DecoderLM(cfg, device="cuda")
    a, b = torch.randint(3, 512, (1, 70), device="cuda"), torch.randint(3, 512, (1, 33), device="cuda")

    def full(ids):
        T = ids.shape[1]
        return m.forward(ids, torch.arange(T, device="cuda")[None], m.init_cache(1, T), 0, last_only=False)[0].float()
    fa, fb = full(a), full(b)
    mgr = _planner.KVCacheManager(256)
    cache = m.init_cache_1d(256)
    mgr.allocate(1, 128)
    mgr.allocate(2, 64)

    def run(prompt_ids, prompt_tokens, decode_ids, decode_tokens, budget=128):
        idx = mgr.prepare_inputs(prompt_ids, [len(t) for t in prompt_tokens], decode_ids, budget, 256)
        toks = [x for t in prompt_tokens for x in t] + decode_tokens
        toks += [1] * (budget - len(toks))
        T = lambda x, dt: torch.tensor(x, dtype=dt, device="cuda")  # noqa: E731
        return m.forward_1d(T(toks, torch.long), T(idx["position"], torch.long), T(idx["slot"], torch.long),
                            T(idx["seq_start"], torch.int32), T(idx["ctx_len"], torch.int32), cache, 128,
                            T(idx["logit_index"], torch.long)).float()
    l0 = run([1], [a[0, :69].tolist()], [], [])
    l1 = run([2], [b[0].tolist()], [1], [int(a[0, 69])])
    scale = fa.abs().max().item()
    for got, ref in ((l0[0], fa[68]), (l1[0], fb[32]), (l1[1], fa[69])):
        assert (got - ref).abs().max().item() < 0.04 * scale + 0.02, ((got - ref).abs().max().item(), scale)


def test_dropout_kernel_matches_reference_mask():
    """The CUDA Philox dropout and the torch int64 reference produce identical masks, for whole tensors (vectorised
    path), odd shapes (scalar path) and shards of a larger tensor."""
    from alpa_b200 import ops
    seed = torch.tensor(987654321012, dtype=torch.int64, device="cuda")
    for shape, gshape, off in (((64, 1024), (64, 1024), (0, 0)), ((7, 33), (7, 33), (0, 0)),
                               ((4, 16, 128), (8, 32, 512), (4, 16, 256)), ((5, 6), (10, 12), (5, 6))):
        for dt in (torch.bfloat16, torch.float32):
            x = torch.randn(*shape, device="cuda", dtype=dt)
            y = ops.dropout(x, 0.3, seed, 5, list(gshape), list(off))
            keep = ops.dropout_keep_mask(shape, 0.3, seed, 5, gshape, off, device="cuda")
            ref = torch.where(keep, x.float() / 0.7, torch.zeros((), device="cuda")).to(dt)
            assert torch.equal(y != 0, keep & (x != 0)), (shape, dt)
            assert torch.allclose(y.float(), ref.float(), rtol=1e-2, atol=1e-3), (shape, dt)

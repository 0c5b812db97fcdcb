"""GPU checks of the iteration-level batching path (new this round; runs after the other GPU tests)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


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

"""Serving Llama-style models without a GPU: `DecoderLM(arch="llama")` against Hugging Face `LlamaForCausalLM` and
`GPTModel(arch="llama")` with the same parameters (prompt logits, greedy generation), its cached decode, chunked
prefill, ragged batches, beam search and tensor parallelism, the .npy loader, and the float64 rule that the GPU tests
apply to the grouped decode kernel (it must reject the results of the defects that kernel could have)."""
import os
import sys

import numpy as np
import pytest
import torch

from alpa_b200.model.gpt_model import GPTModel, llama_config_from_hf, llama_params_from_hf
from alpa_b200.model.opt_model import (DecoderLM, OPTConfig, get_config, gpt_config_from_serving,
                                       serving_config_from_gpt)
from alpa_b200.ops import primitives as P
from alpa_b200.serve.generator import Generator, load_params_np
from alpa_b200.testing import assert_allclose

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import BF16, F64, _bf, bf16_rule  # noqa: E402

transformers = pytest.importorskip("transformers")
from transformers import LlamaConfig, LlamaForCausalLM  # noqa: E402

V = 96


def _hf(kv, tied, seed=0, layers=2):
    torch.manual_seed(seed)
    cfg = LlamaConfig(vocab_size=V, hidden_size=64, intermediate_size=96, num_hidden_layers=layers,
                      num_attention_heads=4, num_key_value_heads=kv, max_position_embeddings=128, rms_norm_eps=1e-5,
                      tie_word_embeddings=tied, rope_theta=10000.0)
    return LlamaForCausalLM(cfg).float().eval()


def _served(hf, **kw):
    gcfg = llama_config_from_hf(hf.config, dtype=torch.float32)
    params = llama_params_from_hf(hf.state_dict(), gcfg)
    return DecoderLM(serving_config_from_gpt(gcfg, **kw), device="cpu", params=params), gcfg, params


CASES = [(kv, tied) for kv in (1, 2, 4) for tied in (False, True)]


@pytest.mark.parametrize("kv,tied", CASES)
def test_prompt_logits_match_hf_and_gpt_model(kv, tied):
    hf = _hf(kv, tied)
    m, gcfg, params = _served(hf)
    ids = torch.randint(0, V, (2, 13), generator=torch.Generator().manual_seed(1))
    pos = torch.arange(13).repeat(2, 1)
    got = Generator(m, 2, 32).forward(ids)
    with torch.no_grad():
        want = hf(input_ids=ids).logits
        gm = GPTModel(gcfg)
        gm.load_state_dict(params)
        want_gpt = gm(ids, pos)
    assert_allclose(got, want, 1e-4, 1e-4)
    assert_allclose(got, want_gpt, 1e-4, 1e-4)


@pytest.mark.parametrize("kv,tied", CASES)
def test_greedy_generate_matches_hf(kv, tied):
    hf = _hf(kv, tied, seed=2)
    m, _, _ = _served(hf)
    ids = torch.randint(0, V, (2, 7), generator=torch.Generator().manual_seed(3))
    out = Generator(m, 2, 32).generate(ids, max_new_tokens=8)
    hf.generation_config.eos_token_id = None              # generate all 8 tokens, as Generator does without an EOS
    with torch.no_grad():
        want = hf.generate(ids, attention_mask=torch.ones_like(ids), max_new_tokens=8, do_sample=False,
                           pad_token_id=0)
    assert torch.equal(out.sequences, want), (out.sequences, want)


@pytest.mark.parametrize("kv", [1, 2, 4])
def test_cached_decode_and_decode_step_equal_recompute(kv):
    m, _, _ = _served(_hf(kv, False, seed=4))
    B, T, N = 2, 6, 5
    ids = torch.randint(0, V, (B, T + N), generator=torch.Generator().manual_seed(5))
    full = m.forward(ids, torch.arange(T + N).repeat(B, 1), m.init_cache(B, T + N), 0, last_only=False)
    cache, cache2 = m.init_cache(B, 32), m.init_cache(B, 32)
    m.forward(ids[:, :T], torch.arange(T).repeat(B, 1), cache, 0)
    m.forward(ids[:, :T], torch.arange(T).repeat(B, 1), cache2, 0)
    for t in range(T, T + N):
        pos = torch.full((B, 1), t)
        step = m.forward(ids[:, t:t + 1], pos, cache, t)
        dec = m.decode_step(ids[:, t:t + 1], pos, cache2, torch.tensor(t + 1, dtype=torch.int32))
        assert_allclose(step[:, 0], full[:, t], 1e-4, 1e-4)
        assert_allclose(dec, step, 1e-4, 1e-4)
    for (k1, v1), (k2, v2) in zip(cache, cache2):
        assert_allclose(k1, k2, 1e-5, 1e-5)
        assert_allclose(v1, v2, 1e-5, 1e-5)


def test_chunked_prefill_equals_single_pass():
    m, _, _ = _served(_hf(2, False, seed=6))
    ids = [list(range(3, 3 + 19))]
    a = Generator(m, 1, 40).generate(ids, max_new_tokens=6)
    b = Generator(m, 1, 40, prefill_chunk=4).generate(ids, max_new_tokens=6)
    assert torch.equal(a.sequences, b.sequences)


@pytest.mark.parametrize("kv", [1, 2])
def test_unequal_prompts_equal_solo_generation(kv):
    """Prompts of different lengths run as a ragged 1-D batch (SequenceGenerator, the model worker's engine, over the
    grouped ragged attention); each equals its own greedy generation."""
    m, _, _ = _served(_hf(kv, True, seed=7))
    prompts = [[5, 6, 7, 8, 9, 10, 11], [12, 13, 14], [20, 21, 22, 23, 24]]
    out = Generator(m, 4, 40).generate(prompts, max_new_tokens=6)
    for i, p in enumerate(prompts):
        solo = Generator(m, 1, 40).generate([p], max_new_tokens=6).sequences[0]
        assert out.sequences[i, :len(solo)].tolist() == solo.tolist()


def test_beam_search_runs():
    m, _, _ = _served(_hf(2, False, seed=8))
    out = Generator(m, 4, 40).generate([[3, 4, 5, 6]], max_new_tokens=5, num_beams=3)
    assert out.sequences.shape[0] == 1 and out.sequences.shape[1] >= 5
    assert out.sequences[0, :4].tolist() == [3, 4, 5, 6]


def _tp_worker(rank, world, port):
    """One rank of the tensor-parallel check: Llama (Hkv = 2 split over the ranks) served with tp = world generates what
    tp = 1 generates (same seed -> same full weights, sliced per rank)."""
    import torch.distributed as dist
    dist.init_process_group("gloo", init_method=f"tcp://127.0.0.1:{port}", rank=rank, world_size=world)
    try:
        cfg = OPTConfig(arch="llama", vocab_size=90, hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                        num_key_value_heads=2, ffn_dim=96, dtype=torch.float32)
        ref = DecoderLM(cfg, device="cpu", seed=5)
        tp = DecoderLM(cfg, device="cpu", group=dist.group.WORLD, seed=5)
        prompts = [[5, 6, 7, 8, 9], [9, 10, 11, 12, 13]]
        o_ref = Generator(ref, 2, 32).generate(prompts, max_new_tokens=5)
        o_tp = Generator(tp, 2, 32).generate(prompts, max_new_tokens=5)
        assert torch.equal(o_ref.sequences, o_tp.sequences), (o_ref.sequences, o_tp.sequences)
        print(f"rank {rank}: llama tp ok", flush=True)
    finally:
        dist.destroy_process_group()


def test_tensor_parallel_world2():
    import socket
    import subprocess
    here = os.path.dirname(os.path.abspath(__file__))
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    code = ("import sys; sys.path[:0] = [{!r}, {!r}]; import test_llama_serving as t; t._tp_worker({{}}, 2, {})"
            .format(os.path.dirname(here), here, port))
    procs = [subprocess.Popen([sys.executable, "-c", code.format(r)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT,
                              text=True) for r in range(2)]
    try:
        outs = [p.communicate(timeout=240)[0] for p in procs]
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
    for r, (p, out) in enumerate(zip(procs, outs)):
        assert p.returncode == 0 and f"rank {r}: llama tp ok" in out, out[-3000:]


def test_kv_heads_not_divisible_by_tp_raises():
    class Group:
        pass
    cfg = OPTConfig(arch="llama", vocab_size=V, hidden_size=64, num_hidden_layers=1, num_attention_heads=4,
                    num_key_value_heads=1, ffn_dim=96, dtype=torch.float32)
    import torch.distributed as dist
    orig = dist.get_world_size, dist.get_rank
    dist.get_world_size, dist.get_rank = (lambda g=None: 2), (lambda g=None: 0)
    try:
        with pytest.raises(ValueError, match="num_key_value_heads"):
            DecoderLM(cfg, device="cpu", group=Group())
    finally:
        dist.get_world_size, dist.get_rank = orig


def test_npy_loader_round_trips_hf_names(tmp_path):
    hf = _hf(2, False, seed=9)
    for name, t in hf.state_dict().items():
        if name.endswith(".weight"):
            with open(tmp_path / name, "wb") as f:
                np.save(f, t.numpy())
    m_ref, gcfg, params = _served(hf)
    cfg = serving_config_from_gpt(gcfg)
    loaded = load_params_np(cfg, str(tmp_path))
    assert set(loaded) == set(params)
    for k in params:
        assert torch.equal(loaded[k], params[k]), k
    assert gpt_config_from_serving(cfg) == gcfg
    m = DecoderLM(cfg, device="cpu", params=loaded)
    ids = torch.randint(0, V, (1, 9), generator=torch.Generator().manual_seed(9))
    assert torch.equal(Generator(m, 1, 16).forward(ids), Generator(m_ref, 1, 16).forward(ids))


def test_named_configs():
    c = get_config("llama-3-8b")
    assert (c.arch, c.num_key_value_heads, c.num_attention_heads, c.head_dim, c.rope_theta) == \
        ("llama", 8, 32, 128, 500000.0)
    assert not c.tie_word_embeddings
    assert get_config("llama-2-70b").num_key_value_heads == 8 and get_config("llama-2-7b").num_key_value_heads == 32
    with pytest.raises(ValueError):
        OPTConfig(arch="opt", num_attention_heads=4, num_key_value_heads=2)


def test_rms_linear_decode_reference():
    torch.manual_seed(0)
    x, w, g = torch.randn(3, 64), torch.randn(32, 64), torch.randn(64)
    y = P.linear_decode(x, w, None, ln=P.RMSNormArgs(g, 1e-5))
    want = torch.nn.functional.rms_norm(x, (64,), g, 1e-5) @ w.T
    assert_allclose(y, want, 1e-5, 1e-5)


def test_decode_attention_gqa_reference_matches_prefill():
    """The op's PyTorch path: rotate like rotary_packed, append, attend with query head g * ... of K/V head g // G."""
    torch.manual_seed(1)
    B, Hkv, G, D, n = 2, 2, 3, 32, 7
    qkv = torch.randn(B, n, Hkv, G + 2, D)
    pos = torch.arange(n).repeat(B, 1) + 50
    rot = P.rotary_packed(qkv, pos, 10000.0, False)
    want, _ = P.attention(rot[:, :, :, :G], rot[:, :, :, G], rot[:, :, :, G + 1], D ** -0.5, True)
    kc, vc = torch.zeros(B, 16, Hkv, D), torch.zeros(B, 16, Hkv, D)
    kc[:, :n - 1], vc[:, :n - 1] = rot[:, :n - 1, :, G], rot[:, :n - 1, :, G + 1]
    o = P.decode_attention_gqa(qkv[:, n - 1:], kc, vc, torch.tensor(n, dtype=torch.int32), pos[:, n - 1:],
                               D ** -0.5, 10000.0)
    assert_allclose(o.view(B, Hkv, G, D), want[:, -1], 1e-5, 1e-5)
    assert torch.equal(kc[:, n - 1], rot[:, n - 1, :, G]) and torch.equal(vc[:, n - 1], qkv[:, n - 1, :, G + 1])


def test_ragged_reference_groups_heads():
    torch.manual_seed(2)
    q, kc, vc = torch.randn(3, 4, 16), torch.randn(10, 2, 16), torch.randn(10, 2, 16)
    st, ln = torch.tensor([0, 0, 5], dtype=torch.int32), torch.tensor([3, 4, 2], dtype=torch.int32)
    got = P.ragged_attention(q, kc, vc, st, ln, 0.25, 8)
    want = P.ragged_attention(q, kc.repeat_interleave(2, 1), vc.repeat_interleave(2, 1), st, ln, 0.25, 8)
    assert_allclose(got, want, 0, 0)


# ---- the rule the GPU tests apply rejects the grouped decode kernel's possible defects ------------------------------
def gqa_decode_ref(qkv_rot, k, v, scale):
    """o [B, Hkv, G, D] float64 of the rotated packed row qkv_rot [B, Hkv, G + 2, D] over k / v [B, n, Hkv, D]."""
    G = qkv_rot.shape[2] - 2
    s = torch.einsum("bhgd,bnhd->bhgn", qkv_rot[:, :, :G].to(F64), k.to(F64)) * scale
    return torch.einsum("bhgn,bnhd->bhgd", torch.softmax(s, -1), v.to(F64))


def test_rule_rejects_gqa_decode_defects():
    g = torch.Generator().manual_seed(0)
    B, Hkv, G, D, n, theta = 2, 2, 4, 128, 512, 500000.0
    scale = D ** -0.5
    pos = torch.full((B, 1), n - 1 + 3000)
    qkv = (torch.randn(B, 1, Hkv, G + 2, D, generator=g) * 2).to(BF16)
    k = torch.randn(B, n, Hkv, D, generator=g).to(BF16)
    v = torch.randn(B, n, Hkv, D, generator=g).to(BF16)
    rot = P.rotary_packed(qkv.float(), pos, theta, False).to(BF16)[:, 0]
    k[:, n - 1], v[:, n - 1] = rot[:, :, G], rot[:, :, G + 1]
    ref = gqa_decode_ref(rot, k, v, scale)
    base = _bf(ref)
    assert not bf16_rule("baseline", base, ref, base)[0]
    k_unrot = k.clone()
    k_unrot[:, n - 1] = qkv[:, 0, :, G]
    rot_wrong = P.rotary_packed(qkv.float(), pos - 1, theta, False).to(BF16)[:, 0]
    k_wrong = k.clone()
    k_wrong[:, n - 1] = rot_wrong[:, :, G]
    # query head g (of all Hkv * G) paired with K/V head g (mod Hkv) instead of g // G
    q_flat = rot[:, :, :G].reshape(B, Hkv * G, D)
    kv_of = torch.arange(Hkv * G) % Hkv
    s = torch.einsum("bhd,bnhd->bhn", q_flat.to(F64), k[:, :, kv_of].to(F64)) * scale
    wrong_head = torch.einsum("bhn,bnhd->bhd", torch.softmax(s, -1), v[:, :, kv_of].to(F64)).view(B, Hkv, G, D)
    wrong = {
        "attends to the unrotated new key": gqa_decode_ref(rot, k_unrot, v, scale),
        "rotates by the wrong position": gqa_decode_ref(torch.cat([rot_wrong[:, :, :G], rot[:, :, G:]], 2), k_wrong,
                                                        v, scale),
        "query head g reads K/V head g": wrong_head,
    }
    for name, w in wrong.items():
        assert bf16_rule(name, _bf(w), ref, base)[0], name

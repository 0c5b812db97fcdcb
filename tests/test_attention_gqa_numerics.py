"""Grouped-query attention kernels on the GPU.

* Forward: a grouped call computes, per query head, exactly what the multi-head kernel computes on K/V expanded to one
  head per query head, so O and lse must equal that bit for bit.  Checked in a child process per forward configuration
  (ALPA_B200_ATTN_FWD = gen4 / gen2), like tests/test_kernel_numerics.py's forward matrix.
* Backward: dQ, dK and dV against float64 under `bf16_rule` of tests/test_kernel_numerics.py.  The reference and
  baseline are the expanded-head ones of `attn_bwd_ref`, with dK / dV summed over each group in float64 and rounded to
  bf16 once (the kernel accumulates a group in fp32 and rounds once).  Shapes on both sides of the dK / dV group split.
* The packed op's slot writes, its equality with `attention_qkvpacked` for groups of one, run-to-run reproducibility,
  and one bf16 training step of a GQA GPTModel.
"""
import json
import os
import subprocess
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import (BF16, F64, Checker, _bf, _bhsd, _report, attn_bwd_terms,  # noqa: E402
                                  attn_fwd_ref, visible)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _inputs(B, Sq, Skv, Hkv, G, D, seed, packed=False):
    """q [B,Sq,Hkv,G,D], k / v [B,Skv,Hkv,D], do like q; packed: views of one [B,S,Hkv,G+2,D] tensor (Sq == Skv)."""
    gen = torch.Generator(device="cuda").manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=gen, device="cuda").to(BF16)  # noqa: E731
    do = rn(B, Sq, Hkv, G, D)
    if packed:
        qkv = rn(B, Sq, Hkv, G + 2, D)
        return qkv[:, :, :, :G], qkv[:, :, :, G], qkv[:, :, :, G + 1], do, qkv
    return rn(B, Sq, Hkv, G, D), rn(B, Skv, Hkv, D), rn(B, Skv, Hkv, D), do, None


def _expand(q, k, v):
    """The multi-head operands of a grouped call: q [B,Sq,Hq,D] (contiguous), K/V repeated per query head."""
    B, Sq, Hkv, G, D = q.shape
    return q.reshape(B, Sq, Hkv * G, D).contiguous(), k.repeat_interleave(G, 2), v.repeat_interleave(G, 2)


# ---------------------------------------------------------------------------------------------------------------------
# forward: bit-exact against the multi-head kernel on expanded K/V
# ---------------------------------------------------------------------------------------------------------------------
def _fwd_cases():
    cases = []
    for D in (64, 80, 128):
        for G in (1, 2, 4, 8):
            for Hkv in (1, 2):
                cases += [dict(D=D, G=G, Hkv=Hkv, Sq=200, Skv=200, causal=True, packed=True),
                          dict(D=D, G=G, Hkv=Hkv, Sq=200, Skv=200, causal=False, packed=False),
                          dict(D=D, G=G, Hkv=Hkv, Sq=100, Skv=300, causal=True, packed=False),
                          dict(D=D, G=G, Hkv=Hkv, Sq=300, Skv=100, causal=True, packed=False),
                          dict(D=D, G=G, Hkv=Hkv, Sq=130, Skv=130, causal=False, packed=True)]
    for causal in (False, True):
        for L in (0, 1, 63, 64, 65, 192, 199):
            cases.append(dict(D=64, G=4, Hkv=2, Sq=65, Skv=192, causal=causal, packed=False, kv_len=L))
    return cases


def _fwd_child_main():
    from alpa_b200 import ops
    C = ops.native_module()
    fails = []
    cases = _fwd_cases()
    for i, c in enumerate(cases):
        B = 2
        q, k, v, _, _ = _inputs(B, c["Sq"], c["Skv"], c["Hkv"], c["G"], c["D"], 300 + i, c["packed"])
        kl = None if "kv_len" not in c else torch.tensor([c["kv_len"]], dtype=torch.int32, device="cuda")
        scale = c["D"] ** -0.5
        o, lse = C.attention_fwd(q, k, v, scale, c["causal"], kl)
        oe, lsee = C.attention_fwd(*_expand(q, k, v), scale, c["causal"], kl)
        Hq = c["Hkv"] * c["G"]
        if tuple(o.shape) != tuple(q.shape) or tuple(lse.shape) != (B, c["Hkv"], c["G"], c["Sq"]):
            fails.append(f"{c}: output shapes {tuple(o.shape)} {tuple(lse.shape)}")
        elif not (torch.equal(o.reshape(B, c["Sq"], Hq, c["D"]), oe) and torch.equal(lse.reshape(B, Hq, c["Sq"]), lsee)):
            fails.append(f"{c}: grouped O / lse differ from the multi-head kernel on expanded K/V")
    torch.cuda.synchronize()
    print(json.dumps({"config": os.environ.get("ALPA_B200_ATTN_FWD", "gen4"), "cases": len(cases), "fails": fails}),
          flush=True)
    return 0


@pytest.mark.gpu
@pytest.mark.parametrize("config", ["gen4", "gen2"])
def test_gqa_forward_equals_expanded_mha(config):
    env = dict(os.environ, ALPA_B200_ATTN_FWD=config)
    env["PYTHONPATH"] = ROOT + os.pathsep + env.get("PYTHONPATH", "")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), "fwd"]
    r = subprocess.run(cmd, env=env, cwd=ROOT, capture_output=True, text=True, timeout=900)
    lines = [ln for ln in r.stdout.splitlines() if ln.startswith("{")]
    assert r.returncode == 0 and lines, f"child exited with {r.returncode}:\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    res = json.loads(lines[-1])
    assert res["config"] == config and res["cases"] == len(_fwd_cases())
    assert not res["fails"], "\n".join(res["fails"])


# ---------------------------------------------------------------------------------------------------------------------
# backward: float64 reference with the group summed once
# ---------------------------------------------------------------------------------------------------------------------
def gqa_bwd_ref(do, q, k, v, o, lse, scale, vis, G, rounded):
    """(dq [B,Sq,Hq,D], dk, dv [B,Skv,Hkv,D]) in float64 from expanded-head operands (as `attn_bwd_ref`); dK / dV are
    summed over each group of G query heads in float64.  rounded=True rounds P and dS before their products and each
    result once, to bf16 (the baseline)."""
    qf, kf, vf, dof, of = _bhsd(q), _bhsd(k), _bhsd(v), _bhsd(do), _bhsd(o)
    lse = lse.to(F64)
    s = (qf @ kf.transpose(-1, -2) * scale).masked_fill(~vis, float("-inf"))
    p = torch.exp(s - lse.masked_fill(lse == float("-inf"), 0.0)[..., None])
    r = _bf if rounded else (lambda t: t)
    dv = r(p).transpose(-1, -2) @ dof
    ds = r(p * (dof @ vf.transpose(-1, -2) - (dof * of).sum(-1, keepdim=True)))
    dq = ds @ kf * scale
    dk = ds.transpose(-1, -2) @ qf * scale
    B, Hq, Skv, D = dk.shape
    gsum = lambda t: t.view(B, Hq // G, G, Skv, D).sum(2)  # noqa: E731
    return tuple(r(t.permute(0, 2, 1, 3)) for t in (dq, gsum(dk), gsum(dv)))


BWD_CASES = [  # (B, Sq, Skv, Hkv, G, D, causal): the dK / dV grid B * Hkv * ceil(Skv / 64) against 2 x 132 SMs
    (1, 4096, 4096, 1, 8, 128, True),     # 64 CTAs: split into 8 (the tensor-parallel 70B-like shape)
    (2, 2048, 2048, 4, 4, 128, True),     # 256 CTAs: split into 2, two heads per part
    (2, 100, 300, 2, 4, 80, True),        # Sq != Skv, split
    (2, 300, 100, 2, 4, 64, True),        # rows without keys, split
    (4, 1024, 1024, 8, 2, 64, False),     # 512 CTAs: unsplit
    (2, 1024, 1024, 8, 4, 128, True),     # 256 CTAs: split into 2
    (8, 512, 512, 8, 4, 64, False),       # 512 CTAs: unsplit
]


@pytest.mark.gpu
@pytest.mark.parametrize("B,Sq,Skv,Hkv,G,D,causal", BWD_CASES)
def test_gqa_backward(B, Sq, Skv, Hkv, G, D, causal):
    from alpa_b200 import ops
    C = ops.native_module()
    q, k, v, do, _ = _inputs(B, Sq, Skv, Hkv, G, D, Sq + 7 * G + D)
    scale = D ** -0.5
    splits = C.attention_bwd_splits(q, k, v)
    ctas = B * Hkv * ((Skv + 63) // 64)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert (splits > 1) == (ctas < 2 * sms) and G % splits == 0
    if (B, Sq, Hkv) == (1, 4096, 1):
        assert splits > 1, "one K/V head at B = 1, S = 4096 must take the split path"
    o, lse = C.attention_fwd(q, k, v, scale, causal)
    dq, dk, dv = C.attention_bwd(do, q, k, v, o, lse, scale, causal)
    qe, ke, ve = _expand(q, k, v)
    Hq = Hkv * G
    vis = visible(Sq, Skv, causal, device="cuda")
    oe, doe = o.reshape(B, Sq, Hq, D), do.reshape(B, Sq, Hq, D)
    ref_o, ref_lse = attn_fwd_ref(qe, ke, ve, scale, vis)
    base_o, _ = attn_fwd_ref(qe, ke, ve, scale, vis, p_round=_bf)
    ref = gqa_bwd_ref(doe, qe, ke, ve, ref_o, ref_lse, scale, vis, G, rounded=False)
    base = gqa_bwd_ref(doe, qe, ke, ve, base_o, ref_lse, scale, vis, G, rounded=True)
    tq, tk, tv = attn_bwd_terms(doe, qe, ke, ve, ref_o, ref_lse, scale, vis)
    terms = (tq, tk.view(B, Skv, Hkv, G, D).sum(3), tv.view(B, Skv, Hkv, G, D).sum(3))
    del oe
    ck = Checker()
    name = f"gqa bwd B{B} q{Sq} k{Skv} Hkv{Hkv} G{G} D{D} {'causal' if causal else 'full'} splits={splits}"
    for nm, got, r, b, t in zip(("dq", "dk", "dv"), (dq.reshape(B, Sq, Hq, D), dk, dv), ref, base, terms):
        ck.bf16(f"gqa bwd {nm}", f"{name} {nm}", got, r, b, t)
    empty = ~vis.any(-1)
    if empty.any():
        ck.require(bool((dq[:, empty] == 0).all()), f"{name}: rows without keys have dq != 0")
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,Hkv,G,D", [(1, 4096, 1, 8, 128), (4, 1024, 8, 2, 64)])
def test_gqa_backward_is_reproducible(B, S, Hkv, G, D):
    from alpa_b200 import ops
    C = ops.native_module()
    q, k, v, do, _ = _inputs(B, S, S, Hkv, G, D, 17)
    o, lse = C.attention_fwd(q, k, v, D ** -0.5, True)
    a = C.attention_bwd(do, q, k, v, o, lse, D ** -0.5, True)
    b = C.attention_bwd(do, q, k, v, o, lse, D ** -0.5, True)
    for nm, x, y in zip(("dq", "dk", "dv"), a, b):
        assert torch.equal(x, y), f"{nm} differs between two runs (splits {C.attention_bwd_splits(q, k, v)})"


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,Hkv,G,D", [(2, 200, 2, 4, 80), (4, 1024, 8, 2, 64), (2, 256, 3, 1, 64)])
def test_gqa_backward_into_packed_slots(B, S, Hkv, G, D):
    """attention_gqa_packed_bwd writes dQ / dK / dV into the slots of one [B,S,Hkv,G+2,D] buffer: every element of a
    slot is written, the other slots are not touched, and the values equal the contiguous outputs bit for bit."""
    from alpa_b200 import ops
    C = ops.native_module()
    q, k, v, do, qkv = _inputs(B, S, S, Hkv, G, D, 11, packed=True)
    scale = D ** -0.5
    o, lse = C.attention_fwd(q, k, v, scale, True)
    want = C.attention_bwd(do, q, k, v, o, lse, scale, True)
    slots = [slice(0, G), G, G + 1]
    full = torch.full_like(qkv, float("nan"))
    C.attention_bwd(do, q, k, v, o, lse, scale, True, *[full[:, :, :, s] for s in slots])
    assert not full.isnan().any(), "an element of a slot was not written"
    for i, s in enumerate(slots):
        assert torch.equal(full[:, :, :, s], want[i]), f"slot {i} differs from the contiguous result"
        one = torch.full_like(qkv, float("nan"))
        outs = [None, None, None]
        outs[i] = one[:, :, :, s]
        C.attention_bwd(do, q, k, v, o, lse, scale, True, *outs)
        assert torch.equal(one[:, :, :, s], want[i]), f"slot {i} written alone differs"
        rest = torch.ones(G + 2, dtype=torch.bool)
        rest[s] = False
        assert one[:, :, :, rest].isnan().all(), f"writing slot {i} touched another slot"
    assert torch.equal(ops.attention_gqa_packed_bwd(do, qkv, o, lse, scale, True), full)


@pytest.mark.gpu
@pytest.mark.parametrize("D,causal", [(64, True), (128, False), (80, True)])
def test_group_of_one_equals_qkvpacked(D, causal):
    from alpa_b200 import ops
    B, S, H = 2, 300, 3
    gen = torch.Generator(device="cuda").manual_seed(D)
    qkv = torch.randn(B, S, H, 3, D, generator=gen, device="cuda").to(BF16)
    scale = D ** -0.5
    o1, l1 = ops.attention_qkvpacked(qkv, scale, causal)
    o2, l2 = ops.attention_gqa_packed(qkv, scale, causal)
    assert torch.equal(o1, o2.view(B, S, H, D)) and torch.equal(l1, l2.view(B, H, S))
    do = torch.randn(B, S, H, D, generator=gen, device="cuda").to(BF16)
    g1 = ops.attention_qkvpacked_bwd(do, qkv, o1, l1, scale, causal)
    g2 = ops.attention_gqa_packed_bwd(do.view(B, S, H, 1, D), qkv, o2, l2, scale, causal)
    assert torch.equal(g1, g2)


@pytest.mark.gpu
def test_gqa_gpt_trains_one_step_natively():
    """A small GQA GPTModel trains one bf16 step through alpa.parallelize on the native kernels only; its loss matches
    the same step on the PyTorch path."""
    import alpa_b200 as alpa
    from alpa_b200 import ops
    from alpa_b200.model.gpt_model import GPTConfig, GPTModel, gpt_lm_loss
    from alpa_b200.model.model_util import TrainState, functional_call, params_of, sgd
    from alpa_b200.ops.primitives import library_fallbacks

    def run(native):
        alpa.global_config.use_native_kernels = native
        alpa.init(cluster="local")
        try:
            cfg = GPTConfig(vocab_size=1024, hidden_size=512, num_hidden_layers=2, num_attention_heads=8,
                            num_key_value_heads=2, max_position_embeddings=256, causal=True, dtype=torch.bfloat16)
            torch.manual_seed(0)
            model = GPTModel(cfg, device="cuda")
            state = TrainState.create(apply_fn=None, params=params_of(model), tx=sgd(1e-2))
            g = torch.Generator().manual_seed(1)
            B, S = 4, 256
            batch = {"input_ids": torch.randint(1, 1024, (B, S), generator=g).cuda(),
                     "position_ids": torch.arange(S, device="cuda").repeat(B, 1),
                     "labels": torch.randint(1, 1024, (B, S), generator=g).cuda()}

            def train_step(state, batch):
                def loss_fn(p):
                    return gpt_lm_loss(functional_call(model, p, (batch["input_ids"], batch["position_ids"])),
                                       batch["labels"])
                loss, grads = alpa.value_and_grad(loss_fn)(state.params)
                return state.apply_gradients(grads=grads), loss

            step = alpa.parallelize(train_step, method=alpa.ShardParallel(), donate_argnums=(0,))
            n0 = ops.native_module().launch_count()
            state, loss = step(state, batch)
            torch.cuda.synchronize()
            launches = ops.native_module().launch_count() - n0
            text = step.get_last_executable().get_hlo_text()
            return float(loss._value), launches, text
        finally:
            alpa.shutdown()
            alpa.global_config.use_native_kernels = True

    try:
        loss_n, launches, text = run(True)
        assert "attention_gqa_packed" in text and "attention_gqa_packed_bwd" in text
        assert launches > 0 and library_fallbacks() == [], library_fallbacks()
        loss_ref, _, _ = run(False)
    finally:
        alpa.clear_executable_cache()
    assert loss_n == loss_n and abs(loss_n - loss_ref) <= 1e-2 * abs(loss_ref), (loss_n, loss_ref)


if __name__ == "__main__":
    if sys.argv[1:] == ["fwd"]:
        sys.exit(_fwd_child_main())
    sys.exit(f"usage: {sys.argv[0]} fwd")

"""The Llama-style block without a GPU: the RMSNorm, rotary and SwiGLU primitives' PyTorch paths against independent
PyTorch / Hugging Face code, a converted HF `LlamaForCausalLM` against `GPTModel(arch="llama")` (logits and gradients),
the parameter set, and the planner's treatment of the new ops under each parallel method."""
import pytest
import torch
import torch.nn.functional as F

import alpa_b200 as alpa
from alpa_b200 import PipeshardParallel, ShardParallel, Zero3Parallel
from alpa_b200.model.gpt_model import (GPTConfig, GPTModel, gpt_lm_loss, llama_config_from_hf, llama_params_from_hf,
                                       num_params)
from alpa_b200.model.model_util import TrainState, functional_call, params_of, sgd
from alpa_b200.ops import primitives as P
from alpa_b200.parallel.pipeline.layer_construction import ManualLayerOption
from alpa_b200.parallel.pipeline.stage_construction import UniformStageOption
from alpa_b200.testing import assert_allclose, clone_state

transformers = pytest.importorskip("transformers")
from transformers import LlamaConfig, LlamaForCausalLM  # noqa: E402
from transformers.models.llama.modeling_llama import apply_rotary_pos_emb  # noqa: E402


# ---- primitives ----------------------------------------------------------------------------------------------------
def test_rms_norm_matches_torch():
    torch.manual_seed(0)
    x, r = torch.randn(3, 5, 48, requires_grad=True), torch.randn(3, 5, 48, requires_grad=True)
    g = torch.randn(48, requires_grad=True)
    y, rstd = P.rms_norm(x, g, 1e-5)
    ref = F.rms_norm(x, (48,), g, 1e-5)
    assert_allclose(y, ref, 1e-6, 1e-6)
    assert rstd.shape == (3, 5) and rstd.dtype == torch.float32
    dy = torch.randn_like(y)
    assert_allclose(torch.autograd.grad(y, (x, g), dy), torch.autograd.grad(ref, (x, g), dy), 1e-5, 1e-5)

    y2, s, _ = P.add_rms_norm(x, r, g, 1e-5)
    ref2 = F.rms_norm(x + r, (48,), g, 1e-5)
    assert_allclose(s, x + r, 0, 0)
    assert_allclose(y2, ref2, 1e-6, 1e-6)
    ds = torch.randn_like(s)
    got = torch.autograd.grad((y2, s), (x, r, g), (dy, ds))
    want = torch.autograd.grad((ref2, x + r), (x, r, g), (dy, ds))
    assert_allclose(got, want, 1e-5, 1e-5)


def _hf_rotary(q, k, pos, theta):
    """HF's rotary on q [B,S,nq,D], k [B,S,nk,D] with HF's own cos / sin."""
    D = q.shape[-1]
    inv = 1.0 / (theta ** (torch.arange(0, D, 2, dtype=torch.int64).float() / D))
    freqs = (inv[None, :, None] @ pos[:, None, :].float()).transpose(1, 2)
    emb = torch.cat((freqs, freqs), -1)
    qo, ko = apply_rotary_pos_emb(q.transpose(1, 2), k.transpose(1, 2), emb.cos(), emb.sin())
    return qo.transpose(1, 2), ko.transpose(1, 2)


@pytest.mark.parametrize("G,Hkv,D", [(1, 2, 16), (4, 2, 32), (2, 1, 64)])
def test_rotary_matches_hf(G, Hkv, D):
    torch.manual_seed(G + D)
    B, S, theta = 2, 9, 500000.0
    qkv = torch.randn(B, S, Hkv, G + 2, D, requires_grad=True)
    pos = torch.randint(0, 40000, (B, S))
    out = P.rotary_packed(qkv, pos, theta, False)
    q, k = _hf_rotary(qkv[:, :, :, :G].reshape(B, S, Hkv * G, D), qkv[:, :, :, G], pos, theta)
    assert_allclose(out[:, :, :, :G].reshape(B, S, Hkv * G, D), q, 1e-5, 1e-5)
    assert_allclose(out[:, :, :, G], k, 1e-5, 1e-5)
    assert torch.equal(out[:, :, :, G + 1], qkv[:, :, :, G + 1])
    assert_allclose(P.rotary_packed(out, pos, theta, True), qkv, 1e-5, 1e-5)
    # the gradient is the inverse rotation (an orthogonal map's transpose)
    dy = torch.randn_like(out)
    (got,) = torch.autograd.grad(out, qkv, dy)
    assert_allclose(got, P.rotary_packed(dy, pos, theta, True), 0, 0)
    ref = torch.cat([torch.cat([q.view(B, S, Hkv, G, D), k[:, :, :, None]], 3), qkv[:, :, :, G + 1:]], 3)
    (want,) = torch.autograd.grad(ref, qkv, dy)
    assert_allclose(got, want, 1e-5, 1e-5)


def test_rotary_position_ids_broadcast_and_int32():
    """HF passes one [1, S] row of positions for the batch; any integer dtype works."""
    torch.manual_seed(3)
    qkv = torch.randn(3, 10, 2, 4, 32)
    pos = torch.arange(5, 15)
    want = P.rotary_packed(qkv, pos.repeat(3, 1), 10000.0, False)
    assert torch.equal(P.rotary_packed(qkv, pos[None].to(torch.int32), 10000.0, False), want)
    assert torch.equal(P.rotary_packed(qkv, pos[None], 10000.0, False), want)


def test_swiglu_matches_torch():
    torch.manual_seed(1)
    gu = (torch.randn(3, 7, 12, 2) * 4).requires_grad_()
    h = P.swiglu(gu)
    g, u = gu[..., 0], gu[..., 1]
    ref = F.silu(g) * u
    assert_allclose(h, ref, 1e-6, 1e-6)
    dh = torch.randn_like(h)
    assert_allclose(torch.autograd.grad(h, gu, dh), torch.autograd.grad(ref, gu, dh), 1e-5, 1e-5)


# ---- Hugging Face parity -------------------------------------------------------------------------------------------
def _hf_model(kv, tied, seed=0):
    torch.manual_seed(seed)
    cfg = LlamaConfig(vocab_size=128, hidden_size=64, intermediate_size=96, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=kv, max_position_embeddings=64, rms_norm_eps=1e-5,
                      tie_word_embeddings=tied, rope_theta=10000.0)
    return LlamaForCausalLM(cfg).float().eval()


def _converted(hf, **kw):
    cfg = llama_config_from_hf(hf.config, dtype=torch.float32, **kw)
    model = GPTModel(cfg)
    params = llama_params_from_hf(hf.state_dict(), cfg)
    assert set(params) == set(params_of(model))
    return cfg, model, params


@pytest.mark.parametrize("kv", [4, 2])
@pytest.mark.parametrize("tied", [False, True])
def test_hf_llama_logits_and_grads(kv, tied):
    hf = _hf_model(kv, tied)
    cfg, model, params = _converted(hf)
    B, S = 2, 11
    ids = torch.randint(0, 128, (B, S))
    pos = torch.arange(S).repeat(B, 1) + torch.tensor([[0], [17]])
    labels = torch.randint(1, 128, (B, S))
    params = {k: v.clone().requires_grad_() for k, v in params.items()}
    logits = functional_call(model, params, (ids, pos))
    ref = hf(input_ids=ids, position_ids=pos).logits
    assert_allclose(logits, ref, 1e-5, 1e-5)

    loss = F.cross_entropy(logits.reshape(-1, 128), labels.reshape(-1))
    grads = dict(zip(params, torch.autograd.grad(loss, list(params.values()))))
    hf_loss = F.cross_entropy(hf(input_ids=ids, position_ids=pos).logits.reshape(-1, 128), labels.reshape(-1))
    names = [n for n, _ in hf.named_parameters()]
    hf_grads = dict(zip(names, torch.autograd.grad(hf_loss, [p for _, p in hf.named_parameters()])))
    want = llama_params_from_hf(hf_grads, cfg)        # HF's gradients in this model's layout
    for k in params:
        assert_allclose(grads[k], want[k], 1e-5, 1e-5)


@pytest.mark.parametrize("change,match", [
    (dict(rope_scaling={"rope_type": "linear", "factor": 2.0}), "rope"),
    (dict(attention_bias=True), "bias"),
    (dict(mlp_bias=True), "bias"),
    (dict(head_dim=32), "head_dim"),
    (dict(hidden_act="gelu"), "hidden_act"),
])
def test_hf_config_rejects_what_the_model_does_not_compute(change, match):
    cfg = LlamaConfig(vocab_size=128, hidden_size=64, intermediate_size=96, num_hidden_layers=1, num_attention_heads=4,
                      **change)
    with pytest.raises(ValueError, match=match):
        llama_config_from_hf(cfg)


def test_hf_config_rejects_sliding_window():
    cfg = LlamaConfig(vocab_size=128, hidden_size=64, intermediate_size=96, num_hidden_layers=1, num_attention_heads=4)
    cfg.sliding_window = 32
    with pytest.raises(ValueError, match="sliding"):
        llama_config_from_hf(cfg)


# ---- parameters ----------------------------------------------------------------------------------------------------
def _llama_cfg(kv=2, **kw):
    args = dict(arch="llama", vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=8,
                num_key_value_heads=kv, intermediate_size=384, max_position_embeddings=16, causal=True,
                dtype=torch.float32)
    args.update(kw)
    return GPTConfig(**args)


@pytest.mark.parametrize("tied", [False, True])
def test_llama_parameter_set(tied):
    cfg = _llama_cfg(tie_word_embeddings=tied)
    ps = params_of(GPTModel(cfg))
    blk = {"qkv_w": (cfg.qkv_features, 256), "proj_w": (256, 256), "ln1_g": (256,), "ln2_g": (256,),
           "fc1_w": (768, 256), "fc2_w": (256, 384)}
    want = {"wte": (512, 256), "ln_f_g": (256,), **({} if tied else {"decoder_w": (512, 256)})}
    want.update({f"blocks.{i}.{k}": v for i in range(2) for k, v in blk.items()})
    assert {k: tuple(v.shape) for k, v in ps.items()} == want
    assert num_params(cfg) == sum(v.numel() for v in ps.values())


def test_default_config_unchanged():
    """The default arch builds the GPT model it always built: the same parameter names and count, and bidirectional
    attention; arch="llama" attends causally unless told otherwise, and unsupported options raise."""
    cfg = GPTConfig(vocab_size=128, hidden_size=64, num_hidden_layers=2, num_attention_heads=4,
                    max_position_embeddings=8, dtype=torch.float32)
    assert cfg.arch == "gpt" and cfg.causal is False
    assert GPTConfig(arch="llama").causal is True and GPTConfig(arch="llama", causal=False).causal is False
    torch.manual_seed(0)
    model = GPTModel(cfg)
    names = {"wte", "wpe", "emb_ln_g", "emb_ln_b", "decoder_w", "decoder_b"} | {
        f"blocks.{i}.{k}" for i in range(2) for k in ("qkv_w", "qkv_b", "proj_w", "proj_b", "ln1_g", "ln1_b", "fc1_w",
                                                        "fc1_b", "fc2_w", "fc2_b", "ln2_g", "ln2_b")}
    assert set(params_of(model)) == names
    assert num_params(cfg) == sum(v.numel() for v in params_of(model).values())
    with pytest.raises(ValueError):
        GPTConfig(arch="llama", hidden_dropout_prob=0.1)
    with pytest.raises(ValueError):
        GPTConfig(arch="mamba")


# ---- planner -------------------------------------------------------------------------------------------------------
def _train(cfg, method, B=4, shared_positions=False):
    """One SGD step of the serial and the parallel train step against each other (tolerances of
    tests/test_attention_gqa.py); returns the parallel state and executable.  shared_positions: one int32 [1, S] row of
    positions for the whole batch, as HF passes them."""
    torch.manual_seed(0)
    model = GPTModel(cfg)
    state = TrainState.create(apply_fn=None, params=params_of(model), tx=sgd(1e-2))
    S = cfg.max_position_embeddings
    pos = (torch.arange(S, dtype=torch.int32)[None] if shared_positions
           else torch.arange(S).repeat(B, 1) + torch.arange(B)[:, None] * 3)
    batch = {"input_ids": torch.randint(1, cfg.vocab_size, (B, S)), "position_ids": pos,
             "labels": torch.randint(1, cfg.vocab_size, (B, S))}

    def train_step(state, batch):
        def loss_fn(p):
            return gpt_lm_loss(functional_call(model, p, (batch["input_ids"], batch["position_ids"])), batch["labels"])
        loss, grads = alpa.value_and_grad(loss_fn)(state.params)
        return state.apply_gradients(grads=grads), loss

    expected, eloss = train_step(clone_state(state), batch)
    p_step = alpa.parallelize(train_step, method=method, donate_argnums=(0,))
    actual, loss = p_step(clone_state(state), batch)
    assert_allclose(eloss, loss, 1e-4, 1e-4)
    assert_allclose(expected.params, actual.params, 2e-3, 2e-3)
    return actual, p_step.get_last_executable()


_AB = torch.ops.alpa_b200


def _assert_pairs_and_slots_whole(ex):
    """No plan shards the SwiGLU pair dim or the rotary slot / D dims."""
    seen = set()
    for node, plans in ex.program.plan.node_plans.items():
        t = node.target
        if t not in (_AB.swiglu.default, _AB.swiglu_bwd.default, _AB.rotary_packed.default):
            continue
        for plan in (plans if isinstance(plans, (list, tuple)) else [plans]):
            if t == _AB.rotary_packed.default:
                spec = plan.in_specs[0]
                assert spec.num_shards(3) == 1 and spec.num_shards(4) == 1, (node.name, str(spec))
            else:
                i = 1 if t == _AB.swiglu_bwd.default else 0
                pair_dim = node.args[i].meta["val"].dim() - 1
                assert plan.in_specs[i].num_shards(pair_dim) == 1, (node.name, str(plan.in_specs[i]))
            seen.add(t)
    assert seen == {_AB.swiglu.default, _AB.swiglu_bwd.default, _AB.rotary_packed.default}, seen


@pytest.mark.parametrize("shape", [(1, 4), (2, 2)])
def test_shard_parallel(local_mesh4, shape):
    actual, ex = _train(_llama_cfg(), ShardParallel(devices=local_mesh4.get_logical_mesh(shape)))
    _assert_pairs_and_slots_whole(ex)
    text = ex.get_hlo_text()
    assert all(op in text for op in ("rotary_packed", "swiglu", "add_rms_norm", "rms_norm_bwd"))
    if shape == (1, 4):
        for i in range(2):
            assert str(actual.params[f"blocks.{i}.fc1_w"].sharding_spec) == "S1R"   # column parallel


def test_shard_parallel_shared_positions(local_mesh4):
    """position_ids broadcast over the batch ([1, S], int32) while the batch dim of qkv shards."""
    _, ex = _train(_llama_cfg(), ShardParallel(devices=local_mesh4.get_logical_mesh((4, 1))), shared_positions=True)
    _assert_pairs_and_slots_whole(ex)


def test_zero3(local_mesh4):
    _train(_llama_cfg(), Zero3Parallel(devices=local_mesh4.get_logical_mesh((4, 1))))


def test_pipeshard_two_stages(local_mesh4):
    """Two stages: the second stage's blocks read position_ids (a step input) and the (branch, residual) pair."""
    cfg = _llama_cfg(add_manual_pipeline_markers=True, pipeline_mp_size=2)
    method = PipeshardParallel(num_micro_batches=2, layer_option=ManualLayerOption(),
                               stage_option=UniformStageOption(num_stages=2))
    _, ex = _train(cfg, method, B=8)
    assert ex.config.num_meshes == 2

"""Grouped-query attention without a GPU: the primitives' PyTorch path against torch's SDPA with `enable_gqa`, the
planner's treatment of `attention_gqa_packed` (only batch and K/V heads shard, a group is never split), and a GQA
GPTModel trained under each parallel method against the single-device step."""
import pytest
import torch
import torch.nn.functional as F

import alpa_b200 as alpa
from alpa_b200 import PipeshardParallel, ShardParallel, Zero3Parallel
from alpa_b200.model.gpt_model import GPTConfig, GPTModel, gpt_lm_loss, num_params
from alpa_b200.model.model_util import TrainState, functional_call, params_of, sgd
from alpa_b200.ops import primitives as P
from alpa_b200.parallel.pipeline.layer_construction import ManualLayerOption
from alpa_b200.parallel.pipeline.stage_construction import UniformStageOption
from alpa_b200.testing import assert_allclose, clone_state


def _sdpa(q, k, v, scale, causal):
    """torch's GQA attention on q [B,Sq,Hkv,G,D], k / v [B,Skv,Hkv,D]; causal aligned to the last key (as the kernels)."""
    B, Sq, Hkv, G, D = q.shape
    Skv = k.shape[1]
    qh = q.reshape(B, Sq, Hkv * G, D).transpose(1, 2)
    mask = None
    if causal:
        mask = torch.ones(Sq, Skv, dtype=torch.bool).tril(Skv - Sq)
    o = F.scaled_dot_product_attention(qh, k.transpose(1, 2), v.transpose(1, 2), attn_mask=mask, scale=scale,
                                       enable_gqa=True)
    return o.transpose(1, 2).reshape(B, Sq, Hkv, G, D)


@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("Hkv", [1, 2, 4])
@pytest.mark.parametrize("causal", [False, True])
def test_packed_op_matches_sdpa(G, Hkv, causal):
    torch.manual_seed(G * 10 + Hkv)
    B, S, D = 2, 19, 16
    qkv = torch.randn(B, S, Hkv, G + 2, D, requires_grad=True)
    o, lse = P.attention_gqa_packed(qkv, 0.3, causal)
    assert o.shape == (B, S, Hkv, G, D) and lse.shape == (B, Hkv, G, S)
    ref = _sdpa(qkv[:, :, :, :G], qkv[:, :, :, G], qkv[:, :, :, G + 1], 0.3, causal)
    assert_allclose(o, ref, 1e-5, 1e-5)
    g = torch.randn_like(o)
    got, = torch.autograd.grad(o, qkv, g)
    want, = torch.autograd.grad(ref, qkv, g)
    assert_allclose(got, want, 1e-5, 1e-5)


@pytest.mark.parametrize("G", [1, 2, 4])
@pytest.mark.parametrize("Hkv", [1, 2, 4])
@pytest.mark.parametrize("causal", [False, True])
@pytest.mark.parametrize("Sq,Skv", [(13, 29), (29, 13)])
def test_reference_path_with_unequal_lengths(G, Hkv, causal, Sq, Skv):
    """The unpacked maths the packed op's PyTorch path runs, at Sq != Skv: outputs and gradients match SDPA on the rows
    that see a key; rows that see none (causal, Sq > Skv) give O = 0 and zero dQ instead of NaN."""
    torch.manual_seed(Sq + G)
    B, D = 2, 8
    q = torch.randn(B, Sq, Hkv, G, D, requires_grad=True)
    k = torch.randn(B, Skv, Hkv, D, requires_grad=True)
    v = torch.randn(B, Skv, Hkv, D, requires_grad=True)
    do = torch.randn(B, Sq, Hkv, G, D)
    o, lse = P._gqa_attn_ref(q, k, v, 0.5, causal)
    dq, dk, dv = P._gqa_attn_ref_bwd(do, q, k, v, o, lse, 0.5, causal)
    empty = max(0, Sq - Skv) if causal else 0            # leading query rows without a visible key
    assert (o[:, :empty] == 0).all() and (dq[:, :empty] == 0).all()
    assert torch.isfinite(dk).all() and torch.isfinite(dv).all()
    ref = _sdpa(q, k, v, 0.5, causal)
    ref_o = torch.cat([torch.zeros_like(ref[:, :empty]), ref[:, empty:]], 1)   # SDPA gives NaN on empty rows
    assert_allclose(o, ref_o, 1e-5, 1e-5)
    want = torch.autograd.grad(ref_o, (q, k, v), do)
    for got, w in zip((dq, dk, dv), want):
        assert_allclose(got, w, 1e-5, 1e-5)


def test_default_config_is_multi_head():
    """Without num_key_value_heads (or with it equal to the head count) the block is the multi-head one: the same
    parameters and shapes, and the traced step calls attention_qkvpacked and no grouped op."""
    base = GPTConfig(vocab_size=128, hidden_size=64, num_hidden_layers=1, num_attention_heads=4,
                     max_position_embeddings=8, dtype=torch.float32)
    same = GPTConfig(vocab_size=128, hidden_size=64, num_hidden_layers=1, num_attention_heads=4,
                     num_key_value_heads=4, max_position_embeddings=8, dtype=torch.float32)
    shapes = {k: tuple(v.shape) for k, v in params_of(GPTModel(base)).items()}
    assert shapes == {k: tuple(v.shape) for k, v in params_of(GPTModel(same)).items()}
    assert shapes["blocks.0.qkv_w"] == (192, 64) and num_params(base) == sum(
        v.numel() for v in params_of(GPTModel(base)).values())
    gqa = GPTConfig(vocab_size=128, hidden_size=64, num_hidden_layers=1, num_attention_heads=4,
                    num_key_value_heads=2, max_position_embeddings=8, dtype=torch.float32)
    gp = params_of(GPTModel(gqa))
    assert tuple(gp["blocks.0.qkv_w"].shape) == ((4 + 2 * 2) * 16, 64)
    assert num_params(gqa) == sum(v.numel() for v in gp.values())
    with pytest.raises(AssertionError):
        GPTConfig(hidden_size=64, num_attention_heads=4, num_key_value_heads=3)
    alpa.init(cluster="local", num_devices=1)
    try:
        for cfg, want, unwanted in ((base, "attention_qkvpacked", "attention_gqa"),
                                    (gqa, "attention_gqa_packed", "attention_qkvpacked")):
            text = _train(cfg, ShardParallel(), B=2)[2].get_hlo_text()
            assert want in text and unwanted not in text
    finally:
        alpa.shutdown()


def _train(cfg, method, B=4):
    """One SGD step of the serial and the parallel train step, checked against each other with the tolerances of
    tests/test_shard_parallel_gpt.py; returns both states and the parallel executable."""
    torch.manual_seed(0)
    model = GPTModel(cfg)
    state = TrainState.create(apply_fn=None, params=params_of(model), tx=sgd(1e-2))
    S = cfg.max_position_embeddings
    batch = {"input_ids": torch.randint(1, cfg.vocab_size, (B, S)), "position_ids": torch.arange(S).repeat(B, 1),
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
    return expected, actual, p_step.get_last_executable()


def _gqa_cfg(kv, **kw):
    return GPTConfig(vocab_size=512, hidden_size=256, num_hidden_layers=2, num_attention_heads=8, num_key_value_heads=kv,
                     max_position_embeddings=16, dtype=torch.float32, **kw)


def _assert_groups_whole(ex, kv):
    """Every grouped attention node sees whole groups: its packed qkv operand has the slot dim unsharded and the K/V-head
    dim split into a number of parts that divides the K/V head count."""
    seen = 0
    for node, plans in ex.program.plan.node_plans.items():
        if "attention_gqa" not in str(node.target):
            continue
        for plan in (plans if isinstance(plans, (list, tuple)) else [plans]):
            spec = plan.in_specs[1 if "bwd" in str(node.target) else 0]
            assert spec.num_shards(3) == 1 and kv % spec.num_shards(2) == 0, (node.name, str(spec))
            seen += 1
    assert seen >= 4


@pytest.mark.parametrize("kv", [1, 2, 4])
@pytest.mark.parametrize("shape", [(1, 4), (2, 2)])
def test_shard_parallel(local_mesh4, kv, shape):
    _, actual, ex = _train(_gqa_cfg(kv), ShardParallel(devices=local_mesh4.get_logical_mesh(shape)))
    _assert_groups_whole(ex, kv)
    if kv == 4 and shape == (1, 4):
        for i in range(2):
            assert str(actual.params[f"blocks.{i}.qkv_w"].sharding_spec) == "S1R"   # column parallel = K/V heads


@pytest.mark.parametrize("kv", [1, 2, 4])
def test_zero3(local_mesh4, kv):
    _train(_gqa_cfg(kv), Zero3Parallel(devices=local_mesh4.get_logical_mesh((4, 1))))


@pytest.mark.parametrize("kv", [1, 2, 4])
def test_pipeshard_two_stages(local_mesh4, kv):
    cfg = _gqa_cfg(kv, add_manual_pipeline_markers=True, pipeline_mp_size=2)
    method = PipeshardParallel(num_micro_batches=2, layer_option=ManualLayerOption(),
                               stage_option=UniformStageOption(num_stages=2))
    ex = _train(cfg, method, B=8)[2]
    assert ex.config.num_meshes == 2

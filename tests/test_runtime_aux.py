"""Runtime odds and ends: live-buffer accounting (no leaks after donation / del), metric stacking, dummy-value and
signal send/recv benchmarking knobs, communication counting, OrderedSet, cost-model estimates
(reference: tests/runtime/test_memory_leak.py, tests/util/test_ordered_set.py, test_hlo_cost_model.py)."""
import gc

import torch

import alpa_b200 as alpa
from alpa_b200 import PipeshardParallel, ShardParallel
from alpa_b200.device_mesh import get_live_buffer_bytes, get_live_buffer_uuids
from alpa_b200.testing import assert_allclose, get_mlp_train_state_and_step
from alpa_b200.util import OrderedSet, count_communication_primitives, get_metrics


def test_no_live_buffers_after_delete_shard_parallel(local_mesh4):
    gc.collect()
    base = set(get_live_buffer_uuids())
    state, batch, train_step = get_mlp_train_state_and_step(batch_size=16, hidden_dim=64, num_layers=2)
    p_step = alpa.parallelize(train_step, method=ShardParallel(devices=local_mesh4), donate_argnums=(0,))
    state, loss = p_step(state, batch)
    n1 = len(set(get_live_buffer_uuids()) - base)
    assert n1 > 0 and get_live_buffer_bytes() > 0
    for _ in range(3):                      # donated inputs are consumed: the live set does not grow with steps
        state, loss = p_step(state, batch)
    gc.collect()
    assert len(set(get_live_buffer_uuids()) - base) == n1
    assert set(local_mesh4.get_live_buffer_uuids()) >= set(get_live_buffer_uuids(local_mesh4))
    del state, loss
    gc.collect()
    assert set(get_live_buffer_uuids()) - base == set()


def test_no_live_buffers_after_delete_pipeshard():
    alpa.init(cluster="local", num_devices=4)
    try:
        gc.collect()
        base = set(get_live_buffer_uuids())
        state, batch, train_step = get_mlp_train_state_and_step(batch_size=16, hidden_dim=64, num_layers=4,
                                                                add_manual_pipeline_marker=True)
        p_step = alpa.parallelize(train_step, method=PipeshardParallel(num_micro_batches=2,
                                                                       layer_option=alpa.ManualLayerOption()),
                                  donate_argnums=(0,))
        state, loss = p_step(state, batch)
        state, loss = p_step(state, batch)
        gc.collect()
        n = len(set(get_live_buffer_uuids()) - base)
        state, loss = p_step(state, batch)
        gc.collect()
        assert len(set(get_live_buffer_uuids()) - base) == n
        del state, loss
        gc.collect()
        assert set(get_live_buffer_uuids()) - base == set()
    finally:
        alpa.shutdown()


def test_get_metrics_stacks_steps(local_mesh4):
    state, batch, train_step = get_mlp_train_state_and_step(batch_size=16, hidden_dim=32, num_layers=2)

    def step(state, batch):
        new_state, loss = train_step(state, batch)
        return new_state, {"loss": loss, "twice": loss * 2}
    p_step = alpa.parallelize(step, method=ShardParallel(devices=local_mesh4), donate_argnums=())
    ms = []
    for _ in range(3):
        state, m = p_step(state, batch)
        ms.append(m)
    out = get_metrics(ms)
    assert out["loss"].shape == (3,) and torch.allclose(out["twice"], 2 * out["loss"])
    assert out["loss"][2] < out["loss"][0]


def test_dummy_values_and_signal_send_recv_knobs():
    """Benchmark knobs: inputs replaced by 1e-8 constants / cross-mesh payloads replaced by 1-byte signals.  Results
    are meaningless by design; the step must still run with the right shapes."""
    alpa.init(cluster="local", num_devices=4)
    try:
        state, batch, train_step = get_mlp_train_state_and_step(batch_size=16, hidden_dim=64, num_layers=4,
                                                                add_manual_pipeline_marker=True)
        alpa.global_config.use_dummy_value_for_benchmarking = True
        p = alpa.parallelize(train_step, method=ShardParallel(), donate_argnums=())
        s, loss = p(state, batch)
        assert abs(float(loss._value)) < 1e-6                      # every input was 1e-8
        alpa.global_config.use_dummy_value_for_benchmarking = False
        alpa.global_config.pipeline_use_signal_send_recv = True
        p2 = alpa.parallelize(train_step, method=PipeshardParallel(num_micro_batches=2,
                                                                   layer_option=alpa.ManualLayerOption()),
                              donate_argnums=())
        s2, loss2 = p2(state, batch)
        assert tuple(s2.params["layers.0.weight"].shape) == tuple(state.params["layers.0.weight"].shape)
    finally:
        alpa.global_config.use_dummy_value_for_benchmarking = False
        alpa.global_config.pipeline_use_signal_send_recv = False
        alpa.shutdown()


def test_count_communication_primitives_on_program_text(local_mesh4):
    state, batch, train_step = get_mlp_train_state_and_step(batch_size=16, hidden_dim=64, num_layers=2)
    p = alpa.parallelize(train_step, method=alpa.DataParallel(devices=local_mesh4), donate_argnums=())
    p(state, batch)
    ex = p.get_last_executable()
    text = ex.get_hlo_text() if hasattr(ex, "get_hlo_text") else ex.program.to_string()
    total, ar, ag, rs, a2a = count_communication_primitives(text)
    assert ar >= 1 and ag == 0 and rs == 0 and a2a == 0 and total == ar
    p3 = alpa.parallelize(train_step, method=alpa.Zero3Parallel(devices=local_mesh4), donate_argnums=())
    p3(state, batch)
    ex3 = p3.get_last_executable()
    text3 = ex3.get_hlo_text() if hasattr(ex3, "get_hlo_text") else ex3.program.to_string()
    total3, ar3, ag3, rs3, _ = count_communication_primitives(text3, ignore_scalar_all_reduce=True)
    assert ag3 >= 1 and rs3 >= 1


def test_ordered_set():
    s = OrderedSet([3, 1, 2, 1])
    assert list(s) == [3, 1, 2] and len(s) == 3 and 1 in s
    s.add(5)
    s.discard(1)
    assert list(s) == [3, 2, 5]
    t = OrderedSet([2, 9])
    assert list(s | t) == [3, 2, 5, 9] and list(s & t) == [2] and list(s - t) == [3, 5]
    s.update([7, 3])
    assert list(s) == [3, 2, 5, 7]


def test_profiling_database_estimate(tmp_path):
    from alpa_b200.mesh_profiling import MeshProfilingResult, ProfilingResultDatabase, estimate_stage_cost_from_db
    prof = MeshProfilingResult()
    sizes = (1 << 10, 1 << 20, 1 << 24)
    for table in (prof.all_reduce_cost_dict, prof.all_gather_cost_dict, prof.reduce_scatter_cost_dict,
                  prof.all_to_all_cost_dict):
        table[(4, "bf16")] = [(float(n), 1e-6 + n / 400e9) for n in sizes]
    prof.dot_cost_dict[("bf16",)] = [(2.0 * n ** 3, 2.0 * n ** 3 / 1.2e15) for n in (1024, 4096)]
    db = ProfilingResultDatabase()
    db.update_one_mesh("h100", (1, 4), prof)
    path = str(tmp_path / "prof.pkl")
    db.save(path)
    db2 = ProfilingResultDatabase()
    db2.load(path)
    c_small = estimate_stage_cost_from_db(db2, "h100", (1, 4), 1e12, [("all_reduce", 4, float(1 << 20))])
    c_big = estimate_stage_cost_from_db(db2, "h100", (1, 4), 4e12, [("all_reduce", 4, float(1 << 24))])
    assert 0 < c_small < c_big
    # interpolation inside the table, linear extrapolation above it; unknown mesh -> analytic model
    r = db2.query("h100", (1, 4))
    mid = r.estimate_all_reduce(4, "bf16", 3 * (1 << 19))
    assert r.estimate_all_reduce(4, "bf16", 1 << 20) < mid * 1.0001 or mid > 0
    assert abs(r.estimate_all_reduce(4, "bf16", 1 << 25) - 2 * r.estimate_all_reduce(4, "bf16", 1 << 24)) < 1e-9
    assert estimate_stage_cost_from_db(db2, "unknown", (1, 2), 1e12, [("all_gather", 2, 1e6)]) > 0


def test_timer_survives_exceptions():
    from alpa_b200.timer import timers
    t = timers("unit-test-timer")
    t.reset()
    try:
        with t:
            raise ValueError("x")
    except ValueError:
        pass
    assert not t.started and t.costs == []
    t.start()                      # a region that never stops ...
    t.start()                      # ... does not poison the next start
    t.stop()
    assert len(t.costs) == 1 and len(t.start_times) == 1
    with t:
        pass
    assert len(t.costs) == 2


def test_stream_pool_and_event_registry_are_device_agnostic():
    """On a CPU-only host the stream / event helpers are no-ops with the same bookkeeping (reference:
    collective.py:781-798 comm_wait_compute / compute_wait_comm / record_events / wait_events)."""
    from alpa_b200 import collective as col
    col.reset_events()
    reg = col.get_event_registry()
    col.record_events(["buf-1", ("mesh0", 7, 2)])
    assert len(reg) == 2 and reg.query("buf-1")
    assert col.wait_events(["buf-1", "never-produced"], group_name="pp") == ["never-produced"]
    col.comm_wait_compute("pp")
    col.compute_wait_comm("pp")
    pool = col.get_stream_pool()
    s = pool.get_stream()
    assert (s is None) == (not torch.cuda.is_available())
    reg.discard(["buf-1"])
    assert not reg.query("buf-1") and len(reg) == 1
    col.reset_events()
    assert len(reg) == 0


def test_small_reference_api_helpers():
    """Helpers that exist for parity with the reference's public modules (util, testing, mesh_profiling, schedules,
    data_loader, stage_construction, collective)."""
    import numpy as np
    import torch
    from alpa_b200 import mesh_profiling as mp, util
    from alpa_b200.collective import collective as col
    from alpa_b200.data_loader import get_num_devices_for_whole_batch, next_mesh_data_loader_uuid
    from alpa_b200.parallel.pipeline import schedules as sch
    from alpa_b200.parallel.pipeline.stage_construction import get_last_dp_result
    from alpa_b200.sharding import ShardingSpec
    from alpa_b200.util import OrderedSet
    s = OrderedSet([1, 2, 3, 4])
    s.intersection_update([2, 3, 9])
    assert list(s) == [2, 3]
    s.difference_update([3])
    assert list(s) == [2] and list(OrderedSet([1, 2]).symmetric_difference([2, 5])) == [1, 5]
    assert util.check_arithmetic_sequence([2, 5, 8]) == 3 and util.check_arithmetic_sequence([1, 2, 4]) is None
    assert util.to_int_tuple(np.array([1.0, 2.0])) == (1, 2)
    tree = {"a": torch.zeros(2, 3), "b": [torch.zeros(4, dtype=torch.bfloat16)]}
    assert util.compute_param_number(tree) == 10 and util.compute_bytes(tree) == 2 * 3 * 4 + 4 * 2
    assert util.map_to_shape(tree) == {"a": (2, 3), "b": [(4,)]}
    assert util.map_to_nparray(tree)["b"][0].dtype == np.float32
    assert hash(util.freeze_dict({"x": [1, {"y": 2}]})) is not None
    assert util.env_integer("ALPA_B200_NOT_SET_ANYWHERE", 7) == 7
    res = mp.MeshProfilingResult()
    res.all_reduce_cost_dict[(2, "bf16")] = [(4096.0, 3e-5), (1024.0, 1e-5), (16384.0, 2e-5)]
    res.make_monotonic()
    assert [t for _, t in res.all_reduce_cost_dict[(2, "bf16")]] == [1e-5, 3e-5, 3e-5]
    db = mp.ProfilingResultDatabase()
    db.insert_dummy_mesh_result("c", (1, 4))
    assert db.query("c", (1, 4)).estimate_all_reduce(4, "bf16", 1 << 20) > 0
    assert mp.enumerate_all_collective_spec is mp.enumerate_collective_specs
    dep = sch.gen_linear_pipeline_dependency(4)
    g = sch.GpipeSchedule(dependency=dep, meshes=[0, 1], apply_grad_placement={}, num_batch=4)
    assert g.previous_backward_batch_index(3) == 2 and g.num_mesh == 2
    a, b = next_mesh_data_loader_uuid(), next_mesh_data_loader_uuid()
    assert b == a + 1
    assert get_num_devices_for_whole_batch(ShardingSpec.from_string((2, 4), "S0R")) == 4
    assert get_num_devices_for_whole_batch(ShardingSpec.from_string((2, 4), "RR")) == 8
    assert len(get_last_dp_result()) == 5
    assert col.gloo_available() in (True, False) and callable(col.allreduce_multigpu) and callable(col.comm_wait_compute)

"""The benchmark runner (benchmark/benchmark_one_case.py; reference: benchmark/alpa/benchmark_one_case*.py) on emulated
meshes with a tiny GPT: every parallel mode of the suites -- intra-op methods, the uniform (dp x op x pp) 3-D method
with `CreateStateParallel`, and the auto stage search -- builds, runs and reports the reference's metrics."""
import os
import sys

import pytest

import alpa_b200 as alpa

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "benchmark"))


@pytest.mark.parametrize("mode,args,nmb,ngpu", [
    ("shard", ("auto",), 1, 4),
    ("shard", ("zero2",), 1, 2),
    ("uniform", (True, False, 1, 2, 2, True), 2, 4),          # dp1 x op2 x pp2, like BASELINE config 3 in small
    ("uniform", (True, True, 2, 1, 2, True), 4, 4),           # dp2 x pp2 with rematerialisation
    ("search", (True, False, 2, {"submesh_physical_shape_space": "small_power_of_two",
                                 "submesh_logical_shape_space": "all", "stage_imbalance_tolerance": 1.0,
                                 "use_hlo_cost_model": True}), 2, 4),
])
def test_benchmark_one_case_modes(mode, args, nmb, ngpu):
    from benchmark_one_case import benchmark_one_case
    from suites import BenchmarkCase, SearchParallelArgs, ShardParallelArgs, UniformParallelArgs
    cls = {"shard": ShardParallelArgs, "uniform": UniformParallelArgs, "search": SearchParallelArgs}[mode]
    case = BenchmarkCase(8, "test-tiny", nmb, mode, cls(*args))
    alpa.shutdown()
    alpa.init(cluster="local", num_devices=ngpu)
    try:
        for create_state in ((False, True) if mode == "uniform" else (False,)):
            res = benchmark_one_case("gpt", case, ngpu, niter=1, warmup=1, create_state_parallel=create_state)
            assert res["latency_s"] > 0 and res["tflops_per_gpu"] > 0
            assert isinstance(res["collectives"], dict)
            alpa.clear_executable_cache()
    finally:
        alpa.shutdown()


def test_resharding_benchmark_plans_show_load_balance_and_allgather_effects(tmp_path):
    """benchmark/resharding (plan-only): load balancing halves the busiest sender for a replicated source, the local
    all-gather halves the cross-mesh bytes for a replicated destination (reference: benchmark/alpa/resharding)."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "resharding_plan.jsonl")
    r = subprocess.run([sys.executable, "benchmark/resharding/benchmark_cross_mesh_resharding.py", "--suite", "n-to-m",
                        "--plan-only", "--json", out], cwd=root, capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stderr[-2000:]
    import json
    rows = {(d["case"], d["mode"]): d for d in map(json.loads, open(out))}
    assert rows[("4-to-4 replicated src", "send_recv")]["busiest_sender_MB"] * 2 == \
        rows[("4-to-4 replicated src", "send_recv_no_balance")]["busiest_sender_MB"]
    assert rows[("4-to-4 to replicated", "send_recv_allgather")]["cross_mesh_MB"] * 2 == \
        rows[("4-to-4 to replicated", "send_recv")]["cross_mesh_MB"]
    os.remove(out)


def test_benchmark_inference_suite_case():
    """The inference suites (forward only through the inference pipeline schedule; reference:
    benchmark_one_case_gpt_bert_inference.py) on an emulated mesh, pipelined and intra-op only."""
    from benchmark_one_case import benchmark_one_case
    from suites import BenchmarkCase, ShardParallelArgs, UniformParallelArgs, suites
    assert {"gpt_inference", "moe_inference", "unet"} <= set(suites)
    alpa.shutdown()
    alpa.init(cluster="local", num_devices=4)
    try:
        for case in (BenchmarkCase(8, "test-tiny", 2, "uniform", UniformParallelArgs(False, False, 1, 2, 2, True)),
                     BenchmarkCase(8, "test-tiny", 1, "shard", ShardParallelArgs("auto"))):
            res = benchmark_one_case("gpt_inference", case, 4, niter=1, warmup=1)
            assert res["latency_s"] > 0 and res["tflops_per_gpu"] > 0
            alpa.clear_executable_cache()
    finally:
        alpa.shutdown()


def test_benchmark_helper_scripts(tmp_path):
    """gather_gpu_stat / inspect_prof_database / run_exp / gen_serving_database (reference: benchmark/alpa/*.py)."""
    import json
    import gather_gpu_stat
    import gen_serving_database as gsd
    import inspect_prof_database as ipd
    import run_exp
    from alpa_b200.mesh_profiling import ProfilingResultDatabase

    stats = gather_gpu_stat.gather_gpu_stat()
    assert len(stats) == 1 and isinstance(next(iter(stats.values())), list)

    db = ProfilingResultDatabase()
    db.insert_dummy_mesh_result("default", (1, 8))
    text = ipd.describe(db, "default", (1, 8))
    assert "Meshes:" in text and "(1, 8)" in text
    assert "no entry" in ipd.describe(db, "default", (4, 8))

    res = run_exp.run_exp(str(tmp_path / "exp"), [run_exp.parse_cluster("1x4"), (1, 1)], "gpt_inference",
                          dry_run=True)
    assert [r[0] for r in res] == [(1, 4), (1, 1)]
    cmd = run_exp.command_for("gpt", [], 1, 4, False, "e", 29600)
    assert "torch.distributed.run" in cmd and "--nproc-per-node=4" in cmd
    assert "--emulate" in run_exp.command_for("gpt", [], 1, 4, True, "e", 29600)

    jl = tmp_path / "inf.jsonl"
    rows = [{"suite": "gpt_inference", "model": "1.3B", "n_gpus": 2, "batch": 1, "parallel": "uniform:(1, 2)",
             "latency_s_device_timed_max_over_ranks": 0.02, "tflops_per_gpu": 100.0, "peak_mem_gb": 3.0},
            {"suite": "gpt_inference", "model": "1.3B", "n_gpus": 2, "batch": 1, "parallel": "uniform:(2, 1)",
             "latency_s_device_timed_max_over_ranks": 0.015},
            {"suite": "gpt", "model": "1.3B", "n_gpus": 2, "batch": 8, "parallel": "x",
             "latency_s_device_timed_max_over_ranks": 1.0}]
    jl.write_text("\n".join(json.dumps(r) for r in rows) + "\n")
    sdb = gsd.ServingProfilingDatabase(str(tmp_path / "db.pkl"), new=True)
    sdb.update_from_jsonl(str(jl))
    sdb.materialize()
    again = gsd.ServingProfilingDatabase(str(tmp_path / "db.pkl"))
    best = again.query("1.3B", 2)
    assert list(best) == [1] and best[1]["parallel"] == "uniform:(2, 1)" and "1.3B" in str(again)
    tsv = tmp_path / "r.tsv"
    tsv.write_text("gpt_inference\t2.6B\t4\t2\t1\tuniform:(1, 4)\t0.03\t50.0\t4.0\t1.0\t{}\n")
    again.update_from_csv(str(tsv))
    assert again.query("2.6B")[2]["latency_s"] == 0.03

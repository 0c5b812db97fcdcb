"""Self-check of the default attention forward configuration in a throw-away process.

    python -m alpa_b200.ops.selfcheck attention_fwd            # prints "selfcheck attention_fwd: ok | FAIL ..."

`select_attention_forward()` runs it (on this rank's GPU) before a long job touches CUDA and, if the check fails, times
out or the process dies (a device-side trap poisons the CUDA context, which is why it must not run in the caller's
process), pins the attention forward to its 64-query-tile configuration ("gen2") via ALPA_B200_ATTN_FWD.  bench.py and
__graft_entry__.smoke() call it; the result is reported in bench.py's JSON (`config.attention_fwd_kernel`)."""
import os
import subprocess
import sys


def _check_attention_fwd() -> str:
    import torch
    from alpa_b200 import ops
    if not torch.cuda.is_available() or not ops.native_available():
        return "skipped (no GPU / extension)"
    C = ops.native_module()
    torch.manual_seed(0)
    worst = 0.0
    # (B, query heads, S, D, causal, group): group > 1 is a grouped-query call on a packed [B, S, H / G, G + 2, D] tensor
    for (B, H, S, D, causal, G) in [(2, 4, 256, 64, False, 1), (1, 3, 384, 64, True, 1), (4, 40, 1024, 64, False, 1),
                                    (2, 8, 320, 64, True, 4)]:
        if G == 1:
            qkv = torch.randn(B, S, 3, H, D, device="cuda", dtype=torch.bfloat16)
            q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
            o, lse = C.attention_fwd(q, k, v, D ** -0.5, causal)                   # default dispatch
        else:
            qkv = torch.randn(B, S, H // G, G + 2, D, device="cuda", dtype=torch.bfloat16)
            q, k, v = qkv[:, :, :, :G], qkv[:, :, :, G], qkv[:, :, :, G + 1]
            o, lse = C.attention_fwd(q, k, v, D ** -0.5, causal)
            o, lse = o.reshape(B, S, H, D), lse.reshape(B, H, S)
            q, k, v = q.reshape(B, S, H, D), k.repeat_interleave(G, 2), v.repeat_interleave(G, 2)
        qf, kf, vf = (t.float().permute(0, 2, 1, 3) for t in (q, k, v))
        s = torch.matmul(qf, kf.transpose(-1, -2)) * D ** -0.5
        if causal:
            s = s.masked_fill(~torch.ones(S, S, device="cuda", dtype=torch.bool).tril(), float("-inf"))
        ref = torch.matmul(torch.softmax(s, -1), vf).permute(0, 2, 1, 3)
        ref_lse = torch.logsumexp(s, -1)
        torch.cuda.synchronize()
        err = (o.float() - ref).abs().max().item()
        err_l = (lse - ref_lse).abs().max().item()
        if not (err < 0.03 and err_l < 0.02):
            return f"FAIL B{B} H{H} G{G} S{S} D{D} causal={causal}: max|o - ref| = {err:.4f}, max|lse - ref| = {err_l:.4f}"
        worst = max(worst, err)
    return f"ok (max abs err {worst:.4f})"


def select_attention_forward(timeout: float = 180.0) -> str:
    """Returns the forward configuration that will be used: "gen4" (128-query tiles, the default) or "gen2"."""
    if os.environ.get("ALPA_B200_ATTN_FWD"):
        return os.environ["ALPA_B200_ATTN_FWD"]            # the user chose
    env = dict(os.environ)
    lr = os.environ.get("LOCAL_RANK")
    if lr is not None and "CUDA_VISIBLE_DEVICES" not in env:
        env["CUDA_VISIBLE_DEVICES"] = lr                     # the check runs on this rank's GPU
    for k in ("RANK", "WORLD_SIZE", "LOCAL_RANK", "MASTER_ADDR", "MASTER_PORT"):
        env.pop(k, None)
    root = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    env["PYTHONPATH"] = root + os.pathsep + env.get("PYTHONPATH", "")
    try:
        r = subprocess.run([sys.executable, "-m", "alpa_b200.ops.selfcheck", "attention_fwd"], env=env, cwd=root,
                           capture_output=True, text=True, timeout=timeout)
        line = [l for l in r.stdout.splitlines() if l.startswith("selfcheck attention_fwd:")]
        ok = r.returncode == 0 and line and (" ok" in line[-1] or "skipped" in line[-1])
        detail = line[-1] if line else (r.stderr.strip().splitlines() or ["no output"])[-1]
    except subprocess.TimeoutExpired:
        ok, detail = False, f"timed out after {timeout:.0f} s"
    except Exception as e:  # noqa: BLE001  -- the check itself could not run: stay on the validated kernel
        ok, detail = False, f"{type(e).__name__}: {e}"
    if ok:
        return "gen4"
    import logging
    logging.getLogger(__name__).warning("attention forward self-check failed (%s): using 64-query tiles", detail)
    os.environ["ALPA_B200_ATTN_FWD"] = "gen2"
    return "gen2"


if __name__ == "__main__":
    what = sys.argv[1] if len(sys.argv) > 1 else "attention_fwd"
    res = _check_attention_fwd() if what == "attention_fwd" else f"FAIL unknown check {what}"
    print(f"selfcheck {what}: {res}", flush=True)
    sys.exit(1 if res.startswith("FAIL") else 0)

"""MoE routing, dispatch, combine and combine_wgrad, the embedding gather and the fused AdamW against references written
from each operation's definition.

* `moe_top2_route`: bit for bit against GShard top-2 routing: the first choice is the first index of the largest gate,
  the second the first index of the largest gate once the first choice's gate is replaced by 0 (so rows whose other
  gates are all exactly 0 pick the first choice's expert again when it is expert 0), first choices fill an expert's
  capacity in token order and second choices continue after the kept first choices.
* `moe_dispatch`: every routed row is bf16(fp32(x) * fp32(w)), one rounding of an exact product; unused rows are 0.
* `moe_combine`: bf16(fp32(w1 e1) + fp32(w2 e2)) over the kept choices, again one correct answer.
* `moe_combine_wgrad`: `bf16_rule` against float64, with sum |dout * eo| as the cancellation terms.
* Expert parallelism emulated on one GPU: the experts split over n local buffers whose addresses go in as `peer_ptrs`,
  one call per rank with g_off = rank * G_local; the assembled result must equal the single-buffer one.
* `embedding_fwd`: bit for bit, inside NaN rows so that an off-by-one row read shows.
* AdamW: each step is referenced in float64 from the kernel's own fp32 state before that step, with the fp32 lr, betas
  and eps the kernel receives.  m and v under `fp32_rule` (terms beta |m| + (1 - beta) |g s| and the squared form);
  the master weight within ulp32(p') + TOL32 * lr * (|m_hat| / (sqrt(v_hat) + eps) + wd |p|), a bound that scales with
  the update and not with |p|; the bf16 copy equal to the round-to-nearest-even of the kernel's own fp32 master.  Every
  tensor is a [:n] view of a NaN-filled buffer whose tail must stay bitwise unchanged.

The CPU tests show the rules reject known-wrong results built with the same reference functions.
"""
import math
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernel_numerics import BF16, F64, TOL32, WORST, Checker, _bf, _report, bf16_rule, fp32_rule  # noqa: E402

NAN = float("nan")
F32 = torch.float32


@pytest.fixture(scope="module", autouse=True)
def _print_worst_ratios():
    before = set(WORST)
    yield
    mine = sorted(k for k in WORST if k not in before)
    if mine:
        print("\n[moe / embedding / adamw numerics] worst ratio of kernel error to baseline error (fp32: to the bound):")
        for k in mine:
            print(f"  {k:40s} {WORST[k]:.3f}")


def _f32(x):
    """The fp32 value the kernel receives for the Python float x, as a Python float."""
    return torch.tensor(x, dtype=F32).item()


# ---------------------------------------------------------------------------------------------------------------------
# references
# ---------------------------------------------------------------------------------------------------------------------


def _first_argmax(x):
    """First index of the maximum along the last dim."""
    E = x.shape[-1]
    idx = torch.arange(E, device=x.device).expand_as(x)
    return torch.where(x == x.amax(-1, keepdim=True), idx, E).amin(-1)


def _positions(e, E):
    """Number of earlier tokens (along dim 1) routed to the same expert, and the per-expert totals [G, E]."""
    oh = torch.nn.functional.one_hot(e, E)
    return (oh.cumsum(1) - oh).gather(-1, e[..., None])[..., 0], oh.sum(1)


def route_ref(gates, C):
    """GShard top-2 routing of gates [G, S, E] -> (expert, slot) int64 [G, S, 2]; slot -1 = dropped."""
    E = gates.shape[-1]
    i1 = _first_argmax(gates)
    masked = gates.scatter(-1, i1[..., None], 0.0)
    i2 = _first_argmax(masked)
    p1, count1 = _positions(i1, E)
    p2, _ = _positions(i2, E)
    p2 = p2 + count1.clamp_max(C).gather(-1, i2)
    s1 = torch.where(p1 < C, p1, -1)
    s2 = torch.where(p2 < C, p2, -1)
    return torch.stack([i1, i2], -1), torch.stack([s1, s2], -1)


def old_kernel_second_choice(row):
    """The second choice of the routing kernel before the fix: a strict `v > b2` scan, and the neighbour of the first
    choice when no gate beat -inf."""
    b1 = b2 = -math.inf
    i1 = i2 = 0
    for e, v in enumerate(row):
        if v > b1:
            b2, i2, b1, i1 = b1, i1, v, e
        elif v > b2:
            b2, i2 = v, e
    if b2 == -math.inf or i2 == i1:
        i2 = 1 if i1 == 0 else 0
    return i1, i2


def dispatch_ref(x, expert, slot, weight, E, C):
    """d [E, G*C, M] bf16: row g*C + c of expert e = bf16(fp32(x) * fp32(w)) (x when weight is None); other rows 0."""
    G, S, M = x.shape
    K = expert.shape[-1]
    d = torch.zeros(E, G * C, M, dtype=BF16, device=x.device)
    for k in range(K):
        for g in range(G):
            keep = slot[g, :, k] >= 0
            src = x[g][keep]
            if weight is not None:
                src = (src.float() * weight[g, :, k][keep].float()[:, None]).to(BF16)
            d[expert[g, :, k][keep], g * C + slot[g, :, k][keep]] = src
    return d


def _gather_rows(eo, expert, slot):
    """eo rows [G, S, K, M] of every choice (row 0 for dropped ones) and the kept mask [G, S, K]."""
    E, GC, M = eo.shape
    G = expert.shape[0]
    C = GC // G
    g = torch.arange(G, device=eo.device).view(G, 1, 1)
    ok = slot >= 0
    rows = torch.where(ok, expert * GC + g * C + slot, 0)
    return eo.reshape(E * GC, M)[rows], ok


def combine_ref(eo, expert, slot, weight):
    """bf16(sum over kept choices of fp32(w_k * e_k)), summed in choice order in fp32 (the products are exact)."""
    rows, ok = _gather_rows(eo, expert, slot)
    w = torch.ones(expert.shape, dtype=F32, device=eo.device) if weight is None else weight.float()
    acc = torch.zeros(rows.shape[:2] + rows.shape[3:], dtype=F32, device=eo.device)
    for k in range(expert.shape[-1]):
        acc = torch.where(ok[:, :, k, None], acc + w[:, :, k, None] * rows[:, :, k].float(), acc)
    return acc.to(BF16)


def combine_wgrad_ref(dout, eo, expert, slot, drop_chunk=None):
    """(dw [G, S, K] float64, sum |dout * eo| terms).  drop_chunk=i leaves out channels [256 i, 256 i + 256)."""
    rows, ok = _gather_rows(eo, expert, slot)
    prod = rows.to(F64) * dout.to(F64)[:, :, None, :]
    if drop_chunk is not None:
        prod[..., 256 * drop_chunk:256 * drop_chunk + 256] = 0
    return prod.sum(-1) * ok, prod.abs().sum(-1) * ok


def embedding_ref(ids, wte, vocab_start, pos=None, wpe=None):
    """wte[id - vocab_start] (zeros outside the shard), plus bf16(fp32(wte) + fp32(wpe[pos])) when pos is given."""
    V, H = wte.shape
    local = ids - vocab_start
    ok = (local >= 0) & (local < V)
    out = torch.where(ok[..., None], wte[local.clamp(0, V - 1)], torch.zeros((), dtype=BF16, device=wte.device))
    if pos is not None:
        out = (out.float() + wpe[pos].float()).to(BF16)
    return out


def adam_ref(p, m, v, g, gs, lr, b1, b2, eps, wd, step, variant=None):
    """One AdamW step in float64 from fp32 state (p, m, v) and gradient g times the fp32 scale gs.  Returns
    (m', v', p', m terms, v terms, |m_hat| / (sqrt(v_hat) + eps) + wd |p|).  `variant` builds a known-wrong step."""
    p, m, v, g = (t.to(F64) for t in (p, m, v, g))
    gg = g * gs
    m1 = b1 * m + (1 - b1) * gg
    v1 = b2 * v + (1 - b2) * gg * gg
    t = step - 1 if variant == "stale bias correction" else step
    mh = m1 / (1 - b1 ** t)
    vh = v1 / (1 - b2 ** t)
    u = mh / ((vh + eps).sqrt() if variant == "eps inside sqrt" else (vh.sqrt() + eps))
    if variant == "weight decay after the update":
        p1 = (p - lr * u) * (1 - lr * wd)
    else:
        p1 = p - lr * (u + wd * p)
    tm = b1 * m.abs() + (1 - b1) * gg.abs()
    tv = b2 * v.abs() + (1 - b2) * gg * gg
    scale = mh.abs() / (vh.sqrt() + eps) + wd * p.abs()
    return m1, v1, p1, tm, tv, scale


def _ulp32(x):
    _, e = torch.frexp(x.to(F32))
    return torch.ldexp(torch.ones_like(x, dtype=F64), (e.to(F64) - 24).clamp_min(-149))


def master_rule(name, out, ref, lr, scale):
    """|p' - p'_ref| <= ulp32(p'_ref) + TOL32 * lr * scale elementwise.  Returns (messages, worst ratio)."""
    out, ref = out.to(F64), ref.to(F64)
    if not torch.isfinite(out).all():
        return [f"{name}: {int((~torch.isfinite(out)).sum())} non-finite master weights"], math.inf
    err = (out - ref).abs()
    bound = _ulp32(ref) + TOL32 * lr * scale
    r = err / bound
    i = int(r.argmax())
    ratio = r.flatten()[i].item()
    if ratio <= 1.0:
        return [], ratio
    return [f"{name}: |err| {err.flatten()[i].item():.3e} > bound {bound.flatten()[i].item():.3e} "
            f"(ulp32(p') + TOL32 * lr * update), ratio {ratio:.2f}; {int((r > 1).sum())} of {r.numel()} out of bound"], \
        ratio


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the rules reject the wrong results of these kernels
# ---------------------------------------------------------------------------------------------------------------------


def test_routing_reference_rejects_the_old_second_choice_scan():
    gates = torch.tensor([[[1.0, 0.0, 0.0, 0.0], [0.0, 1.0, 0.0, 0.0], [0.7, 0.1, 0.1, 0.1],
                           [1.0, 0.0, 0.0, 0.0]]])
    # fp32 softmax underflows to an exact one-hot row
    assert torch.equal(torch.softmax(torch.tensor([110.0, 0.0, 0.0, 0.0]), -1), gates[0, 0])
    expert, slot = route_ref(gates, 4)
    assert expert[0, :, 1].tolist() == [0, 0, 1, 0]
    old = torch.tensor([old_kernel_second_choice(r.tolist())[1] for r in gates[0]])
    assert not torch.equal(old, expert[0, :, 1]), "the old scan agrees with the reference on one-hot rows"
    # the second choice then takes a slot of another expert: with capacity 2, the reference drops token 3's second
    # choice (expert 0 is full), while the old scan places it in expert 1
    e2, s2 = route_ref(gates, 2)
    assert s2[0, 3].tolist() == [-1, -1] and e2[0, 3, 1] == 0 and old[3] == 1


def test_rule_rejects_a_dropped_wgrad_lane_chunk():
    g = torch.Generator().manual_seed(5)
    G, S, E, M = 2, 64, 4, 1024
    C = S
    gates = torch.softmax(torch.randn(G, S, E, generator=g), -1)
    expert, slot = route_ref(gates, C)
    eo = torch.randn(E, G * C, M, generator=g).to(BF16)
    dout = torch.randn(G, S, M, generator=g).to(BF16)
    ref, terms = combine_wgrad_ref(dout, eo, expert, slot)
    assert not bf16_rule("baseline", _bf(ref), ref, _bf(ref), terms)[0]
    for chunk in range(M // 256):
        wrong, _ = combine_wgrad_ref(dout, eo, expert, slot, drop_chunk=chunk)
        assert bf16_rule(f"chunk {chunk} dropped", _bf(wrong), ref, _bf(ref), terms)[0], chunk


@pytest.mark.parametrize("variant,lr,wd,step,near_eps", [
    ("stale bias correction", 1e-3, 0.0, 2, False),
    ("stale bias correction", 1e-3, 0.0, 10, False),
    ("eps inside sqrt", 1e-3, 0.0, 1, True),
    ("eps inside sqrt", 1e-3, 0.0, 1000, True),
    ("weight decay after the update", 0.1, 0.5, 2, False),
])
def test_adamw_rules_reject_wrong_steps(variant, lr, wd, step, near_eps):
    g = torch.Generator().manual_seed(6)
    n = 4096
    s = 1e-8 if near_eps else 1.0
    p = torch.randn(n, generator=g)
    m = torch.randn(n, generator=g) * 0.1 * s
    v = torch.rand(n, generator=g) * 0.01 * s * s
    gr = torch.randn(n, generator=g) * s
    args = (p, m, v, gr, 1.0, _f32(lr), _f32(0.9), _f32(0.999), _f32(1e-8), _f32(wd), step)
    m1, v1, p1, tm, tv, sc = adam_ref(*args)
    assert not master_rule("fp32 rounding", p1.float(), p1, _f32(lr), sc)[0]
    assert not fp32_rule("m", m1.float(), m1, tm)[0] and not fp32_rule("v", v1.float(), v1, tv)[0]
    _, _, pw, _, _, _ = adam_ref(*args, variant=variant)
    msgs, ratio = master_rule(variant, pw.float(), p1, _f32(lr), sc)
    assert msgs, f"{variant}: accepted (ratio {ratio:.2f})"


# ---------------------------------------------------------------------------------------------------------------------
# GPU: MoE
# ---------------------------------------------------------------------------------------------------------------------


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _gates(G, S, E, seed):
    """Softmax gates with rows of tied gates, exact one-hot rows with expert 0 first, and one-hot rows elsewhere."""
    g = _gen(seed)
    gates = torch.softmax(torch.randn(G, S, E, generator=g, device="cuda") * 2, -1)
    flat = gates.view(-1, E)
    tie = flat[::7]
    tie.copy_(torch.softmax(torch.randint(0, 3, tie.shape, generator=g, device="cuda").float(), -1))
    flat[1::11] = 0.0
    flat[1::11, 0] = 1.0
    flat[5::13] = 0.0
    flat[5::13, E - 1] = 1.0
    return gates


ROUTE_E = [2, 8, 128, 256]
ROUTE_S = [1, 31, 1000, 1024, 1025, 4096]


@pytest.mark.gpu
@pytest.mark.parametrize("E", ROUTE_E)
def test_moe_top2_route(E):
    from alpa_b200 import ops
    fails = []
    G = 2
    for S in ROUTE_S:
        for C in sorted({1, max(1, 2 * S // E), S, S + 3}):
            gates = _gates(G, S, E, 17 * S + E)
            ex, sl = ops.moe_top2_route(gates, C)
            ex_r, sl_r = route_ref(gates, C)
            if not (torch.equal(ex, ex_r) and torch.equal(sl, sl_r)):
                bad = ((ex != ex_r) | (sl != sl_r)).any(-1)
                i = bad.nonzero()[0].tolist()
                fails.append(f"E{E} S{S} C{C}: {int(bad.sum())} tokens differ; first (g, s) = {i}: kernel "
                             f"expert {ex[i[0], i[1]].tolist()} slot {sl[i[0], i[1]].tolist()}, reference expert "
                             f"{ex_r[i[0], i[1]].tolist()} slot {sl_r[i[0], i[1]].tolist()}")
    assert not fails, "\n".join(fails)


@pytest.mark.gpu
def test_moe_top2_route_one_hot_rows():
    """Exact one-hot gates with expert 0 first: the second choice is expert 0 again, as in the dense top2_gating."""
    from alpa_b200 import ops
    gates = torch.softmax(torch.tensor([[[110.0, 0.0, 0.0, 0.0]] * 3 + [[0.0, 110.0, 0.0, 0.0]]], device="cuda"), -1)
    assert torch.equal(gates[0, 0], torch.tensor([1.0, 0.0, 0.0, 0.0], device="cuda"))
    ex, sl = ops.moe_top2_route(gates, 2)
    ex_r, sl_r = route_ref(gates, 2)
    assert torch.equal(ex, ex_r) and torch.equal(sl, sl_r), (ex.tolist(), sl.tolist(), ex_r.tolist(), sl_r.tolist())


def _moe_case(G, S, E, M, C, seed):
    g = _gen(seed)
    expert, slot = route_ref(_gates(G, S, E, seed), C)
    x = torch.randn(G, S, M, generator=g, device="cuda").to(BF16)
    w = torch.rand(G, S, 2, generator=g, device="cuda").to(BF16)
    eo = torch.randn(E, G * C, M, generator=g, device="cuda").to(BF16)
    dout = torch.randn(G, S, M, generator=g, device="cuda").to(BF16)
    return expert, slot, x, w, eo, dout


MOE_CASES = [(2, 64, 4, 8, 16), (4, 2048, 8, 264, 256), (3, 1000, 16, 1024, 100), (2, 512, 128, 2056, 2),
             (2, 300, 8, 1024, 300)]


@pytest.mark.gpu
@pytest.mark.parametrize("G,S,E,M,C", MOE_CASES)
def test_moe_dispatch_combine_wgrad(G, S, E, M, C):
    from alpa_b200 import ops
    ck = Checker()
    expert, slot, x, w, eo, dout = _moe_case(G, S, E, M, C, G * S + M)
    tag = f"G{G} S{S} E{E} M{M} C{C}"
    both_dropped = (slot < 0).all(-1)
    if C < S:
        ck.require(bool(both_dropped.any()), f"{tag}: no token has both choices dropped")
    for wt in (None, w):
        d = ops.moe_dispatch(x, expert, slot, wt, E, C)
        ck.require(torch.equal(d.view(torch.int16), dispatch_ref(x, expert, slot, wt, E, C).view(torch.int16)),
                   f"moe_dispatch {tag} weight={wt is not None}: differs from bf16(x * w) / zeros")
        o = ops.moe_combine(eo, expert, slot, wt)
        ck.require(torch.equal(o, combine_ref(eo, expert, slot, wt)),
                   f"moe_combine {tag} weight={wt is not None}: differs from bf16(w1 e1 + w2 e2)")
        ck.require(bool((o[both_dropped] == 0).all()), f"moe_combine {tag}: tokens without a kept choice are not 0")
    dw = ops.moe_combine_wgrad(dout, eo, expert, slot)
    ref, terms = combine_wgrad_ref(dout, eo, expert, slot)
    ck.bf16("moe_combine_wgrad", f"moe_combine_wgrad {tag}", dw, ref, _bf(ref), terms)
    _report(ck)


@pytest.mark.gpu
@pytest.mark.parametrize("n", [2, 4])
def test_moe_emulated_expert_parallel(n):
    """The experts split over n local buffers passed as peer pointers; every rank dispatches, combines and takes the
    weight gradient of its own groups (g_off = rank * G_local).  The assembled buffers and outputs equal the
    single-buffer results."""
    from alpa_b200 import ops
    C_ = ops.native_module()
    G_local, S, E, M, C = 2, 256, 8, 264, 40
    G = G_local * n
    E_local = E // n
    expert, slot, x, w, eo, dout = _moe_case(G, S, E, M, C, 50 + n)
    fails = []
    d_full = ops.moe_dispatch(x, expert, slot, w, E, C)
    bufs = [torch.zeros(E_local, G * C, M, device="cuda", dtype=BF16) for _ in range(n)]
    ptrs = [b.data_ptr() for b in bufs]
    gs = lambda t, r: t[r * G_local:(r + 1) * G_local].contiguous()  # noqa: E731
    for r in range(n):
        C_.moe_dispatch_(gs(x, r), gs(expert, r), gs(slot, r), gs(w, r), bufs[r], C, ptrs, r * G_local)
    if not torch.equal(torch.cat(bufs).view(torch.int16), d_full.view(torch.int16)):
        fails.append(f"n={n}: dispatch through peer pointers differs from the single buffer")
    eo_bufs = [eo[i * E_local:(i + 1) * E_local].contiguous() for i in range(n)]
    eptrs = [b.data_ptr() for b in eo_bufs]
    o_full = ops.moe_combine(eo, expert, slot, w)
    dw_full = ops.moe_combine_wgrad(dout, eo, expert, slot)
    for r in range(n):
        o = C_.moe_combine(eo_bufs[r], gs(expert, r), gs(slot, r), gs(w, r), eptrs, r * G_local)
        if not torch.equal(o.view(torch.int16), gs(o_full, r).view(torch.int16)):
            fails.append(f"n={n} rank {r}: combine through peer pointers differs")
        dw = C_.moe_combine_wgrad(gs(dout, r), eo_bufs[r], gs(expert, r), gs(slot, r), eptrs, r * G_local)
        if not torch.equal(dw.view(torch.int16), gs(dw_full, r).view(torch.int16)):
            fails.append(f"n={n} rank {r}: combine_wgrad through peer pointers differs")
    if not torch.equal(o_full, combine_ref(eo, expert, slot, w)):
        fails.append(f"n={n}: single-buffer combine differs from the reference")
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: embedding
# ---------------------------------------------------------------------------------------------------------------------


def _nan_framed(rows, H, g):
    """A [rows, H] bf16 table of random values with a NaN row before and after it in memory."""
    buf = torch.full((rows + 2, H), NAN, device="cuda", dtype=BF16)
    buf[1:rows + 1] = torch.randn(rows, H, generator=g, device="cuda").to(BF16)
    return buf[1:rows + 1]


@pytest.mark.gpu
@pytest.mark.parametrize("H", [8, 1000, 2056])
def test_embedding_fwd(H):
    from alpa_b200 import ops
    C_ = ops.native_module()
    g = _gen(H)
    fails = []
    T = torch.cuda.get_device_properties(0).multi_processor_count * 16 + 900     # above the grid: grid-stride loop
    V, vocab_start, P_ = 700, 300, 64
    wte = _nan_framed(V, H, g)
    wpe = _nan_framed(P_, H, g)
    edges = torch.tensor([vocab_start - 1, vocab_start, vocab_start + 1, vocab_start + V - 2, vocab_start + V - 1,
                          vocab_start + V, vocab_start + V + 1, 0], device="cuda")
    ids = torch.randint(0, 2 * V, (T,), generator=g, device="cuda")
    ids[:len(edges)] = edges
    ids = ids.view(3, -1) if T % 3 == 0 else ids
    pos = torch.randint(0, P_, ids.shape, generator=g, device="cuda")
    pos.view(-1)[:2] = torch.tensor([0, P_ - 1], device="cuda")
    out = C_.embedding_fwd(ids, None, wte, None, vocab_start)
    if not torch.equal(out.view(torch.int16), embedding_ref(ids, wte, vocab_start).view(torch.int16)):
        fails.append(f"H{H}: token-only embedding differs from wte[id - vocab_start] / zeros")
    out = C_.embedding_fwd(ids, pos, wte, wpe, vocab_start)
    if not torch.equal(out.view(torch.int16), embedding_ref(ids, wte, vocab_start, pos, wpe).view(torch.int16)):
        fails.append(f"H{H}: token + position embedding differs from bf16(fp32(wte) + fp32(wpe))")
    out = ops.embedding(ids, wte, vocab_start)
    if not torch.equal(out.view(torch.int16), embedding_ref(ids, wte, vocab_start).view(torch.int16)):
        fails.append(f"H{H}: ops.embedding differs")
    assert not fails, "\n".join(fails)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: AdamW
# ---------------------------------------------------------------------------------------------------------------------
ADAM_SIZES = [1, 3, 4, 5, 65535, 65536, 65537, 3 * 65536 + 3]
ADAM_PAD = 8
LR, BETA1, BETA2, EPS = 1e-3, 0.9, 0.999, 1e-8


def _framed(n, dtype, values):
    buf = torch.full((n + ADAM_PAD,), NAN, device="cuda", dtype=dtype)
    buf[:n] = values.to(dtype)
    return buf, buf[:n]


class AdamSet:
    """Tensors of every configuration: the sizes above, 1 100 tiny tensors (more chunks than the grid), and one tensor
    with gradients near eps; fp32 / bf16 gradients, with / without a bf16 param, wd 0 / 0.01, cycled.  Each tensor is
    (master, m, v, grad, param) as [:n] views of NaN-filled buffers."""

    def __init__(self, seed):
        g = _gen(seed)
        sizes = ADAM_SIZES + [3] * 1100 + [4096]
        self.near_eps = len(sizes) - 1
        self.bufs, self.views, self.wd = [], [], []
        for i, n in enumerate(sizes):
            s = 1e-8 if i == self.near_eps else 1.0
            p = torch.randn(n, generator=g, device="cuda")
            m = torch.randn(n, generator=g, device="cuda") * 0.1 * s
            v = torch.rand(n, generator=g, device="cuda") * 0.01 * s * s
            gr = torch.randn(n, generator=g, device="cuda") * s
            parts = [_framed(n, F32, p), _framed(n, F32, m), _framed(n, F32, v),
                     _framed(n, BF16 if i % 2 else F32, gr), _framed(n, BF16, p) if i % 3 != 1 else (None, None)]
            self.bufs.append([b for b, _ in parts])
            self.views.append([v_ for _, v_ in parts])
            self.wd.append(0.01 if i % 4 < 2 else 0.0)

    def table(self, C_):
        cols = list(zip(*self.views))
        return C_.adam_build_tables(list(cols[3]), list(cols[0]), list(cols[1]), list(cols[2]), list(cols[4]), self.wd)

    def snapshot(self):
        return [[None if b is None else b.clone() for b in bs] for bs in self.bufs]

    def verify(self, ck, name, before, gs, step, lr=LR):
        """Every tensor's step against float64 from `before` (the buffers before the step).  The tensors are checked
        concatenated, the near-eps one on its own."""
        groups = {"adamw master": [i for i in range(len(self.bufs)) if i != self.near_eps],
                  "adamw master (near eps)": [self.near_eps]}
        cat = lambda ts: torch.cat([t.reshape(-1) for t in ts])  # noqa: E731
        for key, idx in groups.items():
            ns = [self.views[i][0].numel() for i in idx]
            old = [cat(before[i][r][:n].to(F64) for i, n in zip(idx, ns)) for r in range(4)]
            wd = cat(torch.full((n,), _f32(self.wd[i]), dtype=F64, device="cuda") for i, n in zip(idx, ns))
            m1, v1, p1, tm, tv, sc = adam_ref(*old, gs, _f32(lr), _f32(BETA1), _f32(BETA2), _f32(EPS), wd, step)
            got = [cat(self.views[i][r] for i in idx) for r in range(3)]
            ck.fp32("adamw m", f"{name} {key} m", got[1], m1, tm)
            ck.fp32("adamw v", f"{name} {key} v", got[2], v1, tv)
            ck._add(key, master_rule(f"{name} {key}", got[0], p1, _f32(lr), sc))
        with_param = [i for i in range(len(self.bufs)) if self.views[i][4] is not None]
        ck.require(torch.equal(cat(self.views[i][4] for i in with_param).view(torch.int16),
                               cat(self.views[i][0] for i in with_param).to(BF16).view(torch.int16)),
                   f"{name}: a bf16 param is not the RNE of the kernel's fp32 master")
        for r, role in enumerate(("master", "m", "v", "grad", "param")):
            for dt, bits in ((F32, torch.int32), (BF16, torch.int16)):
                idx = [i for i in range(len(self.bufs)) if self.bufs[i][r] is not None and self.bufs[i][r].dtype == dt]
                if not idx:
                    continue
                tail = lambda bs: cat(bs[i][r][self.views[i][0].numel():] for i in idx).view(bits)  # noqa: E731
                ck.require(torch.equal(tail(self.bufs), tail(before)), f"{name}: a {role} buffer changed past n")
                if role == "grad":
                    ck.require(torch.equal(cat(self.views[i][3] for i in idx).view(bits),
                                           cat(before[i][3][:self.views[i][0].numel()] for i in idx).view(bits)),
                               f"{name}: a gradient changed")


@pytest.mark.gpu
@pytest.mark.parametrize("device_step", [False, True], ids=["host_step", "device_step"])
@pytest.mark.parametrize("scaled", [False, True], ids=["unscaled", "scale_clip"])
def test_adamw_step(device_step, scaled):
    from alpa_b200 import ops
    C_ = ops.native_module()
    ck = Checker()
    st = AdamSet(70 + 2 * device_step + scaled)
    tt, cc, *_keep = st.table(C_)
    assert cc.numel() // 16 > torch.cuda.get_device_properties(0).multi_processor_count * 8
    grad_scale = 0.75 if scaled else 1.0
    clip = torch.tensor([0.3], device="cuda") if scaled else None
    gs = _f32(_f32(grad_scale) * (_f32(0.3) if scaled else 1.0))
    for step in (1, 2, 1000):
        before = st.snapshot()
        stp = torch.tensor([float(step)], device="cuda") if device_step else None
        C_.adamw_step(tt, cc, LR, BETA1, BETA2, EPS, 1 if device_step else step, grad_scale, clip, stp)
        torch.cuda.synchronize()
        st.verify(ck, f"{'device' if device_step else 'host'} step {step} scale {gs:.4g}", before, gs, step)
    _report(ck)


@pytest.mark.gpu
def test_fused_adamw_primitive_stages_non_contiguous_grads():
    """primitives.fused_adamw_ with a transposed (non-contiguous) gradient: the staging copy feeds the kernel."""
    from alpa_b200.ops import primitives as P
    ck = Checker()
    g = _gen(90)
    shapes = [(64, 40), (1000,)]
    masters = [torch.randn(s, generator=g, device="cuda") for s in shapes]
    ms = [torch.randn(s, generator=g, device="cuda") * 0.1 for s in shapes]
    vs = [torch.rand(s, generator=g, device="cuda") * 0.01 for s in shapes]
    params = [t.to(BF16) for t in masters]
    grads = [torch.randn(40, 64, generator=g, device="cuda").t(), torch.randn(1000, generator=g, device="cuda").to(BF16)]
    assert not grads[0].is_contiguous()
    before = [[t.clone() for t in ts] for ts in (masters, ms, vs)]
    P.fused_adamw_(params, masters, ms, vs, grads, torch.tensor(3, device="cuda"), LR, BETA1, BETA2, EPS, [0.01, 0.0],
                   1.0)
    torch.cuda.synchronize()
    for i in range(2):
        m1, v1, p1, tm, tv, sc = adam_ref(before[0][i], before[1][i], before[2][i], grads[i], 1.0, _f32(LR),
                                          _f32(BETA1), _f32(BETA2), _f32(EPS), _f32([0.01, 0.0][i]), 3)
        ck.fp32("adamw m", f"fused_adamw_ {i} m", ms[i], m1, tm)
        ck.fp32("adamw v", f"fused_adamw_ {i} v", vs[i], v1, tv)
        ck._add("adamw master", master_rule(f"fused_adamw_ {i} master", masters[i], p1, _f32(LR), sc))
        ck.require(torch.equal(params[i].view(torch.int16), masters[i].to(BF16).view(torch.int16)),
                   f"fused_adamw_ {i}: bf16 param is not the RNE of the master")
    _report(ck)


# ---------------------------------------------------------------------------------------------------------------------
# GPU: argument checks raise before any launch
# ---------------------------------------------------------------------------------------------------------------------


@pytest.mark.gpu
def test_bindings_reject_unchecked_inputs():
    from alpa_b200 import ops
    C_ = ops.native_module()
    dev = "cuda"

    def raises(fn, what):
        n0 = C_.launch_count()
        with pytest.raises(RuntimeError):
            fn()
        torch.cuda.synchronize()
        assert C_.launch_count() == n0, f"{what}: launched before raising"

    def off(shape, dtype, elems):
        """A contiguous tensor of `shape` starting `elems` elements past a 16-byte boundary."""
        n = math.prod(shape)
        return torch.zeros(n + 16, device=dev, dtype=dtype)[elems:elems + n].view(shape)

    # decode_attention: every base 16-byte aligned
    B, h, D, S = 2, 4, 64, 32
    q = torch.zeros(B, 1, h, D, device=dev, dtype=BF16)
    kc = torch.zeros(B, S, h, D, device=dev, dtype=BF16)
    kv = torch.tensor([4], dtype=torch.int32, device=dev)
    for i, what in enumerate(("q", "k_new", "v_new", "k_cache", "v_cache")):
        args = [q, q, q, kc, kc.clone()]
        args[i] = off(tuple(args[i].shape), BF16, 4)
        raises(lambda: C_.decode_attention(*args, kv, 0.125), f"decode_attention {what} 8-byte aligned")
    # ragged_attention: cache bases 16-byte aligned; a score buffer above 200 KB
    T = 3
    qr = torch.zeros(T, h, D, device=dev, dtype=BF16)
    cr = torch.zeros(40, h, D, device=dev, dtype=BF16)
    ss = torch.zeros(T, dtype=torch.int32, device=dev)
    cl = torch.ones(T, dtype=torch.int32, device=dev)
    raises(lambda: C_.ragged_attention(qr, off((40, h, D), BF16, 4), cr, ss, cl, 0.125, 8, None), "ragged k_cache")
    raises(lambda: C_.ragged_attention(qr, cr, off((40, h, D), BF16, 4), ss, cl, 0.125, 8, None), "ragged v_cache")
    raises(lambda: C_.ragged_attention(qr, cr, cr, ss, cl, 0.125, 60000, None), "ragged 240 KB score buffer")
    # embedding_fwd
    ids = torch.zeros(4, dtype=torch.long, device=dev)
    pos = torch.zeros(4, dtype=torch.long, device=dev)
    wte = torch.zeros(16, 64, device=dev, dtype=BF16)
    wpe = torch.zeros(8, 64, device=dev, dtype=BF16)
    raises(lambda: C_.embedding_fwd(ids, None, off((16, 64), BF16, 4), None, 0), "embedding wte 8-byte aligned")
    raises(lambda: C_.embedding_fwd(ids, pos, wte, wpe.float(), 0), "embedding fp32 wpe")
    raises(lambda: C_.embedding_fwd(ids, pos, wte, torch.zeros(64, 8, device=dev, dtype=BF16).t(), 0),
           "embedding non-contiguous wpe")
    raises(lambda: C_.embedding_fwd(ids, pos, wte, torch.zeros(8, 56, device=dev, dtype=BF16), 0), "embedding narrow wpe")
    raises(lambda: C_.embedding_fwd(ids, pos, wte, off((8, 64), BF16, 4), 0), "embedding wpe 8-byte aligned")
    raises(lambda: C_.embedding_fwd(ids, pos, wte, None, 0), "embedding pos without wpe")
    raises(lambda: C_.embedding_fwd(ids, None, wte, wpe, 0), "embedding wpe without pos")
    # MoE
    G, Sm, E, M, Cm = 2, 16, 4, 64, 8
    x = torch.zeros(G, Sm, M, device=dev, dtype=BF16)
    ex = torch.zeros(G, Sm, 2, dtype=torch.long, device=dev)
    sl = torch.zeros(G, Sm, 2, dtype=torch.long, device=dev)
    w = torch.zeros(G, Sm, 2, device=dev, dtype=BF16)
    d = torch.zeros(E, G * Cm, M, device=dev, dtype=BF16)
    raises(lambda: C_.moe_dispatch_(x, ex, sl.int(), w, d, Cm, [], 0), "moe_dispatch int32 slot")
    raises(lambda: C_.moe_dispatch_(x, ex[:, :8].contiguous(), sl[:, :8].contiguous(), w[:, :8].contiguous(), d, Cm,
                                    [], 0), "moe_dispatch short expert / slot")
    raises(lambda: C_.moe_dispatch_(x, ex, sl, w[:, :8].contiguous(), d, Cm, [], 0), "moe_dispatch short weight")
    raises(lambda: C_.moe_dispatch_(off((G, Sm, M), BF16, 4), ex, sl, w, d, Cm, [], 0), "moe_dispatch x aligned")
    raises(lambda: C_.moe_dispatch_(x, ex, sl, w, off((E, G * Cm, M), BF16, 4), Cm, [], 0), "moe_dispatch d aligned")
    raises(lambda: C_.moe_combine(d, ex, sl.int(), w, [], 0), "moe_combine int32 slot")
    raises(lambda: C_.moe_combine(d, ex, sl[:, :8].contiguous(), w, [], 0), "moe_combine short slot")
    raises(lambda: C_.moe_combine(d, ex, sl, w[:, :8].contiguous(), [], 0), "moe_combine short weight")
    raises(lambda: C_.moe_combine(off((E, G * Cm, M), BF16, 4), ex, sl, w, [], 0), "moe_combine eo aligned")
    raises(lambda: C_.moe_combine_wgrad(x, d, ex, sl.int(), [], 0), "moe_combine_wgrad int32 slot")
    raises(lambda: C_.moe_combine_wgrad(x[:, :8].contiguous(), d, ex, sl, [], 0), "moe_combine_wgrad short dout")
    raises(lambda: C_.moe_combine_wgrad(off((G, Sm, M), BF16, 4), d, ex, sl, [], 0), "moe_combine_wgrad dout aligned")
    raises(lambda: C_.moe_combine_wgrad(x, off((E, G * Cm, M), BF16, 4), ex, sl, [], 0), "moe_combine_wgrad eo aligned")
    # adam_build_tables: equal numel and aligned bases
    n = 64
    f = lambda: torch.zeros(n, device=dev)  # noqa: E731
    good = dict(g=f(), p=f(), m=f(), v=f(), b=torch.zeros(n, device=dev, dtype=BF16))
    bad = [("g", f()[:n - 4], "short grad"), ("b", torch.zeros(n - 1, device=dev, dtype=BF16), "short param"),
           ("m", f()[:n - 1], "short m"), ("p", off((n,), F32, 1), "master 4-byte aligned"),
           ("m", off((n,), F32, 2), "m 8-byte aligned"), ("v", off((n,), F32, 3), "v 4-byte aligned"),
           ("g", off((n,), BF16, 1), "bf16 grad 2-byte aligned"), ("b", off((n,), BF16, 2), "bf16 param 4-byte aligned")]
    for k, t, what in bad:
        a = dict(good)
        a[k] = t
        raises(lambda: C_.adam_build_tables([a["g"]], [a["p"]], [a["m"]], [a["v"]], [a["b"]], [0.0]),
               f"adam_build_tables {what}")

"""The Q8_0 / Q4_0 streaming matvec (matvec_stream.cu: eager and lazy mode 1) and the ring kernel's streaming MATVEC phase
(mega_ring.cu phase_matvec_ring + mr_producer: lazy mode 2) at the edges of their row dealing, segment layout and fused prologues.

Each case is an op sequence through the Python mirror, flushed twice (the first flush captures, the second replays) on a fresh device
with the persistent grid fixed by set_sm_limit, in lazy modes 0, 1 and 2.  It checks:
  * modes 1 and 2 bit-identical to eager, and no uncached flush;
  * mode 2's kernel variant and phase-table fingerprint, so a case cannot pass without reaching the phase it is about (or, where the
    fuser declines -- the ring does not fit, or an exchange block outgrows its stage -- the declining plan);
  * mode 1's kernel launches per flush, so an epilogue or prologue that silently stops fusing fails;
  * where no norm and no silu pair is fused, the oracle's gemv within the per-op budget of test_gpu_matvec.py.
The cases: 1-3 matrices on one row (three q/k/v-shaped), the gate/up pair and the residual epilogue, four matvecs on one normalised row;
plain, fused-norm, [dup] fused-norm and written-back-norm prologues; row lengths at every segment / group edge up to the 32768-column
limit (and one past it); row counts that give CTAs zero units, one unit, pairs plus an odd unit, several pairs per warp, and units
that straddle two matrices; grid independence; the exchange epilogue in a world of one; edge rows through the prologue quantisers;
and the widest row each prologue kind still runs through the ring."""
import numpy as np
import pytest

from oracle import oracle as oc
from oracle.synth import synth_weight
from crabml_b200.runner import synth_scale
from crabml_b200.tensor import MEGA_NONE, MEGA_RING
from tests.gpu_common import assert_same_bits, full_grid, run_modes
from tests.test_gpu_matvec import gemv_budget
from tests.test_gpu_weight_types import EPS, ORACLE_THREADS, WSEED, _mv_code, flushes

pytestmark = pytest.mark.gpu

TYPES = [oc.Q8_0, oc.Q4_0]
ROUNDS = 2


@pytest.fixture(autouse=True)
def _mega_prof(monkeypatch):
    monkeypatch.setenv("CRABML_MEGA_PROF", "1")       # phase table fingerprints (mega_phase_types)


# Widest row (a multiple of 32 columns) whose streaming phase still gets the ring, by prologue: "norm" = a fused rms_norm * w (the
# working area holds the f32 row and the norm-weight stage as well: 8 bytes per column), "plain" = a merged plain quantise (the f32
# row only).  Past it the table has fewer than 12 ring slots and runs in the CUDA-graph mode.  A phase that reads a quantised row
# (written-back norm, several groups on one row) fits at every k up to the 32768-column limit.  Probed on an NVIDIA H100 80GB HBM3
# (700 W) by test_ring_fit_switch; mega_ring_kernel has 7168 bytes of static shared memory (ptxas, CUDA 12.9), and the layout
# arithmetic of cc_mega_ring_slots gives the same four values:
#   Q8_0: norm 18144, plain 32448      Q4_0: norm 20576, plain 32768 (the limit: always fits)
RING_MAX_K = {(oc.Q8_0, "norm"): 18144, (oc.Q8_0, "plain"): 32448, (oc.Q4_0, "norm"): 20576, (oc.Q4_0, "plain"): 32768}

# ---- group shapes, prologues, row lengths, row counts ---------------------------------------------------------------------------------
NMAT = {"one": 1, "two": 2, "three": 3, "pair": 2, "res": 1, "four": 4}
EPILOGUE = {"one": 0, "two": 0, "three": 0, "pair": 2, "res": 1, "four": 0}
# plain: x quantised in the phase's prologue; norm: rms_norm * w fused into it; dup: [dup] + fused norm, CTA 0 writes the raw row out;
# wb: the normalised row is read again afterwards, so a NORMQ phase writes it back and the matvec phase reads the quantised row
PROLOGUES = ["plain", "norm", "dup", "wb"]
# 32 = one block; 288 = 9; 992 = 31 (a partial first group); 1024 = one group; 1056 = a second group of one block; 4096 = one segment;
# 4128 = a second segment of one block; 5120 = a second segment of one whole group; 11008 / 13824 = partial last groups; 14336;
# 32736 = 8 segments, the last one block short; 32768 = the cc_stream_supported limit
K_ALL = [32, 288, 992, 1024, 1056, 4096, 4128, 5120, 11008, 13824, 14336, 32736, 32768]


def _r4(n, up):
    return (n + 3) & ~3 if up else n & ~3


def row_counts(grid):
    """(rows of a plain group, rows of a group with an epilogue) -- an epilogue's rows are 1 or a multiple of 4: the reference's add / mul
    skips the tail past the last multiple of 4 of a longer row, which a fused epilogue does not (test_gpu_weight_types.TAIL_CASES).
    grid 5: 1; 3 / 4 (CTAs without units); 5 / 8 (one unit each: the lone-unit arm); 6 / 12 and 15 / 16 (pairs plus an odd last unit);
    163 / 164 (every warp claims several pairs).  Full grid: 1, grid - 1, grid, grid + 1, and more rows than 16 warps x 2 x grid."""
    if grid == 5:
        return [(1, 1), (3, 4), (5, 8), (6, 12), (15, 16), (163, 164)]
    g = full_grid()
    return [(1, 1), (g - 1, _r4(g - 1, False)), (g, _r4(g, True)), (g + 1, _r4(g + 1, True)), (33 * g + 7, _r4(33 * g + 7, True))]


def _ms(shape, m):
    """rows of each matrix: q/k/v-shaped (unequal) for three -- at grid 5 with m not a multiple of 5 a CTA's units straddle matrices"""
    if shape == "three":
        return [m, (m + 3) // 4, (m + 3) // 4]
    if shape == "four":
        return [m, (m + 3) // 4, (m + 3) // 4, m]
    return [m] * NMAT[shape]


def _cases():
    """every type x prologue x group shape, k rotating over K_ALL and (grid, rows) over both grids' row counts; plus four matvecs on one
    normalised row.  Q8_0's two widest rows land on the written-back norm, the only prologue with which they still run in the ring."""
    combos = [(5, i) for i in range(6)] + [(0, i) for i in range(5)]
    out = []
    for ti, t in enumerate(TYPES):
        n = 0
        for pi, pro in enumerate(PROLOGUES):
            for si, shape in enumerate(["one", "two", "three", "pair", "res"]):
                k = K_ALL[(5 * pi + si + 6 * ti) % len(K_ALL)]
                grid, ri = combos[(n + 4 * ti) % len(combos)]
                out.append((t, shape, pro, k, grid, ri))
                n += 1
        out.append((t, "four", "norm", [4128, 1056][ti], 5, 3 + ti))
        out.append((t, "four", "dup", [13824, 32736][ti], 0, 4 - ti))
    out += [(oc.Q8_0, "one", "wb", 32736, 5, 2), (oc.Q8_0, "three", "wb", 32768, 0, 1)]
    return out


def _resolve(c):
    t, shape, pro, k, grid, ri = c
    pm, em = row_counts(grid)[ri]
    return t, shape, pro, k, grid, _ms(shape, em if EPILOGUE[shape] else pm)


def _case_id(c):
    t, shape, pro, k, grid, ri = c
    return f"{oc.TYPE_NAMES[t]}-{shape}-{pro}-k{k}-g{grid or 'full'}-r{ri}"


CASES = _cases()


def _inputs(k, n_res, rnd):
    """x, norm weights, residual row of round `rnd`: new values every round, so that a replayed graph cannot pass on a stale result"""
    rng = np.random.default_rng([k, n_res, rnd])
    x = rng.standard_normal(k).astype(np.float32)
    nw = (1.0 + 0.05 * rng.standard_normal(k)).astype(np.float32)
    r = rng.standard_normal(n_res).astype(np.float32)
    return x, nw, r


def _groups(ms):
    """matvec groups the fuser forms on one row: up to three matrices each"""
    return [ms[i:i + 3] for i in range(0, len(ms), 3)]


def _body(case, x_of=None, nw_of=None):
    """-> body(flush, round).  Uploads: x, the norm weights, the residual row (each if used).  The normalised row is dropped before the
    export unless the prologue is "wb"; x_of / nw_of(k, round) override the row / the norm weights (edge rows)."""
    t, shape, pro, k, grid, ms = case

    def body(f, rnd):
        x_h, nw_h, r_h = _inputs(k, ms[0], rnd)
        if x_of:
            x_h = x_of(k, rnd)
        if nw_of:
            nw_h = nw_of(k, rnd)
        x = f.T(x_h)
        outs = []
        if pro != "plain":
            nw = f.T(nw_h)
        if shape == "res":
            res = f.T(r_h)
        if pro != "plain":
            if pro == "dup":
                outs.append(x.dup())
            x.rms_norm_inplace(EPS).mul_inplace(nw)
        ys = [f.W(m, k, t, i + 1).matmul_vec(x) for i, m in enumerate(ms)]
        if pro == "wb":
            outs.append(x)
        del x
        if shape == "pair":
            g, u = ys
            g.silu_inplace().mul_inplace(u)
            del u
            ys = [g]
        elif shape == "res":
            ys[0].add_inplace(res)
        return np.concatenate([y.export() for y in ys + outs])
    return body


def _uploads(case):
    t, shape, pro, k, grid, ms = case
    return 1 + (pro != "plain") + (shape == "res")


def _fits(t, pro, k, n_groups):
    """does the ring take the table (RING_MAX_K)?  A merged prologue stages the f32 row (and a fused norm its weights) in the working
    area; a NORMQ phase of its own leaves the matvec phases a quantised row to read"""
    if pro == "wb" or n_groups > 1:
        return True
    return k <= RING_MAX_K[t, "plain" if pro == "plain" else "norm"]


def _expected(case):
    """(mode-2 variant, fingerprint), mode-1 launches per flush.  Mode 1: one upload each, one quantise / normq, one streaming launch per
    group.  Mode 2: the uploads (48), a NORMQ phase (0) unless the prologue merges into the only group, one MATVEC phase per group."""
    t, shape, pro, k, grid, ms = case
    gs = _groups(ms)
    launches = _uploads(case) + 1 + len(gs)
    if not _fits(t, pro, k, len(gs)):
        return (MEGA_NONE, ()), launches
    normq = (0,) if pro == "wb" or len(gs) > 1 else ()
    return (MEGA_RING, (48,) * _uploads(case) + normq + tuple(_mv_code(len(g), EPILOGUE[shape], k) for g in gs)), launches


def _assert_modes(body, plan, launches, what, grid=0, comm=False, live=True):
    """lazy modes 1 and 2 bit-identical to eager, mode 1 with `launches` launches, mode 2 with plan (variant, fingerprint) -> eager output.
    live: the output is finite and not all zero"""
    res = run_modes(flushes(body, grid, comm))
    ref = res[0][4]
    for mode in (1, 2):
        assert res[mode][2]["uncached"] == 0, (what, mode, res[mode][2])
        assert_same_bits(res[mode][4], ref, f"{what}: lazy={mode} vs eager")
    assert res[1][3] == launches, (what, "mode-1 launches", res[1][3], launches)
    assert res[2][:2] == plan, (what, res[2][:2], plan)
    if live:
        assert np.isfinite(ref).all() and np.abs(ref).max() > 1e-3, what
    return ref


def _assert_oracle(t, k, ms, x, got, what, res=None):
    """each matrix's rows against oc.gemv within gemv_budget (+ one f32 rounding where the residual is added).  Non-finite rows must be
    the oracle's non-finite rows: NaN where it has NaN, inf of the same sign where it has inf."""
    o = 0
    for i, m in enumerate(ms):
        raw = synth_weight(t, m, k, WSEED, i + 1, synth_scale(t, k))
        want = oc.gemv(t, raw, m, k, x, threads=ORACLE_THREADS).astype(np.float64)
        with np.errstate(invalid="ignore"):
            budget = gemv_budget(t, raw, m, k, x)
        if res is not None and i == 0:
            want = want + res[:m].astype(np.float64)
            with np.errstate(invalid="ignore"):
                budget = budget + np.spacing(np.abs(want).astype(np.float32)).astype(np.float64)
        g = got[o:o + m].astype(np.float64)
        fin = np.isfinite(want)
        assert (np.isfinite(g) == fin).all(), (what, i, "finite rows differ", np.flatnonzero(np.isfinite(g) != fin)[:8].tolist())
        assert (np.isnan(g) == np.isnan(want)).all(), (what, i, "NaN rows differ")
        inf = np.isinf(want)
        assert (np.sign(g[inf]) == np.sign(want[inf])).all(), (what, i, "inf of another sign")
        diff = np.abs(g[fin] - want[fin])
        assert (diff <= budget[fin]).all(), (what, i, float((diff / budget[fin]).max()))
        o += m


@pytest.mark.parametrize("c", CASES, ids=[_case_id(c) for c in CASES])
def test_stream_phase_vs_eager_and_oracle(c):
    case = _resolve(c)
    t, shape, pro, k, grid, ms = case
    plan, launches = _expected(case)
    ref = _assert_modes(_body(case), plan, launches, _case_id(c), grid)
    if pro != "plain" or shape == "pair":
        return                   # the eager rms_norm, silu and mul kernels are pinned to the oracle elsewhere; bit-identity is the check
    x, _, r = _inputs(k, ms[0], ROUNDS - 1)
    _assert_oracle(t, k, ms, x, ref, _case_id(c), r if shape == "res" else None)


def test_case_list_reaches_every_edge():
    """(the rotation above) every type meets every row length, every row count of both grids, and every prologue with every shape"""
    for t in TYPES:
        cs = [c for c in CASES if c[0] == t]
        assert {c[3] for c in cs} >= set(K_ALL), oc.TYPE_NAMES[t]
        assert {(c[4], c[5]) for c in cs} >= {(5, i) for i in range(6)} | {(0, i) for i in range(5)}, oc.TYPE_NAMES[t]
        assert any(c[1] == "three" and c[4] == 5 and c[5] in (0, 1, 3, 5) for c in cs)      # m0 % 5 != 0: units straddle matrices
        ring = [c for c in cs if _expected(_resolve(c))[0][0] == MEGA_RING]
        assert {c[3] for c in ring} >= set(K_ALL), (oc.TYPE_NAMES[t], "every k through the ring")


def test_row_past_the_stream_limit():
    """k = 32800: not streamed (cc_stream_supported), so the fuser leaves the matvec to its eager kernel (matvec.cu: quantise +
    warp-per-row matvec) and the flush runs in the CUDA-graph mode -- and the result still matches the oracle"""
    for t in TYPES:
        case = (t, "one", "plain", 32800, 0, [40])
        ref = _assert_modes(_body(case), (MEGA_NONE, ()), 3, f"{oc.TYPE_NAMES[t]}-k32800")
        x, _, _ = _inputs(32800, 40, ROUNDS - 1)
        _assert_oracle(t, 32800, [40], x, ref, f"{oc.TYPE_NAMES[t]}-k32800")


# ---- grid independence -------------------------------------------------------------------------------------------------------------
GRID_CASES = [(oc.Q8_0, "three", "plain", 4128, [163, 41, 41]), (oc.Q4_0, "pair", "norm", 1056, [164, 164]),
              (oc.Q8_0, "res", "dup", 5120, [164]), (oc.Q4_0, "four", "norm", 992, [163, 41, 41, 163])]


@pytest.mark.parametrize("c", GRID_CASES, ids=[f"{oc.TYPE_NAMES[c[0]]}-{c[1]}-{c[2]}-k{c[3]}" for c in GRID_CASES])
def test_rows_do_not_depend_on_the_grid(c):
    """A row's bits do not depend on which warp or CTA computes it: eager and mode 2 at grids of 1, 2, 5, 7 and every SM agree bit for
    bit -- a row dealt twice or never would show up here."""
    t, shape, pro, k, ms = c
    outs = []
    for grid in (1, 2, 5, 7, 0):
        res = run_modes(flushes(_body((t, shape, pro, k, grid, ms)), grid), modes=(0, 2))
        assert res[2][0] == MEGA_RING, (c, grid, res[2][0])
        outs += [(grid, mode, res[mode][4]) for mode in (0, 2)]
    g0, m0, ref = outs[0]
    assert np.isfinite(ref).all() and np.abs(ref).max() > 1e-3
    for grid, mode, out in outs[1:]:
        assert_same_bits(out, ref, f"grid {grid} lazy={mode} vs grid {g0} eager")


# ---- the exchange epilogue in a world of one --------------------------------------------------------------------------------------------
def _xchg_body(t, k, m, kind):
    """reduce: matvec -> all_reduce -> + residual; fold: the same, then [dup] rms_norm * w -> matvec (m x m), whose prologue folds the
    REDUCE in; gather: matvec -> all_gather_from.  Every row is uploaded first: the fuser matches the exchange only when the
    all_reduce directly follows the matvec."""
    def body(f, rnd):
        from crabml_b200 import CudaTensor, capi
        x_h, nw_h, r_h = _inputs(max(k, m), m, rnd)
        x = f.T(x_h[:k])
        if kind != "gather":
            r = f.T(r_h)
        if kind == "fold":
            nw = f.T(nw_h[:m])
        y = f.W(m, k, t, 1).matmul_vec(x)
        if kind == "gather":
            return CudaTensor.alloc([m], capi.F32, f.dev).all_gather_from(y).export()
        y.all_reduce_sum_inplace().add_inplace(r)
        if kind == "reduce":
            return y.export()
        z = y.dup()
        y.rms_norm_inplace(EPS).mul_inplace(nw)
        out = f.W(m, m, t, 2).matmul_vec(y)
        del y
        return np.concatenate([out.export(), z.export()])
    return body


def _xchg_cases():
    """rows: 4 (one CTA's block, the others empty), 4 x grid (one full block each), 4 x grid + 4 (partial and empty trailing blocks),
    4000, 32768 -- "4g" / "4g+4" resolved against the grid at run time"""
    out = []
    for t in TYPES:
        for grid in (5, 0):
            for m in (4, "4g", "4g+4", 4000, 32768):
                out.append((t, "reduce", 2048, m, grid))
        out += [(t, "fold", 1024, 4096, 0), (t, "fold", 1024, 16384, 0), (t, "fold", 1024, 4096, 5)]
        out += [(t, "gather", 4096, 1024, 0), (t, "gather", 4096, 20, 5), (t, "gather", 4096, 4000, 5)]
    return out


def _xchg_rows(m, grid):
    g = grid or full_grid()
    return {"4g": 4 * g, "4g+4": 4 * g + 4}.get(m, m)


def _xchg_id(c):
    t, kind, k, m, grid = c
    return f"{oc.TYPE_NAMES[t]}-{kind}-k{k}-m{m}-g{grid or 'full'}"


def _xchg_expected(c):
    """Exchange phases give each CTA one contiguous block of rpc = ceil(m / grid) rounded up to 4 rows (mega_ring.cu mr_geo): trailing
    CTAs get a partial block or none.  A block larger than the 512-row exchange stage sends the table to the CUDA-graph mode (lazy.cu).
    In mode 1 the all_reduce (with the residual) / all_gather is a launch of its own."""
    t, kind, k, m, grid = c
    g = grid or full_grid()
    uploads = {"gather": 1, "reduce": 2, "fold": 3}[kind]
    launches = uploads + 3 + (2 if kind == "fold" else 0)
    if ((m + g - 1) // g + 3) & ~3 > 512:
        return (MEGA_NONE, ()), launches
    xmv = _mv_code(1, 3, k)
    fp = {"gather": (48, xmv, 80), "reduce": (48, 48, xmv, 64), "fold": (48, 48, 48, xmv, _mv_code(1, 0, m))}[kind]
    return (MEGA_RING, fp), launches


XCHG_CASES = _xchg_cases()


@pytest.mark.parametrize("c", XCHG_CASES, ids=[_xchg_id(c) for c in XCHG_CASES])
def test_exchange_epilogue_world_of_one(c):
    """with one rank the exchange is the identity: bit-identity with eager (which runs the same ops through comm.cu), and the oracle for
    reduce (+ the residual) and gather.  fold at k 4096 sums its row in registers, at 16384 in the 4-chunk loop."""
    t, kind, k, m, grid = c
    m = _xchg_rows(m, grid)
    plan, launches = _xchg_expected((t, kind, k, m, grid))
    ref = _assert_modes(_xchg_body(t, k, m, kind), plan, launches, _xchg_id(c), grid, comm=True)
    if kind == "fold":
        return
    x_h, _, r_h = _inputs(max(k, m), m, ROUNDS - 1)
    _assert_oracle(t, k, [m], x_h[:k], ref, _xchg_id(c), r_h if kind == "reduce" else None)


# ---- edge rows through the prologue quantisers --------------------------------------------------------------------------------------------
F16_MAX_D = 65504.0 * 127.0          # max|x| of a block whose scale d = max|x| / 127 is the largest finite f16


def _edge_row(overflow):
    """k = 4128 (the last block is a segment of its own): an all-zero block (d = 0, every quotient 0/0), a block whose max is ~1e-39
    (d subnormal, rounds to f16 0), the quantize KAT ramp, a block whose max |x| occurs as +a and -a, a block just below the f16
    overflow of d -- and, with `overflow`, a last block whose d rounds to f16 inf (every row becomes +-inf, or NaN where its integer dot
    with that block is 0)"""
    def x_of(k, rnd):
        rng = np.random.default_rng([k, 77, rnd, overflow])
        x = rng.standard_normal(k).astype(np.float32)
        x[0:32] = 0.0
        x[32:64] = (rng.standard_normal(32) * 1e-39).astype(np.float32)
        x[64:96] = np.tile(np.arange(-8, 8, dtype=np.float32), 2)
        b = rng.uniform(-1.0, 1.0, 32).astype(np.float32)
        b[5], b[17] = -2.5, 2.5
        x[96:128] = b
        big = np.float32(F16_MAX_D * 0.999)
        b = (rng.uniform(-0.5, 0.5, 32) * big).astype(np.float32)
        b[11] = -big
        x[128:160] = b
        if overflow:
            x[k - 32:] = (rng.uniform(-0.5, 0.5, 32) * F16_MAX_D).astype(np.float32)
            x[k - 7] = np.float32(F16_MAX_D * 1.001)
        return x
    return x_of


@pytest.mark.parametrize("overflow", [False, True], ids=["finite", "d-overflow"])
@pytest.mark.parametrize("t", TYPES, ids=[oc.TYPE_NAMES[t] for t in TYPES])
def test_plain_quantise_prologue_on_edge_rows(t, overflow):
    """the ring prologue's quant_chunk against the eager quantiser bit for bit (NaN / inf positions included), and against the oracle"""
    case = (t, "two", "plain", 4128, 0, [40, 40])
    x_of = _edge_row(overflow)
    plan, launches = _expected(case)
    what = f"{oc.TYPE_NAMES[t]}-edge-{overflow}"
    ref = _assert_modes(_body(case, x_of=x_of), plan, launches, what, live=False)
    assert np.isfinite(ref).all() != overflow, what
    _assert_oracle(t, 4128, [40, 40], x_of(4128, ROUNDS - 1), ref, what)


def _zero_row(k, rnd):
    return np.zeros(k, np.float32)


def _edge_norm_w(k, rnd):
    nw = (1.0 + 0.05 * np.random.default_rng([k, 78, rnd]).standard_normal(k)).astype(np.float32)
    nw[32:64] = 0.0                                   # a zero block: every quotient 0/0
    nw[64:96] = np.float32(1e-39)                     # subnormal products (the build keeps denormals: -ftz=false)
    return nw


@pytest.mark.parametrize("edge", ["zero-row", "norm-weights"])
@pytest.mark.parametrize("t", TYPES, ids=[oc.TYPE_NAMES[t] for t in TYPES])
def test_fused_norm_prologue_on_edge_rows(t, edge):
    """an all-zero row under rms_norm (rms = sqrt(eps), every block 0/0) and norm weights with a zero and a subnormal block, through
    the fused [dup] norm prologue: bit-identical to the eager rms_norm, mul and quantise kernels"""
    case = (t, "one", "dup", 4128, 0, [40])
    kw = {"x_of": _zero_row} if edge == "zero-row" else {"nw_of": _edge_norm_w}
    plan, launches = _expected(case)
    ref = _assert_modes(_body(case, **kw), plan, launches, f"{oc.TYPE_NAMES[t]}-{edge}", live=edge != "zero-row")
    assert np.isfinite(ref).all()
    if edge == "zero-row":
        assert not ref.any()


# ---- where the ring stops fitting --------------------------------------------------------------------------------------------------------
def _fit_case(t, pro, k):
    return (t, "one", "norm" if pro == "norm" else "plain", k, 0, [64])


def _ring_takes(t, pro, k):
    return run_modes(flushes(_body(_fit_case(t, pro, k)), rounds=1), modes=(2,))[2][0] == MEGA_RING


@pytest.mark.parametrize("pro", ["norm", "plain"])
@pytest.mark.parametrize("t", TYPES, ids=[oc.TYPE_NAMES[t] for t in TYPES])
def test_ring_fit_switch(t, pro):
    """The widest k (a multiple of 32) at which lazy mode 2 still runs a fused-norm / plain-quantise phase in the ring, bisected with
    one fresh device per candidate.  At that k the ring has its fewest slots and the staged row (and norm weights) are at their widest:
    both sides of the switch are bit-identical to eager, and the switch is where RING_MAX_K says."""
    lo, hi = 8192, 32768
    assert _ring_takes(t, pro, lo)
    if _ring_takes(t, pro, hi):
        lo = hi
    else:
        while hi - lo > 32:
            mid = (lo + hi) // 64 * 32
            if _ring_takes(t, pro, mid):
                lo = mid
            else:
                hi = mid
    print(f"ring fit switch: {oc.TYPE_NAMES[t]} {pro}: widest k {lo}")
    assert lo == RING_MAX_K[t, pro], (oc.TYPE_NAMES[t], pro, lo)
    for k in sorted({lo, min(lo + 32, 32768)}):
        case = _fit_case(t, pro, k)
        plan, launches = _expected(case)
        _assert_modes(_body(case), plan, launches, f"{oc.TYPE_NAMES[t]}-{pro}-k{k}")

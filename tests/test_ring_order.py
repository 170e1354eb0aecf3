"""The ring order of mega_ring.cu, restated in Python: the producer warps enumerate a CTA's entries of a streaming MATVEC phase in one
order (mr_producer), the consumer warps claim pairs of units and walk the same entries by index arithmetic (phase_matvec_ring).  Both
sides must agree on which (unit, virtual row, segment) sits in entry e, every entry must be produced exactly once, and the two entries a
pair round touches must be adjacent.  This test pins the arithmetic (a change on one side of the CUDA file has to be mirrored here and on
the other side); the CUDA code itself is checked on the GPU by the bit-identity tests (tests/test_gpu_runner.py) and, at every ragged
shape below and at fixed grids, by tests/test_gpu_stream_phase.py.  The bounds test restates mr_producer's two bulk copies per entry
and the consumer's reads of a landed slot (mr_dot2)."""
import itertools

import pytest

MK_SEG = 4
GRID = 132                     # one CTA per SM of an H100 SXM
GRIDS = [5, 114, 132]          # a small fixed grid (tests/test_gpu_stream_phase.py), an H100 PCIe, an H100 SXM


def _m_cat(m, n_mats, epilogue):
    """rows of the phase: m is the rows of every matrix, or a tuple of each matrix's rows (q/k/v-shaped groups)"""
    ms = list(m) if isinstance(m, tuple) else [m] * n_mats
    return ms[0] if epilogue == 2 else sum(ms)


def geo(m, n_mats, k, epilogue, cta, grid=GRID):
    """mr_geo: rows of the phase that belong to CTA `cta` as units (unit u -> concatenated row first + u * stride)."""
    nb = k // 32
    gr = (nb + 31) // 32
    nseg = (gr + MK_SEG - 1) // MK_SEG
    pair = epilogue == 2
    m_cat = _m_cat(m, n_mats, epilogue)
    if epilogue == 3:
        rpc = ((m_cat + grid - 1) // grid + 3) & ~3
        first, stride = cta * rpc, 1
        n_units = min(rpc, max(0, m_cat - first))
    else:
        first, stride = cta, grid
        n_units = (m_cat - first + stride - 1) // stride if first < m_cat else 0
    v = 2 if pair else 1
    return dict(nb=nb, gr=gr, nseg=nseg, V=v, E=v * nseg, n_units=n_units, first=first, stride=stride)


def producer_order(g):
    """mr_producer: entry index j -> (unit, virtual row, segment)."""
    n, two_e = g["n_units"] * g["E"], 2 * g["E"]
    npair = (g["n_units"] >> 1) * two_e
    out = []
    for j in range(n):
        if j < npair:
            p, w = divmod(j, two_e)
            u, vs = 2 * p + (w & 1), w >> 1
        else:
            u, vs = g["n_units"] - 1, j - npair
        v, sg = divmod(vs, g["nseg"])
        out.append((u, v, sg))
    return out


def consumer_walk(g):
    """phase_matvec_ring: for every claim P the list of (entry index, unit, virtual row, segment) it consumes, in order."""
    e, two_e, npairs = g["E"], 2 * g["E"], g["n_units"] >> 1
    pairs = g["n_units"] > 1                                          # a lone unit: the single-unit arm (same claim either way)
    claims = []
    for p in itertools.count():
        two = pairs and p < npairs
        if pairs:
            if not two and not (p == npairs and (g["n_units"] & 1)):
                break
        elif p >= g["n_units"]:
            break
        u0 = p if not pairs else (2 * p if two else g["n_units"] - 1)
        step = 2 if two else 1
        ea = (p * e) if not pairs else (p * two_e if two else npairs * two_e)
        walk = []
        for v in range(g["V"]):
            for sg in range(g["nseg"]):
                walk.append((ea, u0, v, sg))
                if two:
                    walk.append((ea + 1, u0 + 1, v, sg))
                ea += step
        claims.append(walk)
    return claims


SHAPES = [  # (rows per matrix, matrices, k, epilogue)
    (4096, 3, 4096, 0), (4096, 1, 4096, 1), (11008, 2, 4096, 2), (4096, 1, 11008, 1), (32000, 1, 4096, 0),      # Llama-2-7B, one GPU
    (4096, 1, 2048, 3), (4096, 1, 5504, 3), (16000, 1, 4096, 3),                                                    # shards at N = 2 (exchange phases)
    (512, 3, 4096, 0), (4096, 1, 512, 3), (1376, 2, 4096, 2), (4096, 1, 1376, 3), (4000, 1, 4096, 3),               # shards at N = 8
    (288, 3, 288, 0), (288, 1, 288, 1), (768, 2, 288, 2), (288, 1, 768, 1), (32000, 1, 288, 0),                     # tinyllamas-15M (ragged groups)
    # ragged rows: one block (32), a second group (1056) / segment (4128) of one block, 8 segments one block short (32736), a partial
    # first group (992); rows that leave CTAs of a 5-CTA grid without units (3), give each one unit (5), pairs plus an odd unit (6, 15),
    # several pairs per warp (163), and units that straddle matrices of unequal size
    (1, 1, 32, 0), (3, 1, 1056, 0), (5, 1, 4128, 0), (6, 1, 32736, 0), (15, 2, 992, 2), (163, 1, 5120, 1), ((6, 2, 2), 3, 4128, 0),
    ((163, 41, 41), 3, 32, 0), (4, 1, 1056, 3), (24, 1, 4128, 3), (164, 2, 32736, 2), (133, 1, 32768, 0),
]
SHAPE_IDS = ["-".join(str(v) for v in s) if not isinstance(s[0], tuple) else "x".join(map(str, s[0])) + "-" + "-".join(map(str, s[1:])) for s in SHAPES]
# the H100 SXM ids stay those of the original grid-less parameters
CASES = [pytest.param(*s, grid, id=sid if grid == GRID else f"{sid}-g{grid}") for grid in GRIDS for s, sid in zip(SHAPES, SHAPE_IDS)]


@pytest.mark.parametrize("m,n_mats,k,epilogue,grid", CASES)
def test_producer_and_consumers_agree_on_the_ring_order(m, n_mats, k, epilogue, grid):
    covered_rows = set()
    for cta in sorted({0, 1, 2, grid - 1, 37, 146, 147}):
        g = geo(m, n_mats, k, epilogue, cta, grid)
        order = producer_order(g)
        # every (unit, virtual row, segment) of the CTA exactly once
        want = {(u, v, s) for u in range(g["n_units"]) for v in range(g["V"]) for s in range(g["nseg"])}
        assert len(order) == len(want) and set(order) == want
        seen = []
        for walk in consumer_walk(g):
            for idx, (e, u, v, s) in enumerate(walk):
                assert order[e] == (u, v, s), (cta, e, order[e], (u, v, s))
                seen.append(e)
            if len(walk) == 2 * g["E"]:                                       # a pair round: its two entries of every step are adjacent in the ring
                for a, b in zip(walk[0::2], walk[1::2]):
                    assert b[0] == a[0] + 1
        assert sorted(seen) == list(range(len(order)))                # the consumers release every slot exactly once
        covered_rows.update(g["first"] + u * g["stride"] for u in range(g["n_units"]))
    assert covered_rows                                               # (the sampled CTAs own rows)


@pytest.mark.parametrize("m,n_mats,k,epilogue,grid", CASES)
def test_every_row_of_a_phase_belongs_to_exactly_one_cta(m, n_mats, k, epilogue, grid):
    rows = []
    for cta in range(grid):
        g = geo(m, n_mats, k, epilogue, cta, grid)
        rows += [g["first"] + u * g["stride"] for u in range(g["n_units"])]
    assert sorted(rows) == list(range(_m_cat(m, n_mats, epilogue)))


def d_stride(nb):
    """CC_D_STRIDE: f16 scales per row of the scale plane, padded to 16 bytes"""
    return (nb + 7) // 8 * 8


@pytest.mark.parametrize("bb", [32, 16], ids=["Q8_0", "Q4_0"])
@pytest.mark.parametrize("m,n_mats,k,epilogue,grid", CASES)
def test_every_bulk_copy_stays_inside_its_row(m, n_mats, k, epilogue, grid, bb):
    """mr_producer, entry by entry: the quant copy [sg * 128 * BB, + nbe * BB) lies inside the row's nb * BB bytes, the scale copy
    [sg * 128, + dbytes / 2) inside its CC_D_STRIDE(nb) halves, and sizes and offsets (from the plane's start) are multiples of 16
    bytes; both land inside the slot (quants at 0, scales at MK_SEG * 32 * BB).  Then the consumer (mr_dot2) reads only landed bytes:
    lane l of group g reads 16 bytes at g * GB + 16 l and, for Q8_0, at + 512 -- or + 16 * (blocks of the group) in the last group --
    and the scale at 2 * (32 g + l) past the quants, for the blocks 32 (4 sg + g) + l < nb."""
    slot_bytes = 4352 if bb == 32 else 2304
    doff, gb = MK_SEG * 32 * bb, 32 * bb
    m_cat = _m_cat(m, n_mats, epilogue)
    ctas = range(grid) if m_cat * k <= (1 << 25) else sorted({0, 1, grid - 1})
    for cta in ctas:
        g = geo(m, n_mats, k, epilogue, cta, grid)
        nb = g["nb"]
        last_half_off = 16 * (nb - 32 * (g["gr"] - 1))
        for u, v, sg in set(producer_order(g)):
            r = g["first"] + u * g["stride"]                  # row of the concatenated matrices: the row inside its matrix has the same offsets mod 16
            nbe = min(MK_SEG * 32, nb - MK_SEG * 32 * sg)
            dbytes = (nbe * 2 + 15) & ~15
            q_off, q_len = sg * MK_SEG * 32 * bb, nbe * bb
            d_off, d_len = sg * MK_SEG * 32, dbytes // 2
            assert 0 < nbe and q_off + q_len <= nb * bb, (cta, u, sg)
            assert d_off + d_len <= d_stride(nb), (cta, u, sg, nbe, dbytes)
            for off in (r * nb * bb + q_off, q_len, 2 * (r * d_stride(nb) + d_off), dbytes):
                assert off % 16 == 0, (cta, u, sg, off)
            assert q_len <= doff and doff + dbytes <= slot_bytes
            for gi in range(MK_SEG):
                grp = sg * MK_SEG + gi
                for lane in range(32):
                    if grp * 32 + lane >= nb:
                        continue
                    reads = [gi * gb + 16 * lane]
                    if bb == 32:
                        reads.append(reads[0] + (last_half_off if grp == g["gr"] - 1 else 512))
                    assert all(a + 16 <= q_len for a in reads), (cta, u, sg, gi, lane)
                    assert 2 * (gi * 32 + lane) + 2 <= dbytes, (cta, u, sg, gi, lane)

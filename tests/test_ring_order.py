"""The ring order of mega_ring.cu, restated in Python: the producer warps enumerate a CTA's entries of a streaming MATVEC phase in one
order (mr_producer), the consumer warps claim pairs of units and walk the same entries by index arithmetic (phase_matvec_ring).  Both
sides must agree on which (unit, virtual row, segment) sits in entry e, every entry must be produced exactly once, and the two entries a
pair round touches must be adjacent.  This test pins the arithmetic (a change on one side of the CUDA file has to be mirrored here and on
the other side); the CUDA code itself is checked on the GPU by the bit-identity tests (tests/test_gpu_runner.py)."""
import itertools

import pytest

MK_SEG = 4
GRID = 132                     # one CTA per SM of an H100 SXM


def geo(m, n_mats, k, epilogue, cta, grid=GRID):
    """mr_geo: rows of the phase that belong to CTA `cta` as units (unit u -> concatenated row first + u * stride)."""
    nb = k // 32
    gr = (nb + 31) // 32
    nseg = (gr + MK_SEG - 1) // MK_SEG
    pair = epilogue == 2
    m_cat = m if pair else m * n_mats
    if epilogue == 3:
        rpc = ((m_cat + grid - 1) // grid + 3) & ~3
        first, stride = cta * rpc, 1
        n_units = min(rpc, max(0, m_cat - first))
    else:
        first, stride = cta, grid
        n_units = (m_cat - first + stride - 1) // stride if first < m_cat else 0
    v = 2 if pair else 1
    return dict(nb=nb, nseg=nseg, V=v, E=v * nseg, n_units=n_units, first=first, stride=stride)


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
]


@pytest.mark.parametrize("m,n_mats,k,epilogue", SHAPES)
def test_producer_and_consumers_agree_on_the_ring_order(m, n_mats, k, epilogue):
    covered_rows = set()
    for cta in (0, 1, 37, 146, 147):
        g = geo(m, n_mats, k, epilogue, cta)
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


@pytest.mark.parametrize("m,n_mats,k,epilogue", SHAPES)
def test_every_row_of_a_phase_belongs_to_exactly_one_cta(m, n_mats, k, epilogue):
    rows = []
    for cta in range(GRID):
        g = geo(m, n_mats, k, epilogue, cta)
        rows += [g["first"] + u * g["stride"] for u in range(g["n_units"])]
    m_cat = m if epilogue == 2 else m * n_mats
    assert sorted(rows) == list(range(m_cat))

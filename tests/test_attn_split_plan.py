"""The split plan of the persistent kernels' attention phase, restated in Python: cc_attn_split (mega.cu) picks S CTAs per head, from
AT_SPLIT_MIN_KV cached positions on phase_attn (mega_phases.cuh) uses them (below, one CTA per head), and gives CTA c of a head the positions [c L / S, (c + 1) L / S) of its L = kv_len + 1 scores, the output
dimensions [c hd / S, (c + 1) hd / S), and the Q8_0 blocks of those dimensions.  Every position must be scored once, every dimension
accumulated once and every block quantised once, whatever the head count, grid and KV length; a CTA serves one head at most, so no
CTA waits for a peer that is busy with another head.  The CUDA code itself is checked on the GPU by tests/test_gpu_attention_split.py."""
import pytest

AT_SPLIT_MAX = 4
AT_ARRIVE_WORD = 128
AT_SPLIT_MAX_HEADS = (1024 - AT_ARRIVE_WORD) // 8
AT_SPLIT_MIN_KV = 320
GRIDS = [5, 114, 132]          # a small fixed grid, an H100 PCIe, an H100 SXM


def attn_split(n_heads, hd, grid, scores=True):
    """cc_attn_split"""
    if not scores or n_heads > AT_SPLIT_MAX_HEADS:
        return 1
    for s in (4, 2):
        if hd % (32 * s) == 0 and n_heads * s <= grid:
            return s
    return 1


def effective_split(S, kv_len):
    return S if kv_len >= AT_SPLIT_MIN_KV else 1


def unit(u, n_heads):
    """unit u -> (head, part), part-major: without the split head h is on CTA h"""
    return u % n_heads, u // n_heads


def positions(c, S, kv_len):
    L = kv_len + 1
    return c * L // S, (c + 1) * L // S


def columns(c, S, hd):
    dw = hd // S
    return c * dw, (c + 1) * dw


# (head_dim, n_heads, n_kv): Llama-2-7B, Mistral-7B (GQA 32 / 8), tinyllamas stories15M, a GQA 8 / 2 model with head_dim 64, and the
# Llama-2-7B head slices of 2, 4 and 8 tensor-parallel ranks
SHAPES = {"llama2-7b": (128, 32, 32), "mistral-7b": (128, 32, 8), "tinyllamas": (48, 6, 6), "gqa-hd64": (64, 8, 2),
          "7b-rank-of-2": (128, 16, 16), "7b-rank-of-4": (128, 8, 8), "7b-rank-of-8": (128, 4, 4)}
EXPECTED = {  # grid -> S
    "llama2-7b": {5: 1, 114: 2, 132: 4}, "mistral-7b": {5: 1, 114: 2, 132: 4}, "tinyllamas": {5: 1, 114: 1, 132: 1},
    "gqa-hd64": {5: 1, 114: 2, 132: 2}, "7b-rank-of-2": {5: 1, 114: 4, 132: 4}, "7b-rank-of-4": {5: 1, 114: 4, 132: 4},
    "7b-rank-of-8": {5: 1, 114: 4, 132: 4},
}


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_split_per_shape_and_grid(shape, grid):
    hd, n_heads, _ = SHAPES[shape]
    S = attn_split(n_heads, hd, grid)
    assert S == EXPECTED[shape][grid]
    assert S == 1 or (n_heads * S <= grid and hd % (32 * S) == 0)
    assert attn_split(n_heads, hd, grid, scores=False) == 1


def test_no_split_past_the_arrival_words():
    assert attn_split(AT_SPLIT_MAX_HEADS, 128, 4 * AT_SPLIT_MAX_HEADS) == 4
    assert attn_split(AT_SPLIT_MAX_HEADS + 1, 128, 4 * AT_SPLIT_MAX_HEADS + 4) == 1
    assert AT_ARRIVE_WORD + 8 * (AT_SPLIT_MAX_HEADS - 1) < 1024        # the last head's word lies in the 4096-byte barrier block


KV_LENS = [0, 1, 2, 3, 4, 5, 31, 32, 33, 97, 319, 320, 321, 322, 323, 1000, 4095]


@pytest.mark.parametrize("grid", GRIDS)
@pytest.mark.parametrize("shape", list(SHAPES))
def test_every_position_dimension_and_block_once(shape, grid):
    hd, n_heads, _ = SHAPES[shape]
    S = attn_split(n_heads, hd, grid)
    # units u, dealt to CTAs u, u + grid, ...: with S > 1 every CTA gets at most one; every (head, part) once
    units = list(range(n_heads * S))
    per_cta = {}
    for u in units:
        per_cta.setdefault(u % grid, []).append(u)
    if S > 1:
        assert max(len(v) for v in per_cta.values()) == 1
    assert sorted(unit(u, n_heads) for u in units) == [(h, c) for h in range(n_heads) for c in range(S)]
    assert all(unit(h, n_heads) == (h, 0) for h in range(n_heads))
    for kv_len in KV_LENS:
        L = kv_len + 1
        Se = effective_split(S, kv_len)
        for h in range(n_heads):
            scored = []
            own = []
            for c in range(Se):
                lo, hi = positions(c, Se, kv_len)
                scored += list(range(lo, hi))
                if hi == L:
                    own.append(c)                      # the CTA that scores this token's own position from s_q . s_k
            assert scored == list(range(L)), (shape, grid, kv_len, h)
            assert own == [Se - 1]
    for h in range(n_heads):
        dims, blocks = [], []
        for c in range(S):
            lo, hi = columns(c, S, hd)
            dims += list(range(lo, hi))
            dw = hd // S
            blocks += [h * (hd // 32) + c * (dw // 32) + b for b in range(dw // 32)]
        assert dims == list(range(hd))
        if hd % 32 == 0:
            assert sorted(blocks) == list(range(h * (hd // 32), (h + 1) * (hd // 32)))


def test_split_only_from_the_threshold():
    assert [effective_split(4, n) for n in (0, 1, 319, 320, 321)] == [1, 1, 1, 4, 4]


@pytest.mark.parametrize("S", [2, 4])
def test_empty_ranges_when_fewer_positions_than_ctas(S):
    """phase_attn handles L < S (a CTA with nothing to score still arrives); with AT_SPLIT_MIN_KV >= S it does not happen"""
    assert AT_SPLIT_MIN_KV >= S
    for kv_len in range(S - 1):
        L = kv_len + 1
        ranges = [positions(c, S, kv_len) for c in range(S)]
        empty = [c for c, (lo, hi) in enumerate(ranges) if lo == hi]
        assert len(empty) == S - L
        assert ranges[-1][1] == L and ranges[-1][0] < L       # the last CTA always scores the own position
    # from L = S on every CTA has at least one position
    for kv_len in range(S - 1, 64):
        assert all(hi > lo for lo, hi in (positions(c, S, kv_len) for c in range(S)))


@pytest.mark.parametrize("S", [2, 4])
def test_arrival_word_rounds(S):
    """Each phase adds AT_SPLIT_MAX to a head's word whatever S (every CTA AT_SPLIT_MAX / S), so the value a CTA's add returns,
    rounded down to a multiple of AT_SPLIT_MAX, is the word at the phase's start: target = that + AT_SPLIT_MAX, across u32
    wrap-around and across tables with different S on one device."""
    word = (1 << 32) - 2 * AT_SPLIT_MAX                       # a few phases before the u32 wrap
    for phase in range(5):
        start = word
        targets = set()
        for c in range(S):                                     # any arrival order gives the same target
            old = word
            word = (word + AT_SPLIT_MAX // S) % (1 << 32)
            targets.add(((old & ~(AT_SPLIT_MAX - 1)) + AT_SPLIT_MAX) % (1 << 32))
        assert targets == {(start + AT_SPLIT_MAX) % (1 << 32)} and word == (start + AT_SPLIT_MAX) % (1 << 32)

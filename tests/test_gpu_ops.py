"""Parity of the small ops (SURVEY §8a a12-a19) through the C ABI vs the CPU oracle.
Structure follows the reference's per-backend op tests (crabml-wgpu/src/wgpu_tensor.rs:749-1099)."""
import numpy as np
import pytest

from oracle import oracle as oc
from oracle.tensor_ref import OracleDevice, OracleTensor
from tests.blockgen import random_weight
from tests.gpu_common import both, make_device

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def gdev():
    d = make_device()
    yield d
    d.close()


@pytest.fixture(scope="module")
def odev():
    return OracleDevice()


def test_alloc_export_dup(gdev, odev):
    from crabml_b200 import CudaTensor, TensorError
    t = CudaTensor.alloc([3, 4], oc.F32, gdev)
    assert t.export().tolist() == [0.0] * 12           # zero-filled, cpu_tensor.rs:147
    with pytest.raises(TensorError):
        CudaTensor.alloc([4], oc.Q8_0, gdev)           # only f32/f16
    g, o = both(np.arange(24), [2, 3, 4], gdev, odev)
    d = g.dup()
    assert d.shape() == [2, 3, 4] and d.export().tolist() == o.dup().export().tolist()
    g.scale_inplace(2.0)
    assert d.export().tolist() == list(range(24))      # dup owns its storage


def test_copy_rows_and_view_kats(gdev, odev):
    # cpu_tensor.rs:455-482
    from crabml_b200 import CudaTensor
    t = CudaTensor.new([1, 2, 3, 4, 5, 6], [2, 3], gdev).reshape([3, 2]).reshape([2, 3])
    assert t.to_vec().tolist() == [1, 2, 3, 4, 5, 6]
    t1 = CudaTensor.new([1, 2, 3, 4], [2, 2], gdev)
    t2 = CudaTensor.new([0, 0], [2], gdev)
    t2.copy_rows_from(t1, [1]); assert t2.to_vec().tolist() == [3, 4]
    t2.copy_rows_from(t1, [0]); assert t2.to_vec().tolist() == [1, 2]


def test_rope_kat(gdev):
    # cpu_tensor.rs:509-527
    from crabml_b200 import CudaTensor
    t = CudaTensor.new(np.arange(32), [2, 16], gdev).rope_inplace(0, 1, 2)
    want = [-0.841471, 0.54030234] + [float(v) for v in range(2, 16)] + [-5.6601696, 22.648676] + [float(v) for v in range(18, 32)]
    np.testing.assert_allclose(t.to_vec(), want, atol=1e-5)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("shape,pos,rope_dim", [([1, 6, 48], 0, 48), ([1, 32, 128], 77, 128), ([3, 8, 64], 1000, 32), ([4, 128], 4095, 128)])
def test_rope_vs_oracle(gdev, odev, mode, shape, pos, rope_dim):
    rng = np.random.default_rng(5)
    g, o = both(rng.standard_normal(int(np.prod(shape))), shape, gdev, odev)
    # cosf/sinf differ from glibc by <= 2 ulp: tolerance 1e-5 abs like the reference KAT
    # cos/sin come from the host libm (same calls as the reference): bit-exact
    np.testing.assert_array_equal(g.rope_inplace(mode, pos, rope_dim).export().view(np.uint32), o.rope_inplace(mode, pos, rope_dim).export().view(np.uint32))


def test_matmul_f32_kats(gdev):
    # cpu_tensor.rs:530-541 and wgpu_tensor.rs:880-895 (exact)
    from crabml_b200 import CudaTensor
    w = CudaTensor.new([4.0] * 32, [16, 2], gdev)
    assert w.matmul_vec(CudaTensor.new([1.0, 2.0], [2], gdev)).to_vec().tolist() == [12.0] * 16
    w = CudaTensor.new(np.arange(256), [32, 8], gdev)
    out = w.matmul_vec(CudaTensor.new([2.0] * 8, [8], gdev)).to_vec()
    assert out.tolist() == [float(sum(range(8 * r, 8 * r + 8)) * 2) for r in range(32)]


def test_softmax_silu_kats(gdev):
    # cpu_tensor.rs:544-569
    from crabml_b200 import CudaTensor, TensorError
    t = CudaTensor.new([1, 2, 3, 4, 5, 6], [2, 3], gdev).softmax_inplace(1)
    np.testing.assert_allclose(t.to_vec(), [0.09003057, 0.24472848, 0.66524094] * 2, atol=1e-3)
    with pytest.raises(TensorError):
        CudaTensor.new([1, 2, 3, 4, 5, 6], [2, 3], gdev).softmax_inplace(0)
    t = CudaTensor.new([1, 2, 3, 4, 5, 6], [6], gdev).silu_inplace()
    np.testing.assert_allclose(t.to_vec(), [0.7310586, 1.761594, 2.8577225, 3.928055, 4.9665356, 5.9851646], rtol=2e-3)


@pytest.mark.parametrize("shape", [[32, 1, 1], [6, 1, 37], [32, 1, 257], [4, 3, 2048], [8, 100], [3, 1, 4097]])
def test_softmax_vs_oracle(gdev, odev, shape):
    rng = np.random.default_rng(6)
    g, o = both(rng.standard_normal(int(np.prod(shape))) * 4, shape, gdev, odev)
    ax = len(shape) - 1
    # identical LUT exps; only the order of the f32 sum differs (tree vs sequential)
    np.testing.assert_allclose(g.softmax_inplace(ax).export(), o.softmax_inplace(ax).export(), rtol=5e-6, atol=0)


def test_softmax_long_rows_vs_f64_and_oracle(gdev, odev):
    """Rows of 40 001.  The exps are the same LUT values on both sides, so the f32 sum alone differs.  The oracle sums sequentially (the
    reference's order, softmax.rs:39-54), which drifts by about 5e-5 relative at this length; the kernel's 512-thread tree stays within
    5e-6 of the f64 sum of the same exps.  So the kernel is held to 5e-6 of that f64 normalisation, and to the oracle within 5e-6 plus the
    oracle's own distance from it."""
    rng = np.random.default_rng(6)
    x = (rng.standard_normal(2 * 40001) * 4).astype(np.float32)
    g, o = both(x, [2, 40001], gdev, odev)
    got, want_o = g.softmax_inplace(1).export().reshape(2, -1), o.softmax_inplace(1).export().reshape(2, -1)
    rows = x.reshape(2, -1)
    e = oc.f16_to_f32(oc.exp_lut()[oc.f32_to_f16(rows - rows.max(axis=1, keepdims=True)).astype(np.int64)]).astype(np.float64)
    want = e / e.sum(axis=1, keepdims=True)
    np.testing.assert_allclose(got, want, rtol=5e-6, atol=0)
    drift = float(np.abs(want_o / np.where(want > 0, want, 1) - 1)[want > 0].max())
    np.testing.assert_allclose(got, want_o, rtol=5e-6 + drift, atol=0)


def test_silu_gelu_bit_exact(gdev, odev):
    rng = np.random.default_rng(7)
    v = np.concatenate([rng.standard_normal(11008) * 5, [0.0, -0.0, 100.0, -100.0, 1e-8, 65504.0, -65504.0, 7e4]]).astype(np.float32)
    g, o = both(v, [v.size], gdev, odev)
    np.testing.assert_array_equal(g.silu_inplace().export().view(np.uint32), o.silu_inplace().export().view(np.uint32))
    g, o = both(v, [v.size], gdev, odev)
    np.testing.assert_array_equal(g.gelu_inplace().export().view(np.uint32), o.gelu_inplace().export().view(np.uint32))


def test_rms_norm_kat_and_oracle(gdev, odev):
    # wgpu_tensor.rs:852-877: 1..128 eps 1e-5 ; rms_norm.rs:34 requires len % 32 == 0
    from crabml_b200 import CudaTensor, TensorError
    v = np.arange(1, 129, dtype=np.float32)
    g, o = both(v, [128], gdev, odev)
    np.testing.assert_allclose(g.rms_norm_inplace(1e-5).export(), o.rms_norm_inplace(1e-5).export(), rtol=3e-7)
    rng = np.random.default_rng(8)
    for shape in ([4096], [3, 288], [2, 11008]):
        g, o = both(rng.standard_normal(int(np.prod(shape))), shape, gdev, odev)
        np.testing.assert_allclose(g.rms_norm_inplace(1e-6).export(), o.rms_norm_inplace(1e-6).export(), rtol=1e-6)
    with pytest.raises(TensorError):
        CudaTensor.new(np.zeros(48), [48], gdev).rms_norm_inplace(1e-5)


def test_add_mul_scale_bit_exact(gdev, odev):
    rng = np.random.default_rng(9)
    a = rng.standard_normal(3 * 288)
    b = rng.standard_normal(288)
    for op in ("add_inplace", "mul_inplace"):
        g, o = both(a, [3, 288], gdev, odev)
        gb, ob = both(b, [288], gdev, odev)
        np.testing.assert_array_equal(getattr(g, op)(gb).export(), getattr(o, op)(ob).export())
        g, o = both(a, [3, 288], gdev, odev)
        gb, ob = both(a[::-1].copy(), [3, 288], gdev, odev)
        np.testing.assert_array_equal(getattr(g, op)(gb).export(), getattr(o, op)(ob).export())
    g, o = both(a, [3, 288], gdev, odev)
    s = float(np.float32(1.0) / np.sqrt(np.float32(48)))
    np.testing.assert_array_equal(g.scale_inplace(s).export(), o.scale_inplace(s).export())


def test_contiguous_kats(gdev):
    # cpu_tensor.rs:572-600
    from crabml_b200 import CudaTensor
    t2 = CudaTensor.new([1, 2, 3, 4, 5, 6], [2, 3], gdev).transpose([1, 0]).contiguous()
    assert t2.to_vec().tolist() == [1, 4, 2, 5, 3, 6] and t2.shape() == [3, 2]
    t1 = CudaTensor.new([1, 2, 3, 4, 5, 6], [1, 2, 3], gdev).transpose([2, 1, 0])
    t2 = t1.contiguous()
    assert t2.to_vec().tolist() == [1, 4, 2, 5, 3, 6] and t2.shape() == [3, 2, 1]
    q = CudaTensor.new(np.arange(32 * 128), [1, 32, 128], gdev).transpose([1, 0, 2])
    assert not q.is_contiguous()
    assert q.contiguous().export().tolist() == list(map(float, range(32 * 128)))


@pytest.mark.parametrize("kv_dtype", [oc.F32, oc.F16])
def test_concatenate_kv_cache(gdev, odev, kv_dtype):
    # llama2.rs:65-86,542-554: cache [n_kv, seq_max, hd] resized to 0 then grown along axis 1
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(10)
    n_kv, seq_max, hd = 4, 9, 16
    gc = CudaTensor.alloc([n_kv, seq_max, hd], kv_dtype, gdev).resize(1, 0)
    ocache = OracleTensor.alloc([n_kv, seq_max, hd], kv_dtype, odev).resize(1, 0)
    for pos in range(5):
        k = rng.standard_normal(n_kv * hd)
        gk, ok = both(k, [1, n_kv, hd], gdev, odev)
        gc.concatenate(gk.transpose([1, 0, 2]), 1)
        ocache.concatenate(ok.transpose([1, 0, 2]), 1)
        assert gc.shape() == ocache.shape() == [n_kv, pos + 1, hd]
        assert gc.strider().strides == ocache.strider().strides == [seq_max * hd, hd, 1]
    # read back through batch_matmul with an identity-like probe (F16 caches cannot be exported directly)
    q = rng.standard_normal(n_kv * hd)
    gq, oq = both(q, [n_kv, 1, hd], gdev, odev)
    ga = gq.batch_matmul(gc.transpose([0, 2, 1])).export()
    oa = oq.batch_matmul(ocache.transpose([0, 2, 1])).export()
    np.testing.assert_allclose(ga, oa, rtol=2e-6, atol=1e-6)
    from crabml_b200 import TensorError
    with pytest.raises(TensorError):           # past the pre-allocated length
        for _ in range(6):
            gc.concatenate(CudaTensor.new(np.zeros(n_kv * hd), [1, n_kv, hd], gdev).transpose([1, 0, 2]), 1)


@pytest.mark.parametrize("kv_dtype", [oc.F32, oc.F16])
@pytest.mark.parametrize("heads,kv_heads,hd,seq", [(6, 6, 48, 1), (6, 6, 48, 17), (32, 32, 128, 100), (8, 4, 16, 33), (32, 8, 128, 64),
                                                    (32, 32, 128, 1000), (32, 8, 128, 1000), (32, 32, 128, 4096), (32, 8, 128, 4096)])
def test_batch_matmul_attention_shapes(gdev, odev, kv_dtype, heads, kv_heads, hd, seq):
    """QK^T (B = K cache transposed, stride_k == 1) and PV (B = V cache, stride_n == 1), incl. the
    GQA head mapping: bi % bb for F32 caches (batch_matmul.rs:63), bi / (ab/bb) for F16 (:89-91)."""
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(11)
    seq_max = seq + 3
    gk = CudaTensor.alloc([kv_heads, seq_max, hd], kv_dtype, gdev).resize(1, 0)
    ok = OracleTensor.alloc([kv_heads, seq_max, hd], kv_dtype, odev).resize(1, 0)
    rows = rng.standard_normal((seq, kv_heads, hd)).astype(np.float32)
    g_all, o_all = both(rows, [seq, kv_heads, hd], gdev, odev)
    gk.concatenate(g_all.transpose([1, 0, 2]), 1)
    ok.concatenate(o_all.transpose([1, 0, 2]), 1)
    q = rng.standard_normal(heads * hd)
    gq, oq = both(q, [heads, 1, hd], gdev, odev)
    g_att = gq.batch_matmul(gk.transpose([0, 2, 1]))
    o_att = oq.batch_matmul(ok.transpose([0, 2, 1]))
    assert g_att.shape() == [heads, 1, seq]
    # f32 summation-order noise, budgeted against sum |q_i k_i| per output
    kk = rows.transpose(1, 0, 2)                                  # [kv, seq, hd]
    grp = (np.arange(heads) % kv_heads) if kv_dtype == oc.F32 else (np.arange(heads) // (heads // kv_heads))
    budget = np.einsum("hd,hsd->hs", np.abs(q.reshape(heads, hd)), np.abs(kk[grp])) * 1e-6 + 1e-7
    assert (np.abs(g_att.export() - o_att.export()).reshape(heads, seq) <= budget).all()
    # PV with identical attention weights on both sides
    w = np.abs(rng.standard_normal(heads * seq)).astype(np.float32)
    gw, ow = both(w, [heads, 1, seq], gdev, odev)
    g_out = gw.batch_matmul(gk).export()
    o_out = ow.batch_matmul(ok).export()
    np.testing.assert_array_equal(g_out.view(np.uint32), o_out.view(np.uint32))   # same sequential order -> bit exact


@pytest.mark.parametrize("t", oc.QUANT_TYPES)
def test_block_unpack_bit_exact(gdev, odev, t):
    """north_star: 'block unpack bit-exact'.  copy_rows_from dequantises rows of the repacked device
    layout; must equal BlockQ*::dequantize bit for bit, and the repack must round-trip the GGUF bytes."""
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(100 + t)
    rows, cols = 7, 512
    raw = random_weight(t, rows, cols, rng)
    gw = CudaTensor.from_cpu(raw, [rows, cols], t, gdev)
    ow = OracleTensor.from_cpu(raw, [rows, cols], t, odev)
    pick = [6, 0, 3, 3]
    g = CudaTensor.alloc([len(pick), cols], oc.F32, gdev); g.copy_rows_from(gw, pick)
    o = OracleTensor.alloc([len(pick), cols], oc.F32, odev); o.copy_rows_from(ow, pick)
    np.testing.assert_array_equal(g.export().view(np.uint32), o.export().view(np.uint32))
    back = gw.export_blocks(raw.size)
    if t == oc.Q8_K:            # bsums of a Q8_K *weight* are not kept on device (activation-only field)
        back.reshape(-1, 292)[:, 260:] = raw.reshape(-1, 292)[:, 260:]
    np.testing.assert_array_equal(back, raw)


def test_embedding_row_f16_dst(gdev, odev):
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(12)
    raw = random_weight(oc.Q8_0, 5, 64, rng)
    gw = CudaTensor.from_cpu(raw, [5, 64], oc.Q8_0, gdev)
    g = CudaTensor.alloc([2, 64], oc.F32, gdev); g.copy_rows_from(gw, [4, 1])
    want = oc.dequantize(oc.Q8_0, raw, 5 * 64).reshape(5, 64)[[4, 1]].reshape(-1)
    np.testing.assert_array_equal(g.export(), want)


@pytest.mark.parametrize("act", [oc.Q8_0, oc.Q8_1, oc.Q8_K])
def test_activation_quantize_bit_exact(gdev, act):
    """a3-a5: truncating Q8_0/Q8_1 (B1/B2), half-away Q8_K (B3): the activation blocks must be
    byte-identical to the reference arithmetic, including zero blocks and sign/tie edge cases."""
    from crabml_b200 import CudaTensor
    rng = np.random.default_rng(13)
    n = 256 * 12
    x = (rng.standard_normal(n) * rng.choice([1e-3, 1.0, 30.0], n)).astype(np.float32)
    x[0:256] = 0.0                                  # zero (super-)block
    x[256:512] = np.tile(np.arange(-8, 8, dtype=np.float32), 16)     # reference quantize KAT ramp
    x[512] = -5.0; x[513] = 5.0                     # |max| tie: first occurrence wins (Q8_K sign of scale)
    x[512 + 2:768] = 0.25
    x[768:800] = 127.0
    x[800:832] = [(-1) ** i * (i + 0.5) for i in range(32)]          # .5 values: trunc vs round visible
    gx = CudaTensor.new(x, [n], gdev)
    want = oc.quantize(act, x)
    got = gx.quantize_activation(act, want.size)
    if act == oc.Q8_1:       # zero block: reference gives qs=-128 with d=0 (B2); compare everything
        pass
    np.testing.assert_array_equal(got, want)

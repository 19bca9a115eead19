"""GPU parity of the wgmma tensor-core GEMM (M > 4) against the oracle.

The kernel's arithmetic is bf16 x bf16 -> fp32: w_eff = bf16((q - zp) * bf16(scale)), a_eff = bf16(a).  Checks:
 (1) against an fp64-accumulated GEMM on exactly those operands: rtol 2e-3 (fp32 accumulation order only);
 (2) the reference's CompBf16 UT tolerance (2e-2 abs at K=4096 with U[-0.5,0.5] data, bestla_ut.h:80-94) vs fp32 GEMM on the
     dequantised weights;
 (3) the north-star bar: <= 1e-2 relative (to the logits' range) vs the CPU path's numerics (Q8_0 / u8 activations)."""
import ctypes as C

import numpy as np
import pytest

import oracle
import neural_speed_b200 as ns

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def bf16r(x):
    return oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(np.asarray(x, np.float32)))


def run(w, a, bias=None, residual=None, flags=None):
    m, k = a.shape
    if flags is None:  # this file tests the tensor-core kernel: M <= 16 would take the exact-integer GEMV tiles by default
        flags = ns.MM_FORCE_TC
    ad = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    out = torch.full((m, w.n), float("nan"), device="cuda")
    b = torch.from_numpy(bias).cuda() if bias is not None else None
    r = torch.from_numpy(residual).cuda() if residual is not None else None
    torch.cuda.synchronize()
    ns.mul_mat(w, ad.data_ptr(), k, out.data_ptr(), w.n, m, b.data_ptr() if b is not None else None,
               r.data_ptr() if r is not None else None, flags)
    torch.cuda.synchronize()
    ns.lib().bestla_device_sync(None)
    return out.cpu().numpy()


def expect_bf16(a, q, sc, zp, g):
    k = q.shape[0]
    gi = np.arange(k) // g
    qq = q.astype(np.float32) - (zp[gi].astype(np.float32) if zp is not None else 0.0)
    w_eff = bf16r(qq * bf16r(sc)[gi])
    return oracle.gemm_f64acc(bf16r(a), w_eff)


@pytest.mark.parametrize("m,n,k,g,asym", [(5, 128, 64, 32, False), (8, 128, 256, 128, False), (32, 256, 512, 32, True),
                                          (100, 300, 1024, 128, True), (64, 4096, 4096, 128, False),
                                          (300, 512, 11008, 128, False), (2048, 256, 4096, 32, False), (33, 136, 1056, 32, False)])
def test_tc_gemm_int4_vs_oracle(m, n, k, g, asym):
    rng = np.random.default_rng(m * 7 + n)
    w = rng.uniform(-0.5, 0.5, (k, n)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    q, sc, zp = oracle.btla_quantize(w, g, 4, asym)
    wd = ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S4, ns.S_F32, ns.COMP_INT8)
    got = run(wd, a)
    assert np.isfinite(got).all()
    want = expect_bf16(a, q, sc, zp, g)
    scale = np.abs(want).max()
    assert np.abs(got - want).max() <= 2e-3 * scale
    ref32 = oracle.gemm_f64acc(a, oracle.btla_dequant(q, sc, zp, g))
    # vs fp32 GEMM on the dequantised weights: bf16 operand rounding only (the reference's CompBf16 UT allows 2e-2 abs on
    # outputs of magnitude ~10 at K=4096, bestla_ut.h:80-94); north-star logits bar = 1e-2 of the output range
    assert np.abs(got - ref32).max() <= 1e-2 * np.abs(ref32).max()


@pytest.mark.parametrize("m,n,k,g", [(9, 128, 256, 32), (130, 384, 1024, 128), (300, 512, 4096, 32)])
def test_tc_gemm_nf4_vs_oracle(m, n, k, g):
    """config 4 (NF4): level = table[code] (kernel_ref.h:1325-1368), bf16 operands on the tensor cores"""
    rng = np.random.default_rng(m + n)
    w = rng.uniform(-0.5, 0.5, (k, n)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    q, sc = oracle.btla_quantize_nf4(w, g)
    wd = ns.Weight.from_unpacked(q, sc, None, g, ns.W_NF4, ns.S_F32, ns.COMP_BF16)
    got = run(wd, a)
    wdq = oracle.btla_dequant(q, sc, None, g, nf4=True)
    gi = np.arange(k) // g
    lut = wdq / np.where(sc[gi] == 0, 1, sc[gi])                    # the table levels
    want = oracle.gemm_f64acc(bf16r(a), bf16r(bf16r(lut) * bf16r(sc)[gi]))
    assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max()
    ref32 = oracle.gemm_f64acc(a, wdq)
    assert np.abs(got - ref32).max() <= 1e-2 * np.abs(ref32).max()


@pytest.mark.parametrize("m,n,k,g,asym", [(9, 128, 256, 32, False), (130, 384, 1024, 128, True), (300, 512, 4096, 32, False)])
def test_tc_gemm_int8_weights_vs_oracle(m, n, k, g, asym):
    """config 4 (INT8 weights): 64 packed bytes per row and k block, (q - zp) exact in bf16"""
    rng = np.random.default_rng(m + n + 1)
    w = rng.uniform(-0.5, 0.5, (k, n)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    q, sc, zp = oracle.btla_quantize(w, g, 8, asym)
    wd = ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S8, ns.S_F32, ns.COMP_BF16)
    got = run(wd, a)
    want = expect_bf16(a, q, sc, zp, g)
    assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max()
    ref32 = oracle.gemm_f64acc(a, oracle.btla_dequant(q, sc, zp, g))
    assert np.abs(got - ref32).max() <= 1e-2 * np.abs(ref32).max()


def test_tc_gemm_q4_0_prefill_vs_cpu_path():
    """ggml Q4_0 weights, 128-token prompt batch: tensor-core result vs the reference CPU numerics (Q8_0 activations)"""
    rng = np.random.default_rng(3)
    m, n, k = 128, 512, 4096
    w = rng.normal(0, 0.02, (n, k)).astype(np.float32)
    a = rng.normal(0, 1.0, (m, k)).astype(np.float32)
    rows = oracle.quantize_q4_0(w)
    wd = ns.Weight.from_q4_0_host(rows, n, k)
    got = run(wd, a)
    cpu = oracle.mul_mat_q4_0_f32(rows, a)
    assert np.abs(got - cpu).max() <= 1e-2 * np.abs(cpu).max()
    # exact-operand check: fp16 scales rounded to bf16 by the kernel
    wdq = oracle.dequantize_q4_0(rows, k)  # (nib-8)*d with d fp16
    blocks = rows.reshape(n, k // 32, 18)
    d = np.array([[oracle.lib().orc_fp16_to_fp32(int(b[0]) | int(b[1]) << 8) for b in r] for r in blocks], np.float32)
    qv = np.round(wdq.reshape(n, k // 32, 32) / np.where(d == 0, 1, d)[:, :, None]).astype(np.float32)
    w_eff = bf16r(qv * bf16r(d)[:, :, None]).reshape(n, k)
    want = oracle.gemm_f64acc(bf16r(a), np.ascontiguousarray(w_eff.T))
    assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max()
    # the exact-integer GEMV path can be forced for any M and must agree with the CPU path tightly
    got_gemv = run(wd, a[:9], flags=ns.MM_FORCE_GEMV)
    np.testing.assert_allclose(got_gemv, cpu[:9], rtol=1e-4, atol=1e-4 * np.abs(cpu).max())


def test_tc_gemm_bias_residual_and_small_m_forced():
    rng = np.random.default_rng(5)
    m, n, k, g = 3, 256, 512, 128
    w = rng.uniform(-0.5, 0.5, (k, n)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    bias = rng.normal(0, 1, (n,)).astype(np.float32)
    res = rng.normal(0, 1, (m, n)).astype(np.float32)
    q, sc, zp = oracle.btla_quantize(w, g, 4, False)
    wd = ns.Weight.from_unpacked(q, sc, None, g, ns.W_S4, ns.S_F32, ns.COMP_INT8)
    got = run(wd, a, bias=bias, residual=res, flags=ns.MM_FORCE_TC | ns.MM_BIAS_BCAST)
    want = expect_bf16(a, q, sc, None, g) + bias[None, :] + res
    assert np.abs(got - want).max() <= 2e-3 * np.abs(want).max()


def test_fused_drop_ins_batched():
    """QKV and FFN host drop-ins at a prompt batch go through the tensor-core path"""
    rng = np.random.default_rng(9)
    m, k, n, fmid, g = 48, 512, 256, 1024, 128
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    ws = {}
    def mk(name, r, c):
        wt = rng.uniform(-0.5, 0.5, (r, c)).astype(np.float32)
        ws[name] = wt
        return ns.np_bestla_quantize(wt, "int4", g, "sym", "fp32", "int8")
    bq, bk, bv = mk("q", n, k), mk("k", n, k), mk("v", n, k)
    L = ns.lib()
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    out = np.zeros((3, m, n), np.float32)
    L.bestla_fusion_QKV_f32f32_forward(p(a), p(bq), p(bk), p(bv), p(out), m, n, k, k, n, None)
    for i, b in enumerate((bq, bk, bv)):
        wdq = ns.unpack_blob(b, n, k)
        ref = oracle.gemm_f64acc(a, wdq)
        assert np.abs(out[i] - ref).max() <= 1e-2 * np.abs(ref).max()
    b1, b3, b2 = mk("w1", fmid, k), mk("w3", fmid, k), mk("w2", n, fmid)
    ffn = np.zeros((m, n), np.float32)
    tmp2 = np.zeros((m, fmid), np.float32)
    L.bestla_fusion_FFN_SiLu_f32f32_forward(p(a), p(b1), p(b2), p(b3), None, p(tmp2), p(ffn), m, k, fmid, n, None)
    g1 = oracle.gemm_f64acc(a, ns.unpack_blob(b1, fmid, k))
    u1 = oracle.gemm_f64acc(a, ns.unpack_blob(b3, fmid, k))
    h = (g1 / (1 + np.exp(-g1))) * u1
    assert np.abs(tmp2 - h).max() <= 1e-2 * np.abs(h).max()
    ref = oracle.gemm_f64acc(h.astype(np.float32), ns.unpack_blob(b2, n, fmid))
    assert np.abs(ffn - ref).max() <= 2e-2 * np.abs(ref).max()

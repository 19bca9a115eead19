"""GPU tests of 2/3/5/6/7-bit BesTLA blobs (S2_CLIP .. S7_CLIP): the device load keeps every integer (dequantised image ==
BTLAGemmUnPackB bit for bit), and the matmul through the ne_bestla.h host drop-in matches the oracle's u8 x s8 block arithmetic
(kernel_ref.h:1825 activation quantiser, :2372 integer block dots; bestla_wrapper.h:348-353 routes these dtypes to that GEMV)."""
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
    ns.lib().ns_host_cache_clear()


def close(got, want, rtol=1e-4):
    scale = float(np.abs(want).max()) + 1e-30
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * scale)


@pytest.mark.parametrize("bits", [2, 3, 5, 6, 7])
@pytest.mark.parametrize("alg,m", [("sym", 1), ("asym", 3), ("sym", 40)])
def test_lowbit_blob_load_and_forward(bits, alg, m):
    rng = np.random.default_rng(100 * bits + m)
    n, k, g = 200, 1024, 128
    wt = rng.uniform(-0.5, 0.5, (n, k)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    blob = ns.np_bestla_quantize(wt, f"int{bits}", g, alg, "fp32", "int8")
    wdq = ns.unpack_blob(blob, n, k)
    w = ns.Weight.from_blob(blob)
    dq = torch.zeros((n, k), dtype=torch.float32, device="cuda")
    assert ns.lib().ns_weight_dequant_f32(w.h, C.c_void_p(dq.data_ptr()), k, None) == 0
    torch.cuda.synchronize()
    ns.lib().bestla_device_sync(None)
    assert np.array_equal(dq.cpu().numpy(), wdq.T)  # the device image holds exactly the reference's integers
    out = np.full((m, n), np.nan, np.float32)
    ns.lib().bestla_f32f32_forward(a.ctypes.data_as(C.c_void_p), blob.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), m, n,
                                   k, k, n, None)
    q, sc, zp = oracle.btla_quantize(np.ascontiguousarray(wt.T), g, bits, alg == "asym")
    a8, asc, azp = oracle.btla_quantize_act_u8(a, g)
    want = oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, g)
    if m <= 32:
        close(out, want)  # exact integer block sums (GEMV / integer tensor cores)
    else:
        # > 32 rows: bf16 tensor-core GEMM on the dequantised weight (north-star bar against the fp32 product)
        close(out, oracle.gemm_f64acc(a, wdq), 1e-2)


@pytest.mark.parametrize("name", ["fp4_bnb", "fp4_e2m1", "nf4"])
@pytest.mark.parametrize("cdt,m", [("fp32", 1), ("bf16", 3), ("bf16", 40)])
def test_f4_codebook_blobs(name, cdt, m):
    """F4_BNB / F4_E2M1 / F4_NF4 blobs: the device image dequantises to exactly BTLAGemmUnPackB's values (code -> level table
    chosen per weight), and the matmul meets the reference's UT criterion for float compute types (<= 1e-3 abs against the fp32
    product on the dequantised weight for fp32 compute, bf16 rounding of both operands for bf16 compute)."""
    rng = np.random.default_rng(7 + m)
    n, k, g = 200, 1024, 32
    wt = rng.uniform(-0.5, 0.5, (n, k)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    blob = ns.np_bestla_quantize(wt, name, g, "sym", "fp32", cdt)
    wdq = ns.unpack_blob(blob, n, k)
    w = ns.Weight.from_blob(blob)
    dq = torch.zeros((n, k), dtype=torch.float32, device="cuda")
    assert ns.lib().ns_weight_dequant_f32(w.h, C.c_void_p(dq.data_ptr()), k, None) == 0
    torch.cuda.synchronize()
    ns.lib().bestla_device_sync(None)
    assert np.array_equal(dq.cpu().numpy(), wdq.T)
    out = np.full((m, n), np.nan, np.float32)
    ns.lib().bestla_f32f32_forward(a.ctypes.data_as(C.c_void_p), blob.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), m, n,
                                   k, k, n, None)
    a_eff = a if cdt == "fp32" else oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(a))
    want = oracle.gemm_f64acc(a_eff, wdq)
    # fp32 compute: the reference UT bar; bf16 compute: bf16 rounding of the dequantised weight too (GEMV keeps it in fp32, the tensor-core
    # GEMM for > 16 rows rounds level x scale to bf16 as the reference does)
    assert np.abs(out - want).max() <= (1e-3 if cdt == "fp32" else 2e-2 if m <= 16 else 4e-2)
    if m <= 16:  # the GEMV's stated arithmetic: bf16 (or fp32) activations, the dequantised weight in fp32, fp32 FMAs
        assert oracle.gemv_bound_ratio(out, a_eff, wdq) <= oracle.GEMV_F32_C

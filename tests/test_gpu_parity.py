"""GPU parity tests (run on an H100): the CUDA path, called through the C-ABI, against the CPU oracle on the same
seeded inputs, and against the golden fixtures generated from the reference.

Bars:  integer / byte outputs (quantisers, repack, block sums) -- bit exact.
       fp32 matmul outputs in an integer-activation mode        -- rtol 1e-4 (only the fp32 summation ORDER differs
                                                                   from the reference; every block dot is an exact int).
       fp32 / bf16 compute modes                                 -- the reference's own UT criterion: <= 1e-3 abs vs
                                                                   fp32 GEMM on the dequantised weights (ut_int, bestla_prologue_b.cpp:471-511).
"""
import ctypes as C
import os

import numpy as np
import pytest

import oracle
import neural_speed_b200 as ns

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def sync():
    torch.cuda.synchronize()
    ns.lib().bestla_device_sync(None)


def run_mul_mat(w, a_np, bias=None, residual=None, flags=0):
    a = dev(a_np.astype(np.float32))
    m, k = a_np.shape
    out = torch.full((m, w.n), float("nan"), device="cuda", dtype=torch.float32)
    b = dev(bias) if bias is not None else None
    r = dev(residual) if residual is not None else None
    torch.cuda.synchronize()
    ns.mul_mat(w, a.data_ptr(), k, out.data_ptr(), w.n, m, b.data_ptr() if b is not None else None,
               r.data_ptr() if r is not None else None, flags)
    sync()
    return out.cpu().numpy()


def close(got, want, rtol=1e-4):
    scale = float(np.abs(want).max()) + 1e-30
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * scale)


# ------------------------------------------------------------------------------------------------------- quantisers
def test_device_q4_0_quantiser_bit_exact():
    rng = np.random.default_rng(1)
    w = rng.normal(0, 0.02, (96, 1024)).astype(np.float32)
    w[5, 64:96] = 0
    w[6] *= 1000
    src = dev(w)
    dst = torch.zeros(96 * 1024 // 32 * 18, dtype=torch.uint8, device="cuda")
    assert ns.lib().ns_device_quantize_q4_0(C.c_void_p(src.data_ptr()), C.c_void_p(dst.data_ptr()), 96, 1024, None) == 0
    sync()
    assert np.array_equal(dst.cpu().numpy().reshape(96, -1), oracle.quantize_q4_0(w))


@pytest.mark.parametrize("comp,g", [(ns.COMP_Q8_0, 32), (ns.COMP_INT8, 32), (ns.COMP_INT8, 128), (ns.COMP_INT8_S8, 128),
                                    (ns.COMP_INT8, 300)])
def test_device_activation_quantiser_bit_exact(comp, g):
    rng = np.random.default_rng(2)
    m, k = 5, 1280 if g != 300 else 1500
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    a[1] = np.abs(a[1])
    a[2, :g] = 0
    a[3, :64] = np.round(a[3, :64] * 8) / 8
    ad = dev(a)
    ng = -(-k // g)
    q = torch.zeros((m, k), dtype=torch.uint8, device="cuda")
    sc = torch.zeros((m, ng), dtype=torch.float32, device="cuda")
    zp = torch.zeros((m, ng), dtype=torch.int32, device="cuda")
    assert ns.lib().ns_device_quantize_act(C.c_void_p(ad.data_ptr()), k, m, k, g, comp, C.c_void_p(q.data_ptr()),
                                           C.c_void_p(sc.data_ptr()), C.c_void_p(zp.data_ptr()), None) == 0
    sync()
    qh, sh, zh = q.cpu().numpy(), sc.cpu().numpy(), zp.cpu().numpy()
    if comp == ns.COMP_Q8_0:
        blocks = oracle.quantize_q8_0(a).reshape(m, k // 32, 34)
        want_q = blocks[:, :, 2:].reshape(m, k)
        want_d = np.array([[oracle.lib().orc_fp16_to_fp32(int(b[0]) | int(b[1]) << 8) for b in row] for row in blocks], np.float32)
        assert np.array_equal(qh, want_q) and np.array_equal(sh, want_d)
    elif comp == ns.COMP_INT8:
        wq, ws, wz = oracle.btla_quantize_act_u8(a, g)
        assert np.array_equal(qh, wq) and np.array_equal(sh, ws) and np.array_equal(zh, wz.astype(np.int32))
    else:
        wq, ws = oracle.btla_quantize_act_s8(a, g)
        assert np.array_equal(qh.view(np.int8), wq) and np.array_equal(sh, ws)


# ------------------------------------------------------------------------------------------------------- ggml Q4_0
def _dequant_dev(w):
    out = torch.zeros((w.n, w.k), dtype=torch.float32, device="cuda")
    assert ns.lib().ns_weight_dequant_f32(w.h, C.c_void_p(out.data_ptr()), w.k, None) == 0
    sync()
    return out.cpu().numpy()


def test_q4_0_repack_is_lossless():
    rng = np.random.default_rng(3)
    n, k = 130, 768
    rows = oracle.quantize_q4_0(rng.normal(0, 0.02, (n, k)).astype(np.float32))
    w = ns.Weight.from_q4_0_host(rows, n, k)
    assert np.array_equal(_dequant_dev(w), oracle.dequantize_q4_0(rows, k))


@pytest.mark.parametrize("n,k,m", [(64, 512, 1), (4096, 4096, 1), (1000, 11008, 1), (257, 1024, 3), (96, 4096, 4), (128, 2048, 7),
                                   (600, 14336, 1), (300, 28672, 2)])  # long rows: fewer ring stages than consumer warps
def test_q4_0_mul_mat_vs_oracle(n, k, m):
    rng = np.random.default_rng(100 + n + m)
    w = rng.normal(0, 0.02, (n, k)).astype(np.float32)
    a = rng.normal(0, 1.0, (m, k)).astype(np.float32)
    rows = oracle.quantize_q4_0(w)
    want = oracle.mul_mat_q4_0_f32(rows, a)
    # exact-integer GEMV path (M <= 4 by default; forced for larger M, where the default is the bf16 tensor-core GEMM)
    got = run_mul_mat(ns.Weight.from_q4_0_host(rows, n, k), a, flags=ns.MM_FORCE_GEMV)
    close(got, want)
    # greedy pick parity on this "logit" row
    assert oracle.argmax(got[0]) == oracle.argmax(want[0])


@pytest.mark.parametrize("n,k,m", [(40, 1024, 1), (32000, 4096, 1), (1001, 2048, 3), (64, 4096, 4), (24, 512, 6)])
def test_q6_K_mul_mat_bit_exact(n, k, m):
    """NE_TYPE_Q6_K x Q8_K (lm_head of llama.cpp "Q4_0" GGUF files): the kernel keeps the AVX2 body's lane structure and
    fma order (vec_dot.h:907-983), so the result is bit-identical to the CPU path, not merely close."""
    rng = np.random.default_rng(300 + n + m)
    w = rng.normal(0, 0.02, (n, k)).astype(np.float32)
    a = rng.normal(0, 1.0, (m, k)).astype(np.float32)
    if m > 1:
        a[1, :256] = 0.0
    rows = oracle.quantize_q6_K(w)
    wd = ns.Weight.from_q6_K_host(rows, n, k)
    assert wd.wfmt == ns.W_Q6K
    assert np.array_equal(_dequant_dev(wd), oracle.dequantize_q6_K(rows, k))
    want = oracle.mul_mat_q6_K_f32(rows, a)
    got = run_mul_mat(wd, a)
    assert np.array_equal(got, want)
    assert oracle.argmax(got[0]) == oracle.argmax(want[0])
    bias = rng.normal(0, 1, (1, n)).astype(np.float32)
    assert np.array_equal(run_mul_mat(wd, a, bias=bias, flags=ns.MM_BIAS_BCAST), want + bias)


def test_q6_K_golden_fixture_through_host_abi():
    z = np.load(os.path.join(G, "ggml_q6_K.npz"))
    wq, a, want = np.ascontiguousarray(z["wq"]), np.ascontiguousarray(z["a"]), z["out"]
    n, k = z["w"].shape
    out = np.zeros((a.shape[0], n), np.float32)
    rc = ns.lib().ns_mul_mat_q6_K_f32_host(wq.ctypes.data_as(C.c_void_p), wq.shape[1], a.ctypes.data_as(C.c_void_p),
                                           out.ctypes.data_as(C.c_void_p), k, n, a.shape[0])
    assert rc == 0, ns.last_error()
    assert np.array_equal(out, want)


def test_q6_K_is_rejected_by_the_fused_nodes():
    rows = oracle.quantize_q6_K(np.random.default_rng(1).normal(0, 0.02, (64, 256)).astype(np.float32))
    w = ns.Weight.from_q6_K_host(rows, 64, 256)
    import torch
    x = torch.zeros(1, 256, device="cuda")
    out = torch.zeros(3, 1, 64, device="cuda")
    assert ns.lib().ns_mul_qkv(w.h, w.h, w.h, C.c_void_p(x.data_ptr()), 256, C.c_void_p(out.data_ptr()), 64, 1, None, None) != 0


def test_q4_0_golden_fixture_through_host_abi():
    z = np.load(os.path.join(G, "ggml_q4_0.npz"))
    wq, a, want = np.ascontiguousarray(z["wq"]), np.ascontiguousarray(z["a"]), z["out"]
    n, k = z["w"].shape
    out = np.zeros((a.shape[0], n), np.float32)
    rc = ns.lib().ns_mul_mat_q4_0_f32_host(wq.ctypes.data_as(C.c_void_p), wq.shape[1], a.ctypes.data_as(C.c_void_p),
                                           out.ctypes.data_as(C.c_void_p), k, n, a.shape[0])
    assert rc == 0, ns.last_error()
    close(out, want, 1e-2)  # 5 rows > 4: the host ABI takes the bf16 tensor-core GEMM (north-star logits bar)
    out4 = np.zeros((4, n), np.float32)
    rc = ns.lib().ns_mul_mat_q4_0_f32_host(wq.ctypes.data_as(C.c_void_p), wq.shape[1], a.ctypes.data_as(C.c_void_p),
                                           out4.ctypes.data_as(C.c_void_p), k, n, 4)
    assert rc == 0, ns.last_error()
    close(out4, want[:4])  # <= 4 rows: exact-integer GEMV path


def test_q4_0_block_sums_are_exact_integers():
    """acts = exact small integers, unit scales: every output is an exact integer, so GPU == oracle bit-for-bit."""
    rng = np.random.default_rng(9)
    n, k = 64, 1024
    codes = rng.integers(0, 16, (n, k)).astype(np.int32)
    w = (codes - 8).astype(np.float32)
    w[:, ::32] = -8.0  # pins every block scale to d = 1 (max magnitude element is -8 -> d = -8 / -8)
    a = rng.integers(-127, 128, (2, k)).astype(np.float32)
    a[:, ::32] = 127.0  # pins every activation block scale to 1
    rows = oracle.quantize_q4_0(w)
    assert np.array_equal(oracle.dequantize_q4_0(rows, k), w)
    want = oracle.mul_mat_q4_0_f32(rows, a)
    got = run_mul_mat(ns.Weight.from_q4_0_host(rows, n, k), a)
    assert np.array_equal(want, np.round(want))
    assert np.array_equal(got, want)


# ------------------------------------------------------------------------------------------------------- BesTLA
def _btla_case(seed, n, k, m):
    rng = np.random.default_rng(seed)
    w = rng.uniform(-0.5, 0.5, (k, n)).astype(np.float32)  # bestla_ut.h:130-167 fill convention
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    return w, a


@pytest.mark.parametrize("asym", [False, True])
@pytest.mark.parametrize("g,k", [(32, 1024), (128, 4096), (-1, 1024), (128, 11008)])
@pytest.mark.parametrize("m", [1, 4])
def test_btla_s4_int8_compute(asym, g, k, m):
    n = 192
    w, a = _btla_case(7 + k + m, n, k, m)
    gg = k if g == -1 else g
    q, sc, zp = oracle.btla_quantize(w, gg, 4, asym)
    a8, asc, azp = oracle.btla_quantize_act_u8(a, gg)
    want = oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, gg)
    want_blk = oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, gg, blocksum=True)
    wd = ns.Weight.from_unpacked(q, sc, zp, gg, ns.W_S4, ns.S_F32, ns.COMP_INT8)
    got = run_mul_mat(wd, a)
    close(got, want_blk, 2e-5)
    close(got, want)
    # UT_CompInt8 criterion: vs fp32 GEMM on dequantised W and dequantised A
    adq = (a8.astype(np.float32) - np.repeat(azp, gg, 1)[:, :k].astype(np.float32)) * np.repeat(asc, gg, 1)[:, :k]
    close(got, oracle.gemm_f64acc(adq, oracle.btla_dequant(q, sc, zp, gg)), 1e-4)


@pytest.mark.parametrize("asym", [False, True])
@pytest.mark.parametrize("m", [1, 2, 3, 4, 6])
def test_btla_s4_s8_activations(asym, m):
    n, k, g = 128, 2048, 128
    w, a = _btla_case(50 + m, n, k, m)
    q, sc, zp = oracle.btla_quantize(w, g, 4, asym)
    a8, asc = oracle.btla_quantize_act_s8(a, g)
    want = oracle.btla_gemv_s8s8(a8, asc, q, sc, zp, g)
    got = run_mul_mat(ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S4, ns.S_F32, ns.COMP_INT8_S8), a, flags=ns.MM_FORCE_GEMV)
    close(got, want)


@pytest.mark.parametrize("asym", [False, True])
@pytest.mark.parametrize("g,k,m", [(32, 1024, 1), (128, 4096, 2), (128, 11008, 4)])
def test_btla_s4_fp32_compute(asym, g, k, m):
    n = 96
    w, a = _btla_case(90 + k, n, k, m)
    q, sc, zp = oracle.btla_quantize(w, g, 4, asym)
    got = run_mul_mat(ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S4, ns.S_F32, ns.COMP_F32), a)
    ref = oracle.gemm_f64acc(a, oracle.btla_dequant(q, sc, zp, g))
    assert np.abs(got - ref).max() <= 1e-3          # ut_int criterion (b)
    assert np.abs(got - oracle.gemm_f64acc(a, w)).max() <= 3.5  # criterion (a): INT4 @ K=4096 (bestla_ut.h:80-94)
    close(got, oracle.btla_gemv_fp32(a, q, sc, zp, g), 1e-4)


@pytest.mark.parametrize("g", [32, 128])
def test_btla_nf4(g):
    n, k, m = 160, 2048, 3
    w, a = _btla_case(31, n, k, m)
    q, sc = oracle.btla_quantize_nf4(w, g)
    got = run_mul_mat(ns.Weight.from_unpacked(q, sc, None, g, ns.W_NF4, ns.S_F32, ns.COMP_F32), a)
    ref = oracle.gemm_f64acc(a, oracle.btla_dequant(q, sc, None, g, nf4=True))
    assert np.abs(got - ref).max() <= 1e-3


@pytest.mark.parametrize("comp", ["int8", "fp32", "s8"])
@pytest.mark.parametrize("asym", [False, True])
def test_btla_s8_weights(comp, asym):
    n, k, m, g = 96, 1024, 2, 128
    w, a = _btla_case(77, n, k, m)
    q, sc, zp = oracle.btla_quantize(w, g, 8, asym)
    if comp == "fp32":
        got = run_mul_mat(ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S8, ns.S_F32, ns.COMP_F32), a)
        assert np.abs(got - oracle.gemm_f64acc(a, oracle.btla_dequant(q, sc, zp, g))).max() <= 1e-3
    elif comp == "int8":
        a8, asc, azp = oracle.btla_quantize_act_u8(a, g)
        got = run_mul_mat(ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S8, ns.S_F32, ns.COMP_INT8), a)
        close(got, oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, g))
    else:
        a8, asc = oracle.btla_quantize_act_s8(a, g)
        got = run_mul_mat(ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S8, ns.S_F32, ns.COMP_INT8_S8), a)
        close(got, oracle.btla_gemv_s8s8(a8, asc, q, sc, zp, g))


def test_btla_bf16_scales_and_bf16_compute():
    n, k, m, g = 128, 2048, 2, 128
    w, a = _btla_case(41, n, k, m)
    q, sc, zp = oracle.btla_quantize(w, g, 4, False)
    sc_b = oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(sc))
    got = run_mul_mat(ns.Weight.from_unpacked(q, sc, None, g, ns.W_S4, ns.S_BF16, ns.COMP_F32), a)
    assert np.abs(got - oracle.gemm_f64acc(a, oracle.btla_dequant(q, sc_b, None, g))).max() <= 1e-3
    got = run_mul_mat(ns.Weight.from_unpacked(q, sc, None, g, ns.W_S4, ns.S_F32, ns.COMP_BF16), a)
    a_b = oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(a))
    assert np.abs(got - oracle.gemm_f64acc(a_b, oracle.btla_dequant(q, sc, None, g))).max() <= 2e-2  # BF16 tol, bestla_ut.h:80-94


def test_gptq_act_order_shuffle():
    """desc_act: groups are contiguous after sorting columns by g_idx; the kernel gathers activation columns
    (ShuffleActivationKBlock*, bestla_prologue_a.h:299-424) before quantising them."""
    rng = np.random.default_rng(17)
    n, k, m, g = 64, 1024, 2, 128
    w, a = _btla_case(18, n, k, m)
    perm = rng.permutation(k).astype(np.int32)          # position j of the sorted weight holds original column perm[j]
    q, sc, zp = oracle.btla_quantize(np.ascontiguousarray(w[perm]), g, 4, True)
    wd = ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S4, ns.S_F32, ns.COMP_INT8, shuffle=perm)
    got = run_mul_mat(wd, a)
    a_sh = np.ascontiguousarray(a[:, perm])
    a8, asc, azp = oracle.btla_quantize_act_u8(a_sh, g)
    close(got, oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, g))


@pytest.mark.parametrize("name", ["gptq4_asym", "gptq4_sym", "gptq4_desc", "gptq8_asym", "awq4"])
def test_gptq_awq_checkpoint_tensors_to_device_weight(name):
    """Config 3: HF qweight/qzeros/scales/g_idx -> device weight -> matmul equals the checkpoint's own dequantised weights
    (fp32 compute: sycl_gemm.cpp:404-442 tolerance 1e-3), and the int8 path equals the CPU oracle on the canonical tensors."""
    import os
    from neural_speed_b200 import convert
    gold = np.load(os.path.join(os.path.dirname(__file__), "golden", "gptq_awq.npz"))
    bits, g, sym, desc = (int(v) for v in gold[f"{name}.cfg"])
    cfg = dict(quant_method=str(gold[f"{name}.method"]), bits=bits, group_size=g, sym=bool(sym), desc_act=bool(desc))
    args = (gold[f"{name}.qweight"], gold[f"{name}.scales"], gold[f"{name}.qzeros"], gold[f"{name}.g_idx"])
    c = convert.to_canonical(*args, **cfg)
    k, n = c["q"].shape
    rng = np.random.default_rng(41)
    a = rng.uniform(-0.5, 0.5, (3, k)).astype(np.float32)
    order = np.argsort(gold[f"{name}.g_idx"], kind="stable") if desc else np.arange(k)
    wdq = oracle.btla_dequant(c["q"], c["scales"], c["zp"], g)               # [K, N] in regrouped row order
    got = run_mul_mat(convert.to_weight(*args, comp=ns.COMP_F32, **cfg), a)
    assert np.abs(got - oracle.gemm_f64acc(np.ascontiguousarray(a[:, order]), wdq)).max() <= 1e-3
    if bits == 4:
        got8 = run_mul_mat(convert.to_weight(*args, **cfg), a)
        a8, asc, azp = oracle.btla_quantize_act_u8(np.ascontiguousarray(a[:, order]), g)
        zp = c["zp"] if c["zp"] is not None else None
        close(got8, oracle.btla_gemv_u8s8(a8, asc, azp, c["q"], c["scales"], zp, g))


# ------------------------------------------------------------------------------------------------------- blobs + drop-ins
@pytest.mark.parametrize("cdt,sdt,alg", [("int8", "fp32", "sym"), ("int8", "bf16", "asym"), ("fp32", "fp32", "sym"),
                                         ("bf16", "fp32", "asym")])
def test_blob_load_and_host_forward(cdt, sdt, alg):
    n, k, m, g = 200, 1024, 3, 128  # n not a multiple of NTile
    rng = np.random.default_rng(23)
    wt = rng.uniform(-0.5, 0.5, (n, k)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    blob = ns.np_bestla_quantize(wt, "int4", g, alg, sdt, cdt)
    wdq = ns.unpack_blob(blob, n, k)  # [K,N], host (already checked against the oracle on CPU)
    # device repack of the blob is lossless
    assert np.array_equal(_dequant_dev(ns.Weight.from_blob(blob)), wdq.T)
    # host-buffer drop-in
    L = ns.lib()
    out = np.full((m, n), np.nan, np.float32)
    ws = L.bestla_f32f32_get_workspace_size(m, n, k, blob.ctypes.data_as(C.c_void_p))
    assert ws == m * (-(-k // 128) * 128) * 4
    L.bestla_f32f32_forward(a.ctypes.data_as(C.c_void_p), blob.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p),
                            m, n, k, k, n, None)
    if cdt == "int8":
        q, sc, zp = oracle.btla_quantize(np.ascontiguousarray(wt.T), g, 4, alg == "asym")
        if sdt == "bf16":
            sc = oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(sc))
        a8, asc, azp = oracle.btla_quantize_act_u8(a, g)
        close(out, oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, g))
    else:
        tol = 1e-3 if cdt == "fp32" else 2e-2
        a_eff = a if cdt == "fp32" else oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(a))
        assert np.abs(out - oracle.gemm_f64acc(a_eff, wdq)).max() <= tol
    # bias epilogue (bestla_fusion_add_f32f32_forward)
    bias = rng.normal(0, 1, (1, n)).astype(np.float32)
    out2 = np.zeros((m, n), np.float32)
    assert L.bestla_fusion_add_f32f32_support(blob.ctypes.data_as(C.c_void_p), m, n, k)
    L.bestla_fusion_add_f32f32_forward(a.ctypes.data_as(C.c_void_p), blob.ctypes.data_as(C.c_void_p),
                                       bias.ctypes.data_as(C.c_void_p), out2.ctypes.data_as(C.c_void_p), m, n, k, k, n, True, None)
    close(out2, out + bias, 1e-6)
    # device unpack
    up = np.zeros((n, k), np.float32)
    L.bestla_unpackweight_fp32(blob.ctypes.data_as(C.c_void_p), n, k, up.ctypes.data_as(C.c_void_p), k)
    assert np.array_equal(up, wdq.T)


def test_fused_qkv_and_ffn_drop_ins():
    rng = np.random.default_rng(29)
    m, k, n, fmid, g = 2, 512, 512, 1408, 128
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    mk = lambda r, c: ns.np_bestla_quantize(rng.uniform(-0.5, 0.5, (r, c)).astype(np.float32), "int4", g, "sym", "fp32", "int8")
    bq, bk, bv = mk(n, k), mk(n, k), mk(n, k)
    L = ns.lib()
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    assert L.bestla_fusion_QKV_f32f32_support(p(bq), p(bk), p(bv), m, n, k)
    out = np.zeros((3, m, n), np.float32)
    L.bestla_fusion_QKV_f32f32_forward(p(a), p(bq), p(bk), p(bv), p(out), m, n, k, k, n, None)
    for i, b in enumerate((bq, bk, bv)):
        single = np.zeros((m, n), np.float32)
        L.bestla_f32f32_forward(p(a), p(b), p(single), m, n, k, k, n, None)
        assert np.array_equal(out[i], single)  # same kernel arithmetic, fused or not
    # FFN: out = (silu(x W1) * (x W3)) W2
    b1, b3, b2 = mk(fmid, k), mk(fmid, k), mk(n, fmid)
    assert L.bestla_fusion_FFN_SiLu_f32f32_support(p(b1), p(b2), p(b3), m, k, fmid, n)
    tmp1 = np.zeros((m, fmid), np.float32)
    tmp2 = np.zeros((m, fmid), np.float32)
    ffn = np.zeros((m, n), np.float32)
    L.bestla_fusion_FFN_SiLu_f32f32_forward(p(a), p(b1), p(b2), p(b3), p(tmp1), p(tmp2), p(ffn), m, k, fmid, n, None)
    g1 = np.zeros((m, fmid), np.float32)
    u1 = np.zeros((m, fmid), np.float32)
    L.bestla_f32f32_forward(p(a), p(b1), p(g1), m, fmid, k, k, fmid, None)
    L.bestla_f32f32_forward(p(a), p(b3), p(u1), m, fmid, k, k, fmid, None)
    silu = np.array([[oracle.lib().orc_silu(float(v)) for v in row] for row in g1], np.float32)
    close(tmp2, silu * u1, 1e-5)
    want = np.zeros((m, n), np.float32)
    L.bestla_f32f32_forward(p(np.ascontiguousarray(tmp2)), p(b2), p(want), m, n, fmid, fmid, n, None)
    close(ffn, want, 1e-6)


def _gelu(x):
    x = x.astype(np.float32)
    return (np.float32(0.5) * x * (np.float32(1) + np.tanh(np.float32(0.7978845834732056) *
                                                           (x + np.float32(0.044714998453855515) * x * x * x)))).astype(np.float32)


@pytest.mark.parametrize("m", [2, 8])
def test_gelu_ffn_drop_ins(m):
    """bestla_fusion_FFN_{Gelu_Mul,GeLu,Add_GeLu}_f32f32_forward (ip_fusion_ffn.cpp:745-779): the fused node must equal the
    same matmuls issued one by one with the tanh-GELU of kernel_ref.h:1570 between them."""
    rng = np.random.default_rng(31 + m)
    k, n, fmid, g = 512, 384, 1408, 128
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    mk = lambda r, c: ns.np_bestla_quantize(rng.uniform(-0.5, 0.5, (r, c)).astype(np.float32), "int4", g, "sym", "fp32", "int8")
    b1, b3, b2 = mk(fmid, k), mk(fmid, k), mk(n, fmid)
    L = ns.lib()
    p = lambda x: x.ctypes.data_as(C.c_void_p)
    tol = 1e-5 if m <= 4 else 2e-2  # m > 4 runs the bf16 tensor-core GEMM

    def mm(x, b, rows, cols):
        o = np.zeros((m, rows), np.float32)
        L.bestla_f32f32_forward(p(np.ascontiguousarray(x)), p(b), p(o), m, rows, cols, cols, rows, None)
        return o

    # Gelu_Mul
    assert L.bestla_fusion_FFN_Gelu_Mul_f32f32_support(p(b1), p(b2), p(b3), m, k, fmid, n)
    tmp1, tmp2, out = np.zeros((m, fmid), np.float32), np.zeros((m, fmid), np.float32), np.zeros((m, n), np.float32)
    L.bestla_fusion_FFN_Gelu_Mul_f32f32_forward(p(a), p(b1), p(b2), p(b3), p(tmp1), p(tmp2), p(out), m, k, fmid, n, None)
    want_mid = _gelu(mm(a, b1, fmid, k)) * mm(a, b3, fmid, k)
    close(tmp2, want_mid, tol)
    close(out, mm(tmp2, b2, n, fmid), tol)
    # GeLu
    assert L.bestla_fusion_FFN_GeLu_f32f32_support(p(b1), p(b2), m, k, fmid, n)
    assert not L.bestla_fusion_FFN_GeLu_f32f32_support(p(b1), p(b2), m, k, fmid + 1, n)
    tmp1[:] = 0
    out[:] = 0
    L.bestla_fusion_FFN_GeLu_f32f32_forward(p(a), p(b1), p(b2), p(tmp1), p(out), m, k, fmid, n, None)
    close(tmp1, _gelu(mm(a, b1, fmid, k)), tol)
    close(out, mm(tmp1, b2, n, fmid), tol)
    # Add_GeLu, broadcast and per-row biases
    for bcast in (True, False):
        bias1 = rng.normal(0, 0.5, (1 if bcast else m, fmid)).astype(np.float32)
        bias2 = rng.normal(0, 0.5, (1 if bcast else m, n)).astype(np.float32)
        assert L.bestla_fusion_FFN_Add_GeLu_f32f32_support(p(b1), p(b2), m, k, fmid, n)
        L.bestla_fusion_FFN_Add_GeLu_f32f32_forward(p(a), p(b1), p(b2), p(bias1), p(bias2), p(tmp1), p(out), m, k, fmid, n, bcast,
                                                    None)
        close(tmp1, _gelu(mm(a, b1, fmid, k) + bias1), tol)
        close(out, mm(tmp1, b2, n, fmid) + bias2, tol)


def test_device_set_load_storage_and_forward():
    """the NS_SYCL-style device API: create_device / malloc / load_storage / device forward / memcpy / sync"""
    rng = np.random.default_rng(37)
    n, k, m, g = 256, 1024, 1, 32
    wt = rng.uniform(-0.5, 0.5, (n, k)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    blob = ns.np_bestla_quantize(wt, "int4", g, "sym", "fp32", "int8")
    L = ns.lib()
    d = L.bestla_create_device(False)
    q = L.bestla_get_device_queue(d)
    assert L.bestla_device_gmem_size(d) == torch.cuda.mem_get_info()[1] > (64 << 30)  # the whole device: 80 GB on an H100
    nbytes = L.ns_device_storage_bytes(blob.ctypes.data_as(C.c_void_p))
    assert nbytes >= n * k // 2
    dw = L.bestla_device_malloc(nbytes, q)
    desc = (C.c_char * L.bestla_device_storage_size())()
    L.bestla_device_load_storage(blob.ctypes.data_as(C.c_void_p), desc, dw, q)
    da = L.bestla_device_malloc(a.nbytes, q)
    do = L.bestla_device_malloc(m * n * 4, q)
    L.bestla_device_memcpy_sync(da, a.ctypes.data_as(C.c_void_p), a.nbytes, q)
    L.bestla_device_f32f32_forward(da, desc, do, m, n, k, k, n, None, q)
    out = np.zeros((m, n), np.float32)
    L.bestla_device_memcpy(out.ctypes.data_as(C.c_void_p), do, out.nbytes, q)
    L.bestla_device_sync(q)
    qq, sc, zp = oracle.btla_quantize(np.ascontiguousarray(wt.T), g, 4, False)
    a8, asc, azp = oracle.btla_quantize_act_u8(a, g)
    close(out, oracle.btla_gemv_u8s8(a8, asc, azp, qq, sc, zp, g))
    for ptr in (da, do, dw):
        L.bestla_device_free(ptr, q)
    L.bestla_release_device(d)


def test_btla_golden_fixture():
    z = np.load(os.path.join(G, "btla_quant.npz"))
    a = z["a"]
    for g in (32, 128):
        q, sc, zp = z[f"s4_g{g}_asym_q"], z[f"s4_g{g}_asym_sc"], z[f"s4_g{g}_asym_zp"]
        got = run_mul_mat(ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S4, ns.S_F32, ns.COMP_INT8), a)
        want = oracle.btla_gemv_u8s8(z[f"act_u8_g{g}_q"], z[f"act_u8_g{g}_sc"], z[f"act_u8_g{g}_zp"], q, sc, zp, g)
        close(got, want)


# ------------------------------------------------------------------------------------------------------- full-size properties
def test_full_size_linearity_and_row_independence():
    """Llama-2-7B shapes, too big for the scalar oracle to cover densely: check size-independent properties.
    (1) row independence: any output row equals the same row computed from a 64-row slice of the weight;
    (2) exact homogeneity: scaling the activations by 2 scales every output by exactly 2 (power-of-two scaling commutes
        with Q8_0 quantisation bit-for-bit)."""
    torch.manual_seed(1234)
    n, k = 11008, 4096
    w = (torch.randn(n, k, device="cuda") * 0.02)
    rows = torch.zeros(n * k // 32 * 18, dtype=torch.uint8, device="cuda")
    assert ns.lib().ns_device_quantize_q4_0(C.c_void_p(w.data_ptr()), C.c_void_p(rows.data_ptr()), n, k, None) == 0
    sync()
    nb01 = k // 32 * 18
    wd = ns.Weight.from_q4_0_device(rows.data_ptr(), n, k, nb01)
    a = torch.randn(1, k, device="cuda")
    out = torch.zeros(1, n, device="cuda")
    out2 = torch.zeros(1, n, device="cuda")
    a2 = a * 2
    torch.cuda.synchronize()
    ns.mul_mat(wd, a.data_ptr(), k, out.data_ptr(), n, 1)
    ns.mul_mat(wd, a2.data_ptr(), k, out2.data_ptr(), n, 1)
    sync()
    assert torch.equal(out2, out * 2)
    r0 = 7000
    sub = ns.Weight.from_q4_0_device(rows.data_ptr() + r0 * nb01, 64, k, nb01)
    o_sub = torch.zeros(1, 64, device="cuda")
    ns.mul_mat(sub, a.data_ptr(), k, o_sub.data_ptr(), 64, 1)
    sync()
    assert torch.equal(o_sub[0], out[0, r0:r0 + 64])
    # and the slice against the oracle
    rows_h = rows.view(n, nb01)[r0:r0 + 64].cpu().numpy()
    close(o_sub.cpu().numpy(), oracle.mul_mat_q4_0_f32(rows_h, a.cpu().numpy()))

"""GPU parity of the wgmma tensor-core GEMM (gemm_w4_tc_kernel, M > 4 by default, any M with MM_FORCE_TC) against its stated
arithmetic (oracle.tc_operands, DESIGN.md section 4):
  a_eff = bf16_rn(a), w_eff = bf16_rn(bf16(q - zp) * bf16_rn(s)) or bf16_rn(bf16_rn(level) * bf16_rn(s)); fp32 accumulation on
  the tensor cores in any order; with S > 1 k slices each slice's partial is atomically added into a zeroed dst, slice 0 adding
  bias then residual first; only dst[:m, :n] is written.
Tiers:
  A/B exact: inputs with oracle.tc_exact_budget < 2^24 (sparse activation rows of 8-significant-bit values, asserted per case), so
      every partial sum in any order and any split is exact in fp32 and the result equals the fp64 sum bit for bit.  That rests
      on HGMMA accumulating bf16 products into fp32 without losing bits below 2^24 grid steps: it held on an NVIDIA H100 80GB HBM3
      (700 W power limit) for every case here (budgets up to 2^22.4).  The data
      still needs every rounding: activations off the bf16 grid (ties included), scales off it (ties included), fp16 d values
      (normal and subnormal) off it, a different scale per group, zero points at their extremes, int8 codes -128 and 127.
  C   random data: |got - sum a_eff w_eff| <= (ceil(K/16) + S) 2^-22 sum |a_eff w_eff| per element.
  D   bit-for-bit invariants where the plan has one k slice: row permutations, repeated launches.
  E   the eval step's one-image FFN against the two-step ns_ffn_silu.
Every kernel call passes MM_FORCE_TC, makes 2 launches (activation image + GEMM), and writes into a NaN-filled dst with ldo > n and
3 guard rows that must stay NaN.  Each case reads its token tile and k slices from ns_gemm_tc_plan, the launcher's own function.
The older checks stay: (2) the reference's CompBf16 UT tolerance and (3) the north-star bar, <= 1e-2 relative vs the CPU path."""
import ctypes as C
import functools

import numpy as np
import pytest

import oracle
import neural_speed_b200 as ns
from oracle import btla_blob

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

GUARD = 3        # NaN rows below the output
EXACT = 2 ** 24  # tc_exact_budget bar
PROD_CAP = 2 ** 23  # what the sparse activation rows may spend of it; bias / residual get at most 2^22 more


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def bf16r(x):
    return oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(np.asarray(x, np.float32)))


def plan(m, n, k, aliased=False):
    """(T, k slices S, k blocks per slice) of the launch, from the launcher's own plan on this card"""
    out = (C.c_int * 3)()
    assert ns.lib().ns_gemm_tc_plan(m, n, -(-k // 32) * 32, 1 if aliased else 0, out) == 0, ns.last_error()
    return tuple(out)


def run(w, a, bias=None, residual=None, flags=None, lda=None, ldo=None, offset=False, alias=False):
    """one ns_mul_mat call -> dst[:m, :n].  dst is [m + GUARD][ldo] of NaN (ldo defaults to n + 5) and must keep its NaNs outside
    [0, m) x [0, n); with MM_FORCE_TC (the default) the call must make exactly 2 launches.  lda > k puts NaN in the skipped
    activation columns; offset shifts the activations 4 bytes off their 16-byte alignment.  bias: [n] with MM_BIAS_BCAST in flags,
    else [m][n] laid out [m][ldo]; residual [m][n] laid out [m][ldo], or written into dst itself with alias."""
    m, k = a.shape
    if flags is None:  # this file tests the tensor-core kernel: M <= 16 would take the exact-integer GEMV tiles by default
        flags = ns.MM_FORCE_TC
    lda = lda or k
    ldo = ldo or w.n + 5
    abuf = np.full(m * lda + 4, np.nan, np.float32)
    o0 = 1 if offset else 0
    abuf[o0:o0 + m * lda].reshape(m, lda)[:, :k] = a
    ad = torch.from_numpy(abuf).cuda()
    out = torch.full((m + GUARD, ldo), float("nan"), device="cuda")

    def padded(x):
        buf = np.full((m, ldo), np.nan, np.float32)
        buf[:, :w.n] = x
        return torch.from_numpy(buf).cuda()

    b = None
    if bias is not None:
        b = torch.from_numpy(np.ascontiguousarray(bias, np.float32)).cuda() if flags & ns.MM_BIAS_BCAST else padded(bias)
    r = None
    if residual is not None:
        if alias:
            out[:m, :w.n] = torch.from_numpy(np.ascontiguousarray(residual, np.float32)).cuda()
            r = out
        else:
            r = padded(residual)
    torch.cuda.synchronize()
    lc = ns.lib().ns_launch_count()
    ns.mul_mat(w, ad.data_ptr() + 4 * o0, lda, out.data_ptr(), ldo, m, b.data_ptr() if b is not None else None,
               r.data_ptr() if r is not None else None, flags)
    torch.cuda.synchronize()
    ns.lib().bestla_device_sync(None)
    launches = ns.lib().ns_launch_count() - lc
    if flags & ns.MM_FORCE_TC:
        assert launches == 2, launches
    o = out.cpu().numpy()
    assert np.isnan(o[:, w.n:]).all() and np.isnan(o[m:]).all(), "write outside [0, m) x [0, n)"
    return o[:m, :w.n]


def c_bar_ratio(got, a_eff, w_eff, splits):
    """max over outputs of |got - sum a_eff w_eff| / ((ceil(K/16) + S) 2^-22 sum |a_eff w_eff|): one truncation per k16 MMA and one
    rounding per k slice; a correct kernel stays at or below 1"""
    want, mag = oracle.gemv_stated(a_eff, w_eff)
    unit = (-(-a_eff.shape[1] // 16) + splits) * 2.0 ** -22 * np.maximum(mag, np.finfo(np.float32).tiny)
    return float((np.abs(got.astype(np.float64) - want) / unit).max())


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
    a_eff, w_eff = oracle.tc_operands(a, "s4", q, sc, zp, g)
    assert c_bar_ratio(got, a_eff, w_eff, plan(m, n, k)[1]) <= 1
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
    a_eff, w_eff = oracle.tc_operands(a, "nf4", q, sc, None, g)
    assert c_bar_ratio(got, a_eff, w_eff, plan(m, n, k)[1]) <= 1
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
    a_eff, w_eff = oracle.tc_operands(a, "s8", q, sc, zp, g)
    assert c_bar_ratio(got, a_eff, w_eff, plan(m, n, k)[1]) <= 1
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
    a_eff, w_eff2 = oracle.tc_operands(a, "q4_0", qv.reshape(n, k).T, d.T)
    assert np.array_equal(w_eff2, w_eff.T)
    assert c_bar_ratio(got, a_eff, w_eff2, plan(m, n, k)[1]) <= 1
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
    assert plan(m, n, k)[1] == 1  # one slice; the split epilogue is held exactly below (test_tc_exact_epilogue)


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


# ----------------------------------------------------------------------------------------------------------- exact tier (A, B)
STYPES = {"f32": ns.S_F32, "bf16": ns.S_BF16, "f16": ns.S_F16}


def off_grid_scales(rng, shape, stype="f32"):
    """scales in [1, 2) that bf16 must round, a quarter of them exact ties: fp32 values with 16 bits below the bf16 significand,
    or for fp16 storage fp16 values with 3 (the fp16 grid is what the weight keeps)"""
    m = rng.integers(128, 256, shape)
    tie = rng.random(shape) < 0.25
    if stype == "f16":
        r = np.where(tie, 4, rng.integers(0, 8, shape))
        return ((m * 8 + r) / 1024.0).astype(np.float32)
    r = np.where(tie, 1 << 15, rng.integers(0, 1 << 16, shape))
    return ((m * 65536 + r) / 2.0 ** 23).astype(np.float32)


def fp16_bits(d):
    return np.ascontiguousarray(d, np.float16).view(np.uint8)


class XW:
    """A device weight whose effective operands have a narrow dynamic range (so that sparse activation rows fit the exact budget)
    and need every rounding step of the stated arithmetic, with its w_eff [K, N]."""

    def __init__(self, fmt, n, k, g=32, asym=False, stype="f32", seed=0, shuffle=False, subnormal=False):
        rng = np.random.default_rng(seed)
        self.fmt, self.n, self.k, self.g = fmt, n, k, g
        nb = -(-k // g)
        self.perm = rng.permutation(k).astype(np.int32) if shuffle else None
        zp = None
        if fmt in ("q4_0", "q8_0"):
            g = self.g = 32
            j = rng.integers(128, 256, (k // 32, n))
            if subnormal:  # fp16 subnormals j * 2^-24 with 10 significant bits, ties where the low two are 10
                r = rng.integers(0, 4, j.shape)
                d = ((j * 4 + r) * 2.0 ** -24).astype(np.float16)
            else:
                d = off_grid_scales(rng, j.shape, "f16").astype(np.float16) / 64
            assert (d.astype(np.float32) != bf16r(d.astype(np.float32))).mean() > 0.5
            if fmt == "q4_0":
                nib = rng.integers(0, 16, (k, n))
                q = nib - 8
                x = nib.T.reshape(n, k // 32, 32).astype(np.uint8)
                rows = np.concatenate([fp16_bits(d.T).reshape(n, k // 32, 2), x[:, :, :16] | (x[:, :, 16:] << 4)], axis=2)
                self.rows = rows.reshape(n, k // 32 * 18)
                assert np.array_equal(oracle.dequantize_q4_0(self.rows, k),
                                      (q * d.astype(np.float32)[np.arange(k) // 32]).T.astype(np.float32))
                self.w = ns.Weight.from_q4_0_host(self.rows, n, k)
            else:
                q = np.clip(rng.choice([-1, 1], (k, n)) * rng.integers(64, 129, (k, n)), -128, 127)
                x = q.T.reshape(n, k // 32, 32).astype(np.int8).view(np.uint8)
                rows = np.concatenate([fp16_bits(d.T).reshape(n, k // 32, 2), x], axis=2)
                self.rows = rows.reshape(n, k // 32 * 34)
                self.w = ns.Weight.from_q8_0_host(self.rows, n, k)
            sc = d.astype(np.float32)
        elif fmt in ("f4_bnb", "f4_e2m1"):
            # an fp32 weight that quantises to chosen codes: level x group scale, one +-1 level per group (the absmax); the
            # 2^-7.6 / 2^-6.6 levels (codes 1, 9) are left out, they alone would spend the budget
            lv = oracle.f4_levels(fmt)
            allowed = np.array([c for c in range(16) if c not in (1, 8, 9)])  # 8: -0 quantises to code 0
            codes = rng.choice(allowed, (k, n))
            one = 3 if fmt == "f4_bnb" else 7
            codes[np.arange(0, k, g)] = one + 8 * rng.integers(0, 2, (nb, n))
            s = off_grid_scales(rng, (nb, n))
            wt = (lv[codes] * s[np.arange(k) // g]).astype(np.float32)
            blob = ns.np_bestla_quantize(np.ascontiguousarray(wt.T), fmt.replace("f4_", "fp4_"), g, "sym",
                                         {"f32": "fp32", "bf16": "bf16"}[stype], "bf16")
            got = btla_blob.codes(blob)
            q, sc = got["q"], got["scale"]
            assert np.array_equal(q, codes)
            stype = "f32"  # the parsed scales are the stored values
            self.w = ns.Weight.from_blob(blob)
        else:
            if fmt == "s4":
                q = rng.integers(-8, 8, (k, n))
                if asym:
                    zp = rng.integers(-8, 8, (nb, n))
                    pick = rng.random((nb, n))
                    zp = np.where(pick < 1 / 3, -8, np.where(pick < 2 / 3, 7, zp))
            elif fmt == "s8":
                # |q - zp| in [64, 255] (or 0): codes -128 and 127 come from the clip
                zp = np.zeros((nb, n), np.int64)
                if asym:
                    pick = rng.random((nb, n))
                    zp = np.where(pick < 1 / 3, -128, np.where(pick < 2 / 3, 127, rng.integers(-40, 41, (nb, n))))
                d = rng.choice([-1, 1], (k, n)) * rng.integers(64, 256 if asym else 129, (k, n))
                q = np.clip(zp[np.arange(k) // g] + d, -128, 127)
                assert (q == -128).any() and (q == 127).any()
                if not asym:
                    zp = None
            else:  # nf4
                q = rng.integers(0, 16, (k, n))
            sc = off_grid_scales(rng, (nb, n), stype)
            wfmt = {"s4": ns.W_S4, "s8": ns.W_S8, "nf4": ns.W_NF4}[fmt]
            self.w = ns.Weight.from_unpacked(q.astype(np.int8), sc, zp.astype(np.int8) if zp is not None else None, g, wfmt,
                                             STYPES[stype], ns.COMP_BF16 if fmt != "s4" else ns.COMP_INT8, shuffle=self.perm)
        self.zp = zp
        _, self.w_eff = oracle.tc_operands(None, fmt, q, sc, zp, g, stype)
        assert self.w.n == n and self.w.k == k
        w_abs = np.abs(self.w_eff.astype(np.float64))
        self.lsb = int(np.floor(np.log2(w_abs[w_abs > 0].min()))) - 7
        self.cost_k = w_abs.max(axis=1) / 2.0 ** self.lsb  # the largest product units a unit-range activation can meet in row k

    def act(self, m, seed=1, dense=False):
        """fp32 activations [m][k]: +-(1..2) with 16 bits below the bf16 significand (a quarter exact bf16 ties), zero except on
        a random set of columns per row whose product budget stays within PROD_CAP (every column with dense=True)"""
        rng = np.random.default_rng(seed)
        k = self.k
        mant = rng.integers(128, 256, (m, k))
        r = np.where(rng.random((m, k)) < 0.25, 1 << 15, rng.integers(0, 1 << 16, (m, k)))
        a = (rng.choice([-1.0, 1.0], (m, k)) * (mant * 65536 + r) / 2.0 ** 23).astype(np.float32)
        if dense:
            return a
        src = self.cost_k if self.perm is None else np.empty(k)
        if self.perm is not None:  # image column j reads activation column perm[j]
            src[self.perm] = self.cost_k
        keep = np.zeros((m, k), bool)
        for t in range(m):
            order = rng.permutation(k)
            spent = np.cumsum(256 * src[order])
            keep[t, order[spent <= PROD_CAP]] = True
        return np.where(keep, a, np.float32(0))

    def a_eff(self, a):
        return oracle.tc_operands(a, "s4", np.zeros((self.k, 1)), np.ones((1, 1)), None, self.k, shuffle=self.perm)[0]


@functools.lru_cache(maxsize=None)
def xweight(*args, **kw):
    return XW(*args, **kw)


def check_exact(w, a, bias=None, bcast=False, residual=None, **kw):
    """run and hold the result to the fp64 sum bit for bit; returns (got, plan)"""
    m = a.shape[0]
    a_eff = w.a_eff(a)
    want, mag = oracle.gemv_stated(a_eff, w.w_eff)
    extra = np.zeros_like(want)
    if bias is not None:
        want = want + (bias[None, :] if bcast else bias)
        extra += np.abs(bias[None, :] if bcast else bias)
    if residual is not None:
        want = want + residual
        extra += np.abs(residual)
    budget = oracle.tc_exact_budget(a_eff, w.w_eff, mag, extra)
    assert budget < EXACT, budget
    p = plan(m, w.n, w.k, kw.get("alias", False))
    got = run(w.w, a, bias=bias, residual=residual, flags=ns.MM_FORCE_TC | (ns.MM_BIAS_BCAST if bcast else 0), **kw)
    want32 = want.astype(np.float32)
    assert np.array_equal(want32.astype(np.float64), want)  # the stated sum is an fp32 value
    bad = got != want32
    assert not bad.any(), (f"{bad.sum()} of {bad.size} outputs differ (plan {p}, budget 2^{np.log2(budget):.1f}); first at "
                           f"{np.argwhere(bad)[0]}: got {got[bad][0]!r} want {want32[bad][0]!r}")
    return got, p


def on_grid(w, a, rng, shape, units=2 ** 20):
    """fp32 addends that lie on the product grid of (a, w), |x| < units grid steps"""
    return (rng.integers(-units, units, shape) * 2.0 ** oracle.tc_grid(w.a_eff(a), w.w_eff)).astype(np.float32)


FORMATS = ([("s4", asym, st) for asym in (False, True) for st in ("f32", "bf16", "f16")] +
           [("s8", asym, st) for asym in (False, True) for st in ("f32", "bf16", "f16")] +
           [("nf4", False, "f32"), ("nf4", False, "bf16"), ("f4_bnb", False, "f32"), ("f4_bnb", False, "bf16"),
            ("f4_e2m1", False, "f32"), ("f4_e2m1", False, "bf16")])


@pytest.mark.parametrize("g", [32, 128, 1056])
@pytest.mark.parametrize("fmt,asym,stype", FORMATS)
def test_tc_exact_formats(fmt, asym, stype, g):
    """tier A: every BesTLA format and scale type the kernel takes, groups of 32, 128 and K (per channel), at K = 1056 (the last
    k block half full, the last 128-group a quarter), 65 tokens, 136 weight rows (a partial 128-row tile)"""
    w = xweight(fmt, 136, 1056, g, asym, stype, seed=g + 3 * asym)
    check_exact(w, w.act(65, seed=g))


@pytest.mark.parametrize("fmt,subnormal", [("q4_0", False), ("q4_0", True), ("q8_0", False), ("q8_0", True)])
def test_tc_exact_ggml(fmt, subnormal):
    """tier A: ggml Q4_0 / Q8_0 with fp16 d values off the bf16 grid (ties included), normal and subnormal"""
    w = xweight(fmt, 136, 1024, 32, seed=7 + subnormal, subnormal=subnormal)
    check_exact(w, w.act(65, seed=2))


@pytest.mark.parametrize("m", [1, 5, 17, 32, 33, 64, 65, 128, 129, 300])
def test_tc_exact_m_edges(m):
    """tier B: token tiles T = 32 / 64 / 128 at and across their edges (1 and 5 rows forced onto the kernel)"""
    w = xweight("s4", 136, 1056, 32, True, seed=11)
    check_exact(w, w.act(m, seed=m))


@pytest.mark.parametrize("n", [8, 127, 128, 129, 4097])
def test_tc_exact_n_edges(n):
    """tier B: weight-row tiles of 128 at and across their edges"""
    w = xweight("s8", n, 96, 32, True, seed=n)
    check_exact(w, w.act(33, seed=n))


@pytest.mark.parametrize("k,g", [(32, 32), (96, 32), (1056, 128), (1000, 1000), (11008, 128)])
def test_tc_exact_k_edges(k, g):
    """tier B: half a k block, a k block and a half, per-channel K = 1000 (kpad 1024 > K: the scalar conversion kernel zero-pads),
    Llama's 11008"""
    w = xweight("s4", 129, k, g, seed=k)
    check_exact(w, w.act(65, seed=k, dense=k == 32))


# (m, n, k) -> (T, S, k blocks per slice) on a 132-SM H100, from the launcher's arithmetic
SPLIT_CLASSES = {
    (2048, 4096, 4096): (128, 1, 64),    # enough tiles: one slice
    (100, 11008, 4096): (128, 1, 64),    # 86 tiles, just inside the 2/3 rule
    (40, 4096, 4096): (64, 4, 16),       # even split
    (17, 256, 4160): (32, 8, 9),         # last slice 2 blocks, fewer than the 6-stage packed ring
    (20, 512, 8192): (32, 16, 8),        # the 16-slice cap
    (300, 512, 11008): (128, 11, 16),    # last slice 12 blocks
}


def test_tc_split_classes_on_this_card():
    """the plan entry confirms that every split class of test_tc_exact_split occurs here"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    got = {shape: plan(*shape) for shape in SPLIT_CLASSES}
    if sms != 132:
        pytest.skip(f"the table is for 132 SMs, this card has {sms}: {got}")
    assert got == SPLIT_CLASSES
    assert plan(40, 4096, 4096, aliased=True)[1] == 1


@pytest.mark.parametrize("m,n,k", list(SPLIT_CLASSES))
def test_tc_exact_split(m, n, k):
    """tier B: every split class, exact whatever the slice count and the order of the atomics"""
    w = xweight("s4", n, k, 128, False, seed=n + k)
    _, p = check_exact(w, w.act(m, seed=m))
    assert p == plan(m, n, k)


@pytest.mark.parametrize("m,n,k", [(300, 4096, 1024), (40, 512, 4096)])
def test_tc_exact_epilogue(m, n, k):
    """tier B: broadcast bias, [m][ldo] bias and residual, each at one slice and at several (only slice 0 may add them)"""
    w = xweight("s4", n, k, 32, True, seed=5)
    a = w.act(m, seed=3)
    rng = np.random.default_rng(m)
    S = plan(m, n, k)[1]
    assert (S == 1) == (m == 300), S
    check_exact(w, a, bias=on_grid(w, a, rng, n), bcast=True)
    check_exact(w, a, bias=on_grid(w, a, rng, (m, n)))
    check_exact(w, a, residual=on_grid(w, a, rng, (m, n)))
    check_exact(w, a, bias=on_grid(w, a, rng, n), bcast=True, residual=on_grid(w, a, rng, (m, n)), ldo=n + 1)


def test_tc_exact_residual_in_place():
    """tier B: residual == dst keeps one slice at a shape that would otherwise split, and equals the aliased-free call"""
    m, n, k = 40, 512, 4096
    assert plan(m, n, k)[1] > 1 and plan(m, n, k, aliased=True)[1] == 1
    w = xweight("s4", n, k, 32, True, seed=5)
    a = w.act(m, seed=4)
    res = on_grid(w, a, np.random.default_rng(1), (m, n))
    split, _ = check_exact(w, a, residual=res)
    inplace, p = check_exact(w, a, residual=res, alias=True)
    assert p[1] == 1
    assert np.array_equal(split, inplace)


@pytest.mark.parametrize("how", ["lda", "offset", "shuffle"])
def test_tc_exact_conversion_kernels(how):
    """tier B: the scalar act_to_bf16_kernel (lda % 4 != 0, a misaligned activation pointer, an act-order gather) against the
    exact sum, and against the aligned 8-wide conversion on the same values, bit for bit"""
    m, n, k = 65, 136, 1024
    w = xweight("s4", n, k, 128, True, seed=9, shuffle=how == "shuffle")
    a = w.act(m, seed=6)
    got, _ = check_exact(w, a, lda=k + 1 if how == "lda" else None, offset=how == "offset")
    if how != "shuffle":
        assert np.array_equal(got, run(w.w, a))


# ----------------------------------------------------------------------------------------------------------- random data (C)
@pytest.mark.parametrize("dist", ["uniform", "normal"])
@pytest.mark.parametrize("m,n,k", [(2048, 4096, 4096), (512, 4096, 11008)])
def test_tc_random_bar(m, n, k, dist):
    """tier C: Llama-2-7B prefill shapes, int4 g128 weights, |got - sum a_eff w_eff| <= (ceil(K/16) + S) 2^-22 sum |a_eff w_eff|.
    The constant assumes one truncation per k16 MMA and one rounding per slice; it is not a measurement.  Largest measured ratio
    0.0103 (normal data at 2048 x 4096 x 4096; uniform 0.0078, K = 11008: 0.0050 / 0.0060), NVIDIA H100 80GB HBM3 at a 700 W
    power limit."""
    rng = np.random.default_rng(k + (dist == "normal"))
    draw = (lambda s: rng.uniform(-0.5, 0.5, s)) if dist == "uniform" else (lambda s: rng.normal(0, 1, s))
    w = draw((k, n)).astype(np.float32)
    a = draw((m, k)).astype(np.float32)
    q, sc, zp = oracle.btla_quantize(w, 128, 4, False)
    wd = ns.Weight.from_unpacked(q, sc, zp, 128, ns.W_S4, ns.S_F32, ns.COMP_INT8)
    got = run(wd, a)
    a_eff, w_eff = oracle.tc_operands(a, "s4", q, sc, zp, 128)
    ratio = c_bar_ratio(got, a_eff, w_eff, plan(m, n, k)[1])
    print(f"C-bar ratio {dist} {m}x{n}x{k}: {ratio:.4f}")
    assert ratio <= 1, ratio


# ----------------------------------------------------------------------------------------------------------- invariants (D)
def test_tc_row_permutation_and_repeat():
    """tier D: at one slice an output row depends on its own activation row only, whatever its place in the token tile, and
    repeated launches are identical"""
    m, n, k = 300, 4096, 1024
    assert plan(m, n, k)[1] == 1
    rng = np.random.default_rng(12)
    q = rng.integers(-8, 8, (k, n)).astype(np.int8)
    sc = rng.uniform(0.005, 0.02, (k // 32, n)).astype(np.float32)
    wd = ns.Weight.from_unpacked(q, sc, None, 32, ns.W_S4, ns.S_F32, ns.COMP_INT8)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    got = run(wd, a)
    perm = rng.permutation(m)
    assert np.array_equal(run(wd, a[perm]), got[perm])
    assert np.array_equal(run(wd, a), got)


# ----------------------------------------------------------------------------------------------------------- one-image FFN (E)
def test_ffn_one_image_vs_two_step():
    """tier E: the eval step's prompt FFN (ns_ffn_silu_engine_image: silu(g) * u straight into the down projection's bf16 image)
    against ns_ffn_silu (fp32 product, then the 8-wide conversion): identical without a residual, the fp32 sum with one; and the
    down projection against fp64 on that image within the C bar"""
    m, e, f = 2048, 1024, 2048
    assert plan(m, f, e)[1] == 1 and plan(m, e, f)[1] == 1
    rng = np.random.default_rng(21)

    def weight(n, k):
        q = rng.integers(-8, 8, (k, n)).astype(np.int8)
        sc = rng.uniform(0.01, 0.03, (k // 128, n)).astype(np.float32)
        return ns.Weight.from_unpacked(q, sc, None, 128, ns.W_S4, ns.S_F32, ns.COMP_INT8), q, sc

    (w1, _, _), (w3, _, _), (w2, q2, sc2) = weight(f, e), weight(f, e), weight(e, f)
    x = torch.from_numpy(rng.uniform(-1, 1, (m, e)).astype(np.float32)).cuda()
    res = torch.from_numpy(rng.normal(0, 1, (m, e)).astype(np.float32)).cuda()
    L = ns.lib()

    def call(fn, *extra):
        tmp = torch.full((2, m, f), float("nan"), device="cuda")
        out = torch.full((m, e), float("nan"), device="cuda")
        torch.cuda.synchronize()
        lc = L.ns_launch_count()
        rc = fn(w1.h, w2.h, w3.h, C.c_void_p(x.data_ptr()), e, C.c_void_p(tmp.data_ptr()), C.c_void_p(out.data_ptr()), e, m,
                *extra, None, None)
        torch.cuda.synchronize()
        assert rc == 0, ns.last_error()
        return out.cpu().numpy(), tmp.cpu().numpy(), L.ns_launch_count() - lc

    two, tmp, n2 = call(L.ns_ffn_silu)
    one, _, n1 = call(L.ns_ffn_silu_engine_image, None)
    one_r, _, _ = call(L.ns_ffn_silu_engine_image, C.c_void_p(res.data_ptr()))
    assert (n2, n1) == (6, 5), (n2, n1)  # image, gate, up, product, image, down / image, gate, up, product image, down
    assert np.array_equal(one, two)
    assert np.array_equal(one_r, two + res.cpu().numpy())
    a_eff, w_eff = oracle.tc_operands(tmp[0], "s4", q2, sc2, None, 128)  # tmp[0] = the two-step's fp32 product
    ratio = c_bar_ratio(one, a_eff, w_eff, 1)
    print(f"C-bar ratio one-image FFN down projection: {ratio:.4f}")
    assert ratio <= 1, ratio

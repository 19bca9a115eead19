"""The register-staged GEMV (`gemv_kernel<WFMT, AMODE, M, ASYM>`, csrc/gemv.cu) on its own, through the public entries: NF4 and
the FP4 codebooks, int8 weights and float compute types, against the kernel's stated arithmetic (DESIGN.md section 4).

Stated arithmetic:
  float modes    y = sum_k a_eff[k] * w_eff[k], fp32 FMAs; a_eff = a (F32 compute) or bf16(a) (BF16 compute, rounded by the
                 activation copy), w_eff = fp32((q - zp) * s) or fp32(level[q] * s), s rounded to its storage type
  integer modes  exact integer sums per 32-chunk of the reference's quantised activations (u8 asym / s8), fp32 fma with
                 a_scale * w_scale
Bars:
  1. row invariance, bit-exact: an output row depends on its weight row and its own activation only, so every row equals the
     same row computed by an m = 1 plain call, whatever the tile, template M, pair partner, fused mode, lda / ldo or entry.
     Epilogues are that value plus fp32 adds / products.
  2. exact constructions, bit-exact against fp64: dyadic activations and power-of-two scales make every product and partial sum
     exact in fp32; activations off the bf16 grid give F32 and BF16 compute two different exact results.
  3. random data: |got - model| <= oracle.GEMV_F32_C * sqrt(K) * 2^-24 * sum_k |a_eff w_eff| per element (C_INT for integer
     modes), the model in fp64.
  4. SiLU / GELU: within ELT_ULPS fp32 ulps of the fp32 function of the GPU's own pre-activation.
Every case pins its path by launch count: act_prep + GEMV = 2 launches per tile of 4, 2 or 1 rows.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import neural_speed_b200 as ns
import oracle

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

E_UNSUPPORTED = -4
# Integer modes against the fp64 value of the block sums (only the fp32 accumulation of 32-chunks rounds).  Measured on an H100
# 80GB HBM3 (700 W limit): at most 0.0067.
C_INT = 0.03
# SiLU / GELU epilogues, in fp32 ulps of the function's operand scale (|silu(x)|, 0.5 |x| (1 + |tanh|)).  Measured: 3.
ELT_ULPS = 6
FLOAT = (ns.COMP_F32, ns.COMP_BF16)


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def counted(fn):
    torch.cuda.synchronize()
    lc = ns.lib().ns_launch_count()
    rc = fn()
    ns.lib().bestla_device_sync(None)
    return rc, ns.lib().ns_launch_count() - lc


def bf16(x):
    return oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(np.asarray(x, np.float32)))


def round_scale(sc, stype):
    """the scale as the device stores it (repack.cu: RNE to bf16 / fp16)"""
    if stype == ns.S_BF16:
        return bf16(sc)
    if stype == ns.S_F16:
        return sc.astype(np.float16).astype(np.float32)
    return sc


def tile_rows(k, comp):
    """rows of one GEMV tile (ns_gemv_tile_rows): the activation rows staged in shared memory"""
    kpad = -(-k // 32) * 32
    if comp in FLOAT:
        per_row, cap = kpad * 4, 96 * 1024
    else:
        per_row, cap = -(-kpad // 1024) * 1024 + -(-(kpad // 32) // 2) * 2 * 8, 64 * 1024
    mt = 4
    while mt > 1 and per_row * mt > cap:
        mt //= 2
    return mt


class W:
    """a device weight with the host data of its stated arithmetic"""

    def __init__(self, fmt, comp, n, k, g, asym=False, stype=ns.S_F32, seed=0, exact=False, shuffle=False, unit_scales=False):
        rng = np.random.default_rng(seed)
        self.fmt, self.comp, self.n, self.k, self.g = fmt, comp, n, k, g
        self.tile = tile_rows(k, comp)
        self.perm = rng.permutation(k).astype(np.int32) if shuffle else None
        nb = -(-k // g)
        if fmt.startswith("fp4"):  # F4 codebooks: quantised blobs; levels x scales from the host unpacker
            wt = rng.uniform(-0.5, 0.5, (n, k)).astype(np.float32)
            blob = ns.np_bestla_quantize(wt, fmt, g, "sym", "bf16" if stype == ns.S_BF16 else "fp32",
                                         "bf16" if comp == ns.COMP_BF16 else "fp32")
            self.w = ns.Weight.from_blob(blob)
            self._weff = ns.unpack_blob(blob, n, k)
            self.q = None
        else:
            lo, hi = {"s4": (-8, 8), "s8": (-16, 16) if exact else (-128, 128), "nf4": (0, 16)}[fmt]
            self.q = rng.integers(lo, hi, (k, n), dtype=np.int8)
            self.zp = None
            if asym:
                zlo, zhi = (-4, 4) if fmt == "s4" else (-8, 8) if exact else (-32, 32)
                self.zp = rng.integers(zlo, zhi, (nb, n), dtype=np.int8)
            if unit_scales:
                sc = np.ones((nb, n), np.float32)
            elif exact:
                sc = (2.0 ** -rng.integers(0, 3, (nb, n))).astype(np.float32)
            else:
                sc = rng.uniform(0.5, 1.5, (nb, n)).astype(np.float32) / 16
            self.sc = round_scale(sc, stype)
            wfmt = {"s4": ns.W_S4, "s8": ns.W_S8, "nf4": ns.W_NF4}[fmt]
            self.w = ns.Weight.from_unpacked(self.q, sc, self.zp, g, wfmt, stype, comp, shuffle=self.perm)
            self._weff = None
        assert self.w.comp == comp

    def weff(self, cols=None):
        """w_eff [K, N] (or the given columns): fp32 (q - zp) * s or level * s, as oracle.btla_dequant / BTLAGemmUnPackB"""
        if self._weff is not None:
            return self._weff if cols is None else self._weff[:, cols]
        if cols is None:
            if not hasattr(self, "_full"):
                self._full = oracle.btla_dequant(self.q, self.sc, self.zp, self.g, nf4=self.fmt == "nf4")
            return self._full
        return oracle.btla_dequant(np.ascontiguousarray(self.q[:, cols]), np.ascontiguousarray(self.sc[:, cols]),
                                   None if self.zp is None else np.ascontiguousarray(self.zp[:, cols]), self.g,
                                   nf4=self.fmt == "nf4")

    def a_eff(self, a):
        """the activations the kernel multiplies: gathered by the act-order permutation, bf16-rounded for bf16 compute"""
        a = a if self.perm is None else a[:, self.perm]
        return bf16(a) if self.comp == ns.COMP_BF16 else np.asarray(a, np.float32)

    def model(self, a, cols=None):
        """(fp64 model, sum |terms|) of the stated arithmetic: float modes, or the integer modes' dequantised block operands"""
        if self.comp in FLOAT:
            return oracle.gemv_stated(self.a_eff(a), self.weff(cols))
        return oracle.gemv_stated(self.a_deq(a), self.weff(cols))

    def a_deq(self, a):
        """integer modes: the reference's quantised activation (a8 - za) * a_scale, exact in fp64"""
        a = np.ascontiguousarray(a, np.float32)
        g, k = self.g, self.k
        if self.comp == ns.COMP_INT8:
            a8, asc, azp = oracle.btla_quantize_act_u8(a, g)
            codes = a8.astype(np.float64) - np.repeat(azp, g, 1)[:, :k]
        else:
            a8, asc = oracle.btla_quantize_act_s8(a, g)
            codes = a8.astype(np.float64)
        return codes * np.repeat(asc.astype(np.float64), g, 1)[:, :k]


@functools.lru_cache(maxsize=None)
def weight(*args, **kw):
    return W(*args, **kw)


def mm(w, a, lda=None, ldo=None, bias=None, bcast=False, residual=None):
    """ns.mul_mat on the GEMV tiles; NaN sentinels in the skipped activation and output columns; the launch count pins the path"""
    m, k = a.shape
    lda, ldo = lda or k, ldo or w.n
    abuf = np.full((m, lda), np.nan, np.float32)
    abuf[:, :k] = a
    x = dev(abuf)
    out = torch.full((m, ldo), float("nan"), device="cuda")
    b = dev(bias) if bias is not None else None
    r = dev(residual) if residual is not None else None
    _, n = counted(lambda: ns.mul_mat(w.w, x.data_ptr(), lda, out.data_ptr(), ldo, m, b.data_ptr() if b is not None else None,
                                      r.data_ptr() if r is not None else None, ns.MM_BIAS_BCAST if bcast else 0))
    assert n == 2 * -(-m // w.tile), n
    o = out.cpu().numpy()
    assert np.isnan(o[:, w.n:]).all()
    return o[:, :w.n]


def rows1(w, a):
    """every row computed alone: the reference of bar 1"""
    return np.concatenate([mm(w, a[i:i + 1]) for i in range(a.shape[0])])


def check_bar(w, got, a, cols=None):
    want, mag = w.model(a, cols)
    c = oracle.GEMV_F32_C if w.comp in FLOAT else C_INT
    ratio = (np.abs(got.astype(np.float64) - want) / (np.sqrt(w.k) * 2.0 ** -24 * np.maximum(mag, 1e-30))).max()
    print(f"bar ratio {w.fmt} comp={w.comp} k={w.k}: {ratio:.4f}")
    assert ratio <= c, ratio


def rand_act(m, k, seed):
    return np.random.default_rng(seed).uniform(-0.5, 0.5, (m, k)).astype(np.float32)


# ------------------------------------------------------------------------------------------ random data, row invariance
# (fmt, comp, asym, stype, group (0: K), k, ms); n = 203: the last pair is half valid
CASES = [
    ("s4", ns.COMP_F32, False, ns.S_F32, 32, 1000, (1, 3, 5)),
    ("s4", ns.COMP_F32, True, ns.S_BF16, 64, 4128, (2, 7)),
    ("s4", ns.COMP_BF16, True, ns.S_F16, 128, 4096, (4, 8)),
    ("s4", ns.COMP_BF16, False, ns.S_F32, 0, 1000, (13,)),
    ("nf4", ns.COMP_F32, False, ns.S_F16, 256, 4096, (1, 16)),
    ("nf4", ns.COMP_BF16, False, ns.S_BF16, 32, 4128, (3, 5)),
    ("fp4_bnb", ns.COMP_F32, False, ns.S_F32, 32, 1024, (1, 7)),
    ("fp4_bnb", ns.COMP_BF16, False, ns.S_BF16, 128, 4096, (2, 13)),
    ("fp4_e2m1", ns.COMP_F32, False, ns.S_BF16, 128, 4096, (4, 5)),
    ("fp4_e2m1", ns.COMP_BF16, False, ns.S_F32, 32, 1024, (1, 16)),
    ("s8", ns.COMP_F32, False, ns.S_F32, 128, 4128, (1, 5)),
    ("s8", ns.COMP_F32, True, ns.S_F16, 0, 1000, (3, 8)),
    ("s8", ns.COMP_BF16, True, ns.S_BF16, 64, 4096, (2, 7)),
    ("s8", ns.COMP_INT8, True, ns.S_F32, 128, 4096, (1, 5)),
    ("s8", ns.COMP_INT8, False, ns.S_BF16, 32, 1000, (4, 13)),
    ("s8", ns.COMP_INT8_S8, True, ns.S_F32, 256, 4096, (2, 16)),
    ("s8", ns.COMP_INT8_S8, False, ns.S_F16, 0, 4128, (3, 7)),
]


@pytest.mark.parametrize("fmt,comp,asym,stype,g,k,ms", CASES)
def test_random_against_stated_model(fmt, comp, asym, stype, g, k, ms):
    n = 203
    w = weight(fmt, comp, n, k, g or k, asym, stype, seed=k + n)
    for m in ms:
        a = rand_act(m, k, 10 * m + k)
        got = mm(w, a, lda=k + 33, ldo=n + 3)
        assert np.array_equal(got, rows1(w, a))
        check_bar(w, got, a)


@pytest.mark.parametrize("fmt,comp,k,n,g,tile", [("s4", ns.COMP_F32, 11008, 11008, 128, 2),
                                                 ("nf4", ns.COMP_BF16, 28672, 4400, 128, 1)])
def test_several_pairs_per_warp(fmt, comp, k, n, g, tile):
    """n past 2 x (warps in the grid): warps reload batch 0 for their later pairs (two CTAs per SM at K = 11008, one at 28672)"""
    w = weight(fmt, comp, n, k, g, False, ns.S_F32, seed=3)
    assert w.tile == tile
    cols = np.array(sorted(set(range(0, n, 29)) | {2111, 2112, 2113, 4223, 4224, 4225, n - 2, n - 1}), np.int64)
    cols = cols[cols < n]
    for m in (1, 3, 5):
        a = rand_act(m, k, m)
        got = mm(w, a)
        if m > 1:
            assert np.array_equal(got, rows1(w, a))
        check_bar(w, got[:, cols], a, cols)


@pytest.mark.parametrize("comp", FLOAT)
def test_act_order_shuffle(comp):
    k, n, g, m = 1024, 203, 128, 7
    w = weight("s4", comp, n, k, g, True, ns.S_F32, seed=5, shuffle=True)
    a = rand_act(m, k, 77)
    got = mm(w, a, lda=k + 8)
    assert np.array_equal(got, rows1(w, a))
    check_bar(w, got, a)


# ------------------------------------------------------------------------------------------------- exact constructions
def exact_float_act(m, k, seed):
    return (np.random.default_rng(seed).integers(-8, 9, (m, k)) / 8).astype(np.float32)


def exact_int_act(m, k, g, comp, seed):
    """integers x 2^-6 with every quantisation block's range pinned, so the activation scale is exactly 2^-6"""
    lo = -128 if comp == ns.COMP_INT8 else -127
    ints = np.random.default_rng(seed).integers(lo, 128, (m, k))
    ints[:, ::g] = 127
    if comp == ns.COMP_INT8:
        ints[:, 1::g] = -128
    return (ints * 2.0 ** -6).astype(np.float32)


def assert_exact_in_fp32(a_eff, w_eff, grid):
    """every partial sum of the dot products is a multiple of grid below 2^24 grid: fp32 represents each one exactly"""
    _, mag = oracle.gemv_stated(a_eff, w_eff)
    assert mag.max() < 2.0 ** 24 * grid


EXACT = [("s4", ns.COMP_F32, False, 32, 1000), ("s4", ns.COMP_F32, True, 64, 4128), ("s4", ns.COMP_BF16, False, 128, 4128),
         ("s4", ns.COMP_BF16, True, 0, 1000), ("s8", ns.COMP_F32, True, 256, 4128), ("s8", ns.COMP_F32, False, 0, 4128),
         ("s8", ns.COMP_BF16, True, 32, 1000), ("s8", ns.COMP_BF16, False, 64, 4128), ("s8", ns.COMP_INT8, True, 128, 4128),
         ("s8", ns.COMP_INT8, False, 32, 1000), ("s8", ns.COMP_INT8, True, 256, 4128), ("s8", ns.COMP_INT8_S8, True, 64, 1000),
         ("s8", ns.COMP_INT8_S8, False, 0, 4128)]


@pytest.mark.parametrize("fmt,comp,asym,g,k", EXACT)
def test_exact_dyadic(fmt, comp, asym, g, k):
    n, m, g = 67, 5, g or k
    w = weight(fmt, comp, n, k, g, asym, ns.S_F32, seed=k + g, exact=True)
    if comp in FLOAT:
        a = exact_float_act(m, k, g)
        a_eff, grid = w.a_eff(a), 2.0 ** -3 * 2.0 ** -2
    else:
        a = exact_int_act(m, k, g, comp, g)
        a_eff, grid = w.a_deq(a), 2.0 ** -6 * 2.0 ** -2
        assert np.array_equal(a_eff, a)  # the quantiser kept every value
    assert_exact_in_fp32(a_eff, w.weff(), grid)
    want, _ = oracle.gemv_stated(a_eff, w.weff())
    got = mm(w, a, ldo=n + 1)
    assert np.array_equal(got, want.astype(np.float32))
    if comp == ns.COMP_INT8:
        a8, asc, azp = oracle.btla_quantize_act_u8(a, g)
        assert np.array_equal(got, oracle.btla_gemv_u8s8(a8, asc, azp, w.q, w.sc, w.zp, g, blocksum=True))


@pytest.mark.parametrize("fmt,asym", [("s4", True), ("s8", False), ("s8", True)])
def test_bf16_rounding_is_exact(fmt, asym):
    """activations +-(j + 2^-8), j in {1, 2}: bf16 rounds them to +-j, so F32 and BF16 compute have two different exact results"""
    n, k, g, m = 67, 1000, 128, 3
    rng = np.random.default_rng(8)
    a = (rng.choice([-1, 1], (m, k)) * (rng.integers(1, 3, (m, k)) + 2.0 ** -8)).astype(np.float32)
    wants = {}
    for comp in FLOAT:
        w = weight(fmt, comp, n, k, g, asym, ns.S_F32, seed=9, exact=True, unit_scales=True)
        a_eff = w.a_eff(a)
        assert_exact_in_fp32(a_eff, w.weff(), 2.0 ** -8)
        wants[comp], _ = oracle.gemv_stated(a_eff, w.weff())
        assert np.array_equal(mm(w, a), wants[comp].astype(np.float32))
    assert (wants[ns.COMP_F32] != wants[ns.COMP_BF16]).mean() > 0.9


# ------------------------------------------------------------------------------------------------------------- epilogues
@pytest.mark.parametrize("fmt,comp", [("s8", ns.COMP_F32), ("nf4", ns.COMP_BF16), ("s8", ns.COMP_INT8)])
def test_bias_and_residual(fmt, comp):
    n, k, m = 203, 1000, 7  # per-row biases past the first tile
    w = weight(fmt, comp, n, k, 64, False, ns.S_F32, seed=11)
    rng = np.random.default_rng(12)
    a = rand_act(m, k, 13)
    plain = rows1(w, a)
    ldo = n + 5
    bias_row = rng.uniform(-1, 1, (m, ldo)).astype(np.float32)
    bias_b = rng.uniform(-1, 1, n).astype(np.float32)
    res = rng.uniform(-1, 1, (m, ldo)).astype(np.float32)
    f = np.float32
    assert np.array_equal(mm(w, a, ldo=ldo, bias=bias_b, bcast=True), plain + bias_b)
    assert np.array_equal(mm(w, a, ldo=ldo, bias=bias_row), plain + bias_row[:, :n])
    assert np.array_equal(mm(w, a, ldo=ldo, residual=res), plain + res[:, :n])
    both = mm(w, a, ldo=ldo, bias=bias_row, residual=res)
    assert both.dtype == f and np.array_equal(both, (plain + bias_row[:, :n]) + res[:, :n])
    assert np.array_equal(mm(w, a, ldo=ldo, bias=bias_b, bcast=True, residual=res), (plain + bias_b) + res[:, :n])


def gelu_f32(x):
    """the tanh GELU in fp32 (kernel_ref.h:1570; ns_gelu), and the operand scale its ulp bar is measured in"""
    x = np.asarray(x, np.float32)
    t = np.tanh(np.float32(0.7978845834732056) * (x + np.float32(0.044714998453855515) * x * x * x))
    return np.float32(0.5) * x * (np.float32(1) + t), 0.5 * np.abs(x) * (1 + np.abs(t))


def silu_f32(x):
    y = np.array([oracle.lib().orc_silu(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32).reshape(np.shape(x))
    return y, np.abs(y)


def assert_ulps(got, want, scale, ulps=ELT_ULPS):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    bar = np.spacing(np.maximum(np.asarray(scale, np.float32), np.float32(1e-30)))
    print(f"epilogue ulps {(err / bar).max():.2f}")
    assert (err <= ulps * bar).all(), (err / bar).max()


FFN = [("nf4", ns.COMP_BF16, 1000), ("s8", ns.COMP_INT8, 1000), ("s4", ns.COMP_F32, 4128)]


@pytest.mark.parametrize("fmt,comp,k", FFN)
@pytest.mark.parametrize("m", [1, 7])
@pytest.mark.parametrize("biases", [False, True])
def test_ffn_gelu_plain_epilogue(fmt, comp, k, m, biases):
    """ns_ffn_gelu without w3: tmp = gelu(x W1^T [+ b1]) in the GEMV epilogue, dst = tmp W2^T [+ b2]"""
    fmid, n = 130, 203
    w1, w2 = weight(fmt, comp, fmid, k, 32, False, ns.S_F32, seed=21), weight(fmt, comp, n, fmid, 32, False, ns.S_F32, seed=22)
    rng = np.random.default_rng(23)
    a = rand_act(m, k, 24)
    b1 = rng.uniform(-1, 1, fmid).astype(np.float32) if biases else None
    b2 = rng.uniform(-1, 1, n).astype(np.float32) if biases else None
    x, tmp, out = dev(a), torch.full((m, fmid), float("nan"), device="cuda"), torch.full((m, n), float("nan"), device="cuda")
    d1, d2 = (dev(b1), dev(b2)) if biases else (None, None)
    _, nl = counted(lambda: ns.ffn_gelu(w1.w, w2.w, None, d1.data_ptr() if biases else None, d2.data_ptr() if biases else None, 1,
                                        x.data_ptr(), k, tmp.data_ptr(), out.data_ptr(), n, m))
    assert nl == 2 * -(-m // w1.tile) + 2 * -(-m // w2.tile), nl
    t = tmp.cpu().numpy()
    pre = rows1(w1, a) + (b1 if biases else np.float32(0))
    want, scale = gelu_f32(pre)
    assert_ulps(t, want, scale)
    assert np.array_equal(out.cpu().numpy(), mm(w2, t, bias=b2, bcast=True))


@pytest.mark.parametrize("fmt,comp,k", FFN)
@pytest.mark.parametrize("m", [1, 7])
@pytest.mark.parametrize("gelu", [False, True])
def test_ffn_gate_up(fmt, comp, k, m, gelu):
    """ns_ffn_silu / ns_ffn_gelu with w3: tmp = elt(gate) * up from one gate/up launch per tile, dst = tmp W2^T"""
    fmid, n = 131, 203
    w1, w3 = weight(fmt, comp, fmid, k, 32, False, ns.S_F32, seed=31), weight(fmt, comp, fmid, k, 32, False, ns.S_F32, seed=32)
    w2 = weight(fmt, comp, n, fmid, 32, False, ns.S_F32, seed=33)
    a = rand_act(m, k, 34)
    x = dev(a)
    tmp, out = torch.full((2 * m * fmid,), float("nan"), device="cuda"), torch.full((m, n), float("nan"), device="cuda")
    if gelu:
        fn = lambda: ns.ffn_gelu(w1.w, w2.w, w3.w, None, None, 0, x.data_ptr(), k, tmp.data_ptr(), out.data_ptr(), n, m)
    else:
        fn = lambda: ns.ffn_silu(w1.w, w2.w, w3.w, x.data_ptr(), k, tmp.data_ptr(), out.data_ptr(), n, m)
    _, nl = counted(fn)
    assert nl == 2 * -(-m // w1.tile) + 2 * -(-m // w2.tile), nl
    t = tmp.cpu().numpy()[:m * fmid].reshape(m, fmid)
    g, up = rows1(w1, a), rows1(w3, a)
    sg, scale = gelu_f32(g) if gelu else silu_f32(g)
    assert_ulps(t, sg * up, scale * np.abs(up))
    assert np.array_equal(out.cpu().numpy(), mm(w2, t))


@pytest.mark.parametrize("fmt,comp,k,m", [("nf4", ns.COMP_F32, 1000, 3), ("s8", ns.COMP_INT8, 4128, 4), ("s4", ns.COMP_BF16, 1000, 2),
                                          ("fp4_e2m1", ns.COMP_BF16, 1024, 4)])
def test_gate_up_writes_aux(fmt, comp, k, m):
    """one prepared gate/up launch: aux = silu(gate) within ELT_ULPS of orc_silu, dst = fp32(aux * up) exactly"""
    fmid = 131
    w1, w3 = weight(fmt, comp, fmid, k, 32, False, ns.S_F32, seed=41), weight(fmt, comp, fmid, k, 32, False, ns.S_F32, seed=42)
    a = rand_act(m, k, 43)
    L = ns.lib()
    x = dev(a)
    ws = torch.zeros(L.ns_device_workspace_bytes(m, k) // 4 + 64, device="cuda")
    dst, aux = torch.full((m, fmid + 1), float("nan"), device="cuda"), torch.full((m, fmid + 1), float("nan"), device="cuda")
    wl = (C.c_void_p * 2)(w1.w.h, w3.w.h)

    def run():
        assert L.ns_prepare_activation(w1.w.h, ptr(x), k, m, ptr(ws), None) == 0, ns.last_error()
        assert L.ns_matmul_prepared(wl, 2, 2, ptr(ws), ptr(dst), fmid + 1, m, None, 0, None, ptr(aux), None) == 0, ns.last_error()
    assert counted(run)[1] == 2
    d, s = dst.cpu().numpy(), aux.cpu().numpy()
    assert np.isnan(d[:, fmid]).all() and np.isnan(s[:, fmid]).all()
    d, s = d[:, :fmid], s[:, :fmid]
    want, scale = silu_f32(rows1(w1, a))
    assert_ulps(s, want, scale)
    assert np.array_equal(d, s * rows1(w3, a))


@pytest.mark.parametrize("fmt,comp,k", [("nf4", ns.COMP_BF16, 1000), ("s8", ns.COMP_INT8, 4128), ("s4", ns.COMP_F32, 1000),
                                        ("fp4_bnb", ns.COMP_F32, 1024)])
@pytest.mark.parametrize("m", [1, 7])
def test_qkv_concat(fmt, comp, k, m):
    """ns_mul_qkv: one launch per tile over n_q + n_k + n_v rows, dst = [3][m][ldo]; n_v odd (the last pair half valid)"""
    ns_, ldo = (130, 130, 67), 133
    ws = [weight(fmt, comp, nn, k, 32, False, ns.S_F32, seed=50 + i) for i, nn in enumerate(ns_)]
    a = rand_act(m, k, 51)
    x = dev(a)
    out = torch.full((3, m, ldo), float("nan"), device="cuda")
    _, nl = counted(lambda: ns.mul_qkv(ws[0].w, ws[1].w, ws[2].w, x.data_ptr(), k, out.data_ptr(), ldo, m))
    assert nl == 2 * -(-m // ws[0].tile), nl
    o = out.cpu().numpy()
    for i, w in enumerate(ws):
        assert np.isnan(o[i, :, w.n:]).all()
        assert np.array_equal(o[i, :, :w.n], rows1(w, a)), i


@pytest.mark.parametrize("fmt,comp", [("nf4", ns.COMP_BF16), ("s8", ns.COMP_INT8), ("s8", ns.COMP_F32)])
@pytest.mark.parametrize("m", [5, 16])
def test_mul_mat_id(fmt, comp, m):
    """grouped expert ids (no gather / scatter): each expert's slice runs its own GEMV tiles; rows equal the expert's plain call"""
    n, k = 203, 1000
    experts = [weight(fmt, comp, n, k, 64, True if fmt == "s8" else False, ns.S_F32, seed=60 + e) for e in range(2)]
    c0 = (m + 1) // 2
    ids = np.array([[0]] * c0 + [[1]] * (m - c0), np.int32)
    a = rand_act(m, k, 61)
    x = dev(a)
    out = torch.full((m, n), float("nan"), device="cuda")
    _, nl = counted(lambda: ns.mul_mat_id([e.w for e in experts], ids, 0, x.data_ptr(), k, out.data_ptr(), n, m))
    assert nl == 2 * -(-c0 // experts[0].tile) + 2 * -(-(m - c0) // experts[1].tile), nl
    o = out.cpu().numpy()
    assert np.array_equal(o[:c0], rows1(experts[0], a[:c0]))
    assert np.array_equal(o[c0:], rows1(experts[1], a[c0:]))


# ------------------------------------------------------------------------------------------------------------ largest K
@pytest.mark.parametrize("fmt,comp", [("nf4", ns.COMP_F32), ("s8", ns.COMP_BF16)])
def test_longest_float_row(fmt, comp):
    """a float-mode tile stages K fp32 values per row in at most 200 KB of shared memory: K = 51200 runs, longer rows are refused
    before anything is launched"""
    n, L = 8, ns.lib()
    w = W(fmt, comp, n, 51200, 128, seed=70)
    assert w.tile == 1
    a = rand_act(1, 51200, 71)
    check_bar(w, mm(w, a), a)
    long = W(fmt, comp, n, 51232, 128, seed=72)
    x, out = dev(rand_act(1, 51232, 73)), torch.zeros((1, n), device="cuda")
    rc, nl = counted(lambda: L.ns_mul_mat(long.w.h, ptr(x), 51232, ptr(out), n, 1, None, None, 0, None, None))
    assert (rc, nl) == (E_UNSUPPORTED, 0), ns.last_error()
    assert "shared memory" in ns.last_error()
    rc, nl = counted(lambda: L.ns_mul_mat(long.w.h, ptr(x), 51232, ptr(out), n, 1, None, None, ns.MM_FORCE_GEMV, None, None))
    assert (rc, nl) == (E_UNSUPPORTED, 0)

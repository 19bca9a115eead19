"""Batched decode (3..32 activation rows) on the integer tensor cores (csrc/gemm_imma.cu) against the CPU oracle.

The reference runs M > 4 through its int8 GEMM cores (bestla_wrapper.h:214-350): activations quantised per K-block
(kernel_ref.h:1825 / :1886, quantize_row_q8_0 for ggml weights), exact integer block dots, fp32 accumulation of the scaled
block sums -- the oracle functions used for the M <= 4 GEMV describe exactly that arithmetic, so the bar is the same 1e-4
(fp32 summation order is the only freedom), and the results must agree with the forced-GEMV path of the library itself.

The second half holds the kernel to its stated arithmetic (oracle.imma_stated, DESIGN.md section 4): per (row, output, activation
block b) an exact integer isum_b = sum (a - za)(q - zp), c_b = fp32(a_scale_b * w_scale_b), t_b = isum_b * c_b.
Bars:
  1. exact constructions (power-of-two scales, small integers; each case asserts sum |t_b| < 2^24 of the smallest unit, so every
     fp32 partial sum is exact): bit-exact against sum t_b, whatever the split count and summation order.
  2. random data: |got - sum t_b| <= gamma_n sum |t_b| per element, n = blocks + 16 (one fma per block, at most 16 split
     partials).  Measured on an H100 80GB HBM3 (700 W limit): largest ratio 0.14 of that bound.
  3. row invariance, bit-exact within one token-tile class (m in 3..8, 9..16, 17..32: the split count depends on the class).
  4. epilogues as fp32 operations on the plain result of the same plan; GELU / SiLU within ELT_ULPS of the fp32 function.
Every case pins its path by launch count: activation image + matmul = 2 launches per integer tensor-core call."""
import ctypes as C
import functools
import itertools

import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
import oracle

pytestmark = pytest.mark.gpu


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
    lc = ns.lib().ns_launch_count()
    ns.mul_mat(w, a.data_ptr(), k, out.data_ptr(), w.n, m, b.data_ptr() if b is not None else None,
               r.data_ptr() if r is not None else None, flags)
    sync()
    return out.cpu().numpy(), ns.lib().ns_launch_count() - lc


def close(got, want, rtol=1e-4):
    scale = float(np.abs(want).max()) + 1e-30
    np.testing.assert_allclose(got, want, rtol=rtol, atol=rtol * scale)


@pytest.mark.parametrize("n,k,m", [(128, 512, 8), (4096, 4096, 8), (4096, 4096, 32), (1000, 11008, 16), (257, 1024, 5), (96, 4096, 13),
                                   (4096, 11008, 27), (300, 14336, 32), (32000, 4096, 8), (4096, 4096, 3), (640, 11008, 4)])
def test_q4_0_batch_vs_oracle(n, k, m):
    """ggml Q4_0 x Q8_0: row counts off the 8/16/32 tiles, n off the 128-row tile, K = 11008 (43 slices: uneven K splits)"""
    rng = np.random.default_rng(300 + n + m)
    w = rng.normal(0, 0.02, (n, k)).astype(np.float32)
    a = rng.normal(0, 1.0, (m, k)).astype(np.float32)
    rows = oracle.quantize_q4_0(w)
    want = oracle.mul_mat_q4_0_f32(rows, a)
    wd = ns.Weight.from_q4_0_host(rows, n, k)
    got, launches = run_mul_mat(wd, a)
    assert launches == 2, launches            # activation image + one matmul: the weights are read once
    close(got, want)
    ref, _ = run_mul_mat(wd, a, flags=ns.MM_FORCE_GEMV)
    close(got, ref, 2e-6)                     # same block sums, different fp32 summation order
    for i in range(m):
        assert oracle.argmax(got[i]) == oracle.argmax(want[i])


def test_q4_0_block_sums_exact_and_deterministic():
    """integer-valued inputs with unit scales: every fp32 operation is exact, so the tensor-core path must reproduce the oracle
    bit for bit; and repeated launches (split-K partials summed in split order) give identical bits"""
    rng = np.random.default_rng(5)
    n, k, m = 512, 4096, 24
    blk = np.zeros((n, k // 32, 18), np.uint8)
    blk[:, :, 0:2] = np.frombuffer(np.float16(1.0).tobytes(), np.uint8)
    blk[:, :, 2:] = rng.integers(0, 256, (n, k // 32, 16), dtype=np.uint8)
    rows = blk.reshape(n, -1)
    a = np.zeros((m, k), np.float32)
    a[:] = rng.integers(-60, 61, (m, k)).astype(np.float32)
    a[:, ::32] = 127.0  # every block's amax is 127 -> activation scale exactly 1
    want = oracle.mul_mat_q4_0_f32(rows, a)
    wd = ns.Weight.from_q4_0_host(rows, n, k)
    got, _ = run_mul_mat(wd, a)
    assert np.array_equal(want, np.round(want))
    assert np.array_equal(got, want)
    w2 = rng.normal(0, 0.02, (n, k)).astype(np.float32)
    a2 = rng.normal(0, 1, (m, k)).astype(np.float32)
    wd2 = ns.Weight.from_q4_0_host(oracle.quantize_q4_0(w2), n, k)
    first, _ = run_mul_mat(wd2, a2)
    for _ in range(5):
        again, _ = run_mul_mat(wd2, a2)
        assert np.array_equal(first, again)


@pytest.mark.parametrize("asym", [False, True])
@pytest.mark.parametrize("g,k", [(32, 1024), (128, 4096), (128, 11008), (64, 2048), (256, 4096)])
@pytest.mark.parametrize("m", [4, 8, 20, 32])
def test_btla_s4_int8_compute_batch(asym, g, k, m):
    """BesTLA int4 blobs, int8 compute: u8 activations with zero points per K-block (kernel_ref.h:1825), weight zero points"""
    n = 320
    rng = np.random.default_rng(7 + k + m + g)
    w = rng.uniform(-0.5, 0.5, (k, n)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    q, sc, zp = oracle.btla_quantize(w, g, 4, asym)
    a8, asc, azp = oracle.btla_quantize_act_u8(a, g)
    want = oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, g)
    want_blk = oracle.btla_gemv_u8s8(a8, asc, azp, q, sc, zp, g, blocksum=True)
    for stype in (ns.S_F32, ns.S_BF16):
        wd = ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S4, stype, ns.COMP_INT8)
        got, launches = run_mul_mat(wd, a)
        assert launches == 2
        if stype == ns.S_F32:
            close(got, want_blk, 2e-5)
            close(got, want)
        ref, _ = run_mul_mat(wd, a, flags=ns.MM_FORCE_GEMV)
        close(got, ref, 2e-6)


@pytest.mark.parametrize("asym", [False, True])
@pytest.mark.parametrize("m", [6, 16, 31])
def test_btla_s4_s8_activations_batch(asym, m):
    n, k, g = 256, 2048, 128
    rng = np.random.default_rng(50 + m)
    w = rng.uniform(-0.5, 0.5, (k, n)).astype(np.float32)
    a = rng.uniform(-0.5, 0.5, (m, k)).astype(np.float32)
    q, sc, zp = oracle.btla_quantize(w, g, 4, asym)
    a8, asc = oracle.btla_quantize_act_s8(a, g)
    want = oracle.btla_gemv_s8s8(a8, asc, q, sc, zp, g)
    got, launches = run_mul_mat(ns.Weight.from_unpacked(q, sc, zp, g, ns.W_S4, ns.S_F32, ns.COMP_INT8_S8), a)
    assert launches == 2
    close(got, want)


def test_bias_and_residual_epilogue():
    rng = np.random.default_rng(9)
    n, k, m = 384, 2048, 12
    rows = oracle.quantize_q4_0(rng.normal(0, 0.02, (n, k)).astype(np.float32))
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    bias = rng.normal(0, 1, n).astype(np.float32)
    res = rng.normal(0, 1, (m, n)).astype(np.float32)
    want = oracle.mul_mat_q4_0_f32(rows, a) + bias[None, :] + res
    got, _ = run_mul_mat(ns.Weight.from_q4_0_host(rows, n, k), a, bias=bias, residual=res, flags=ns.MM_BIAS_BCAST)
    close(got, want)


@pytest.mark.parametrize("m", [8, 19, 32])
def test_fused_qkv_and_ffn_nodes_batch(m):
    """ns_mul_qkv ([3][m][n] layout, GQA-sized k/v) and ns_ffn_silu (SiLU(gate) * up inside the matmul epilogue, then down)"""
    import ctypes as C
    L = ns.lib()
    rng = np.random.default_rng(21 + m)
    E, KV, FF = 1024, 256, 2816
    mk = lambda n, k: oracle.quantize_q4_0(rng.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32))
    rq, rk, rv, r1, r3, r2 = mk(E, E), mk(KV, E), mk(KV, E), mk(FF, E), mk(FF, E), mk(E, FF)
    x = rng.normal(0, 1, (m, E)).astype(np.float32)
    W = lambda r, n, k: ns.Weight.from_q4_0_host(r, n, k)
    wq, wk, wv, w1, w3, w2 = W(rq, E, E), W(rk, KV, E), W(rv, KV, E), W(r1, FF, E), W(r3, FF, E), W(r2, E, FF)
    xd = dev(x)
    qkv = torch.full((3, m, E), float("nan"), device="cuda")
    assert L.ns_mul_qkv(wq.h, wk.h, wv.h, C.c_void_p(xd.data_ptr()), E, C.c_void_p(qkv.data_ptr()), E, m, None, None) == 0, ns.last_error()
    sync()
    got = qkv.cpu().numpy()
    close(got[0], oracle.mul_mat_q4_0_f32(rq, x))
    close(got[1][:, :KV], oracle.mul_mat_q4_0_f32(rk, x))
    close(got[2][:, :KV], oracle.mul_mat_q4_0_f32(rv, x))
    tmp = torch.zeros(2, m, FF, device="cuda")
    out = torch.full((m, E), float("nan"), device="cuda")
    assert L.ns_ffn_silu(w1.h, w2.h, w3.h, C.c_void_p(xd.data_ptr()), E, C.c_void_p(tmp.data_ptr()), C.c_void_p(out.data_ptr()), E, m,
                         None, None) == 0, ns.last_error()
    sync()
    g = oracle.mul_mat_q4_0_f32(r1, x)
    u = oracle.mul_mat_q4_0_f32(r3, x)
    silu = np.array([[oracle.lib().orc_silu(float(z)) for z in row] for row in g], np.float32)
    mid = silu * u
    mid_gpu = tmp[0].cpu().numpy()
    close(mid_gpu, mid, 2e-5)
    # the down projection is checked on the GPU's own intermediate: a 1e-7 difference in `mid` can flip a Q8_0 rounding, which is
    # a property of the quantiser (see test_llama2_7b_shaped_greedy_decode_matches_the_reference_engine), not of this matmul
    close(out.cpu().numpy(), oracle.mul_mat_q4_0_f32(r2, np.ascontiguousarray(mid_gpu)))


# ------------------------------------------------------------------------------------------------ the stated arithmetic
COMP = {"q8_0": ns.COMP_Q8_0, "int8": ns.COMP_INT8, "int8_s8": ns.COMP_INT8_S8}
STYPES = {"f32": ns.S_F32, "bf16": ns.S_BF16, "f16": ns.S_F16}
ELT_ULPS = 6      # SiLU / GELU epilogues, fp32 ulps of the function's operand scale (as tests/test_gpu_gemv.py)
RATIOS = []       # bar 2: observed |got - model| / bound


def round_scale(sc, stype):
    """the scale as the device stores it (repack.cu: RNE to bf16 / fp16)"""
    if stype == ns.S_BF16:
        return oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(sc))
    if stype == ns.S_F16:
        return sc.astype(np.float16).astype(np.float32)
    return sc.astype(np.float32)


class IW:
    """a device int4 weight with its host codes q [K,N] (signed), stored scales [K/g, N] and zero points.
    comp 'q4_0': a ggml Q4_0 weight (fp16 d, groups of 32); otherwise ns_weight_from_unpacked with that compute type."""

    def __init__(self, comp, n, k, g=32, asym=False, stype="f32", seed=0, exact=False, q=None, zp=None, sc=None):
        rng = np.random.default_rng(seed)
        if comp == "q4_0":
            g, asym, stype = 32, False, "f16"
        self.comp, self.n, self.k, self.g = comp, n, k, g
        nb = k // g
        self.q = q if q is not None else rng.integers(-8, 8, (k, n)).astype(np.int8)
        self.zp = zp if zp is not None else (rng.integers(-8, 8, (nb, n)).astype(np.int8) if asym else None)
        if sc is None:
            sc = (2.0 ** -rng.integers(0, 3, (nb, n))) if exact else rng.uniform(0.5, 1.5, (nb, n)) / 16
        st = STYPES[stype]
        self.sc = round_scale(np.asarray(sc, np.float32), st)
        if comp == "q4_0":
            nib = (self.q.T.astype(np.int16) + 8).astype(np.uint8).reshape(n, nb, 32)
            rows = np.zeros((n, nb, 18), np.uint8)
            rows[:, :, :2] = np.ascontiguousarray(self.sc.T.astype(np.float16)).view(np.uint8).reshape(n, nb, 2)
            rows[:, :, 2:] = nib[:, :, :16] | (nib[:, :, 16:] << 4)
            self.w = ns.Weight.from_q4_0_host(rows.reshape(n, -1), n, k)
        else:
            self.w = ns.Weight.from_unpacked(self.q, self.sc, self.zp, g, ns.W_S4, st, COMP[comp])

    @property
    def acomp(self):
        return "q8_0" if self.comp == "q4_0" else self.comp

    def model(self, a):
        codes, asc, ab = oracle.imma_act(a, self.acomp, self.g)
        return oracle.imma_stated(codes, asc, ab, self.q, self.sc, self.zp, self.g)

    def ablock(self):
        return 32 if self.acomp == "q8_0" else self.g


def exact_acts(m, k, ab, comp, seed, r=4):
    """activations whose blocks quantise to power-of-two scales and small integer codes: per block of ab values an anchor
    (+-127 for s8 / Q8_0; 127 and -128 for u8, zero point 128) sets the scale 2^e, the rest are integers in [-r, r] times 2^e"""
    rng = np.random.default_rng(seed)
    nb = k // ab
    e = 2.0 ** -rng.integers(0, 3, (m, nb, 1))
    v = rng.integers(-r, r + 1, (m, nb, ab)).astype(np.float64)
    if comp == "int8":
        v[:, :, 0], v[:, :, 1] = 127, -128
    else:
        v[:, :, 0] = 127 * rng.choice([-1, 1], (m, nb))
    return (v * e).reshape(m, k).astype(np.float32)


def assert_exact_construction(w, a, mag):
    """every partial sum of t_b is exact in fp32: sum |t_b| < 2^24 x the smallest unit (power-of-two scales)"""
    codes, asc, ab = oracle.imma_act(a, w.acomp, w.g)
    live = (codes.reshape(asc.shape[0], asc.shape[1], ab) != 0).any(axis=2)  # blocks that contribute (a zero block's scale is tiny)
    unit = float(asc[live].min()) * float(w.sc[w.sc > 0].min())
    assert np.log2(unit) == np.round(np.log2(unit))
    assert mag.max() < 2.0 ** 24 * unit, mag.max() / unit


def mm(w, a, flags=0, ws=None, lda=None, ldo=None, bias=None, bcast=False, residual=None, rows_out=None):
    """one ns_mul_mat call into a NaN-filled dst; returns (dst [rows_out][ldo], launches)"""
    m, k = a.shape
    lda, ldo = lda or k, ldo or w.n
    x = torch.zeros((m, lda), device="cuda")
    x[:, :k] = torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    out = torch.full((rows_out or m, ldo), float("nan"), device="cuda")
    b = dev(np.asarray(bias, np.float32)) if bias is not None else None
    r = dev(np.asarray(residual, np.float32)) if residual is not None else None
    torch.cuda.synchronize()
    lc = ns.lib().ns_launch_count()
    ns.mul_mat(w.w if isinstance(w, IW) else w, x.data_ptr(), lda, out.data_ptr(), ldo, m, b.data_ptr() if b is not None else None,
               r.data_ptr() if r is not None else None, flags | (ns.MM_BIAS_BCAST if bcast else 0), ws_ptr=ws)
    sync()
    return out.cpu().numpy(), ns.lib().ns_launch_count() - lc


def check_bound(got, model):
    tot, mag, nb = model
    ratio = oracle.imma_bound_ratio(got, tot, mag, nb)
    RATIOS.append(ratio)
    assert ratio <= 1.0, ratio
    return ratio


# planner mirror (make_plan, csrc/gemm_imma.cu): which split count a launch takes, and whether it has a plan at all
def plan(n_tiles, k, g, ss, asym, m, sms=132):
    mt = 8 if m <= 8 else 16 if m <= 16 else 32
    nsl, cpg = -(-k // 256), g // 32
    kstage = 16384 + -(-(mt * 320) // 1024) * 1024
    best, ksplit = -1, 0
    for ks in range(1, min(16, nsl) + 1):
        if ks > 1 and n_tiles * ks > 640:
            continue
        max_sl = -(-nsl // ks)
        ng = ((max_sl + 1) * 8 + cpg - 1) // cpg + 1
        sc_zp = -(-(15 + ss * ng) // 16) * 16
        sc_row = sc_zp + (-(-(15 + ng) // 16) * 16 if asym else 0)
        if 128 * sc_row + 256 + 64 + 1024 + min(max_sl, 3) * kstage > 111 * 1024:
            continue
        cost = -(-(n_tiles * ks) // (2 * sms)) * (2 * max_sl + 2) * 16 + ks
        if best < 0 or cost < best:
            best, ksplit = cost, ks
    return ksplit  # 0: no plan


def plan_of(n, k, g, stype, asym, m, gate_up=False):
    tiles = -(-n // 64) if gate_up else -(-n // 128)
    return plan(tiles, k, g, 4 if stype == "f32" else 2, asym, m)


FORMATS = list(itertools.product(["q8_0", "int8", "int8_s8"], [False, True], ["f32", "bf16", "f16"], [32, 64, 128, 256]))
# (n, k, m): one tile (the largest split), overhangs of the 128-row tile, many tiles; every token-tile class
SHAPES = [(8, 4096, 3), (136, 11008, 9), (320, 14336, 17), (4160, 4096, 32), (136, 256, 8), (320, 4096, 16), (8, 14336, 32),
          (136, 4096, 3), (320, 11008, 32), (4160, 256, 9), (8, 11008, 17), (320, 4096, 8)]


def fmt_id(f):
    return f"{f[0]}-{'asym' if f[1] else 'sym'}-{f[2]}-g{f[3]}"


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "random"])
@pytest.mark.parametrize("i", range(len(FORMATS)), ids=[fmt_id(f) for f in FORMATS])
def test_block_sums_against_stated_arithmetic(i, exact):
    """bars 1 and 2 for every compute type x zero points x scale type x group; Q8_0 takes weight groups of 32..256 (activation
    blocks of 32 under one weight scale)"""
    comp, asym, stype, g = FORMATS[i]
    n, k, m = SHAPES[(i + (5 if exact else 0)) % len(SHAPES)]
    w = IW(comp, n, k, g, asym, stype, seed=100 + i, exact=exact)
    a = exact_acts(m, k, w.ablock(), comp, 200 + i) if exact else np.random.default_rng(300 + i).normal(0, 1, (m, k)).astype(np.float32)
    model = w.model(a)
    got, launches = mm(w, a)
    assert launches == 2, launches
    if exact:
        assert_exact_construction(w, a, model[1])
        assert np.array_equal(got, model[0].astype(np.float32))
    else:
        check_bound(got, model)


@pytest.mark.parametrize("exact", [True, False], ids=["exact", "random"])
def test_q4_0_ggml_against_stated_arithmetic(exact):
    for j, (n, k, m) in enumerate(SHAPES[:6]):
        w = IW("q4_0", n, k, seed=400 + j, exact=exact)
        a = exact_acts(m, k, 32, "q8_0", 410 + j) if exact else np.random.default_rng(420 + j).normal(0, 1, (m, k)).astype(np.float32)
        model = w.model(a)
        got, launches = mm(w, a)
        assert launches == 2
        if exact:
            assert_exact_construction(w, a, model[1])
            assert np.array_equal(got, model[0].astype(np.float32)), (n, k, m)
        else:
            check_bound(got, model)


SPLIT_FORMATS = [("int8", True, "bf16", 64), ("int8_s8", True, "f16", 256), ("q8_0", False, "f32", 32), ("int8", False, "f32", 128),
                 ("q8_0", True, "bf16", 128), ("int8_s8", False, "f16", 64)]


@pytest.mark.parametrize("fmt", SPLIT_FORMATS, ids=[fmt_id(f) for f in SPLIT_FORMATS])
def test_every_split_count(fmt):
    """one 8-row weight tile over k = 256 s takes s splits of one slice each (s = 1..16): splits that start in the middle of a
    16-byte segment of 2-byte scales and of zero points (groups >= 64), exact and random data, repeated launches bit-identical"""
    comp, asym, stype, g = fmt
    for s in range(1, 17):
        k = 256 * s
        assert plan_of(8, k, g, stype, asym, 3) == s
        w = IW(comp, 8, k, g, asym, stype, seed=500 + s, exact=True)
        a = exact_acts(3, k, w.ablock(), comp, 510 + s)
        model = w.model(a)
        assert_exact_construction(w, a, model[1])
        got, launches = mm(w, a)
        assert launches == 2
        assert np.array_equal(got, model[0].astype(np.float32)), s
        wr = IW(comp, 8, k, g, asym, stype, seed=520 + s)
        ar = np.random.default_rng(530 + s).normal(0, 1, (3, k)).astype(np.float32)
        first, _ = mm(wr, ar)
        check_bound(first, wr.model(ar))
        for _ in range(2):
            assert np.array_equal(mm(wr, ar)[0], first), s


@functools.lru_cache(maxsize=None)
def big_random(n, k, g, stype, asym, seed=1):
    return ns.Weight.random(n, k, g, ns.W_S4, stype, ns.COMP_INT8, asym, seed)


def test_row_invariance_within_a_token_tile_class():
    """a row's output depends on its weight rows and its own activations only: not on the other rows, its position or m, within
    one class (n = 4096, k = 11008, g32: 8 splits up to 16 rows, 15 from 17)"""
    n, k = 4096, 11008
    assert (plan_of(n, k, 32, "f32", False, 16), plan_of(n, k, 32, "f32", False, 17)) == (8, 15)
    w = big_random(n, k, 32, ns.S_F32, False)
    x = np.random.default_rng(600).normal(0, 1, (32, k)).astype(np.float32)
    rng = np.random.default_rng(601)
    for lo, hi in ((3, 8), (9, 16), (17, 32)):
        full, launches = mm(w, x[:hi])
        assert launches == 2
        for sub in (lo, (lo + hi) // 2, hi):
            pick = rng.permutation(hi)[:sub]
            got, _ = mm(w, x[pick])
            assert np.array_equal(got, full[pick]), (lo, hi, sub)


def test_across_classes_rigorous_bound():
    n, k = 320, 11008
    w = IW("int8", n, k, 32, True, "bf16", seed=610)
    x = np.random.default_rng(611).normal(0, 1, (32, k)).astype(np.float32)
    tot, mag, nb = w.model(x)
    for m in (3, 8, 9, 16, 17, 32):
        got, launches = mm(w, x[:m])
        assert launches == 2
        check_bound(got, (tot[:m], mag[:m], nb))


def test_extremes_of_the_block_sum_fields():
    """a u8 block of 256 codes 255 (Sa = 65280, the top of the 16-bit field) against q - zp = +-15 (|isum| = 979200, the edge
    of the exact int -> float conversion), an s8 block of 256 codes -127 (Sa = -32512: sign extension), an all-zero block"""
    k, n, g = 1024, 136, 256
    rng = np.random.default_rng(700)
    q = rng.integers(-8, 8, (k, n)).astype(np.int8)
    zp = rng.integers(-8, 8, (k // g, n)).astype(np.int8)
    q[:, 0], zp[:, 0] = 7, -8     # q - zp = 15
    q[:, 1], zp[:, 1] = -8, 7     # q - zp = -15
    sc = 2.0 ** -rng.integers(0, 3, (k // g, n))
    for comp, fill, code, sa in (("int8", 255.0 / 256, 255, 65280), ("int8_s8", -127.0 / 128, -127, -32512)):
        a = exact_acts(3, k, g, comp, 701)
        a[0, :g] = fill       # block 0: one code everywhere
        a[0, g:2 * g] = 0     # block 1: all zero
        a[2] = 0              # a whole zero row
        codes, asc, _ = oracle.imma_act(a, comp, g)
        assert (codes[0, :g] == code).all() and codes[0, :g].sum() == sa  # u8: zero point 0 (the block's minimum is 0)
        w = IW(comp, n, k, g, True, "f32", q=q, zp=zp, sc=sc)
        tot, mag, _ = w.model(a)
        isum0 = (codes[0, :g].astype(np.int64) @ (q[:g, :2].astype(np.int64) - zp[0, :2]))
        assert abs(int(isum0[0])) == 256 * abs(code) * 15 and isum0[1] == -isum0[0]
        got, launches = mm(w, a)
        assert launches == 2
        assert_exact_construction(w, a, mag)
        assert np.array_equal(got, tot.astype(np.float32)), comp
        assert (got[2] == 0).all()


def test_output_masking_lda_ldo():
    """dst NaN-filled with MT rows and ldo > n, lda > k: only rows < m and columns < n are written"""
    for n, k, m, g in ((136, 1024, 5, 64), (320, 2048, 13, 128), (8, 4096, 27, 32)):
        w = IW("int8", n, k, g, True, "bf16", seed=800 + m, exact=True)
        a = exact_acts(m, k, g, "int8", 801 + m)
        mt = 8 if m <= 8 else 16 if m <= 16 else 32
        got, launches = mm(w, a, lda=k + 40, ldo=n + 24, rows_out=mt)
        assert launches == 2
        assert np.isnan(got[m:]).all() and np.isnan(got[:m, n:]).all()
        assert np.array_equal(got[:m, :n], w.model(a)[0].astype(np.float32))


def test_bias_residual_epilogue_bit_exact():
    """bias (broadcast and per row) and residual are fp32 adds on the plain result of the same plan: fl(fl(v + b) + r)"""
    n, k, m, ldo = 320, 4096, 11, 336
    w = IW("int8", n, k, 128, True, "bf16", seed=900)
    rng = np.random.default_rng(901)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    bias_b = rng.normal(0, 1, n).astype(np.float32)
    bias_row = rng.normal(0, 1, (m, ldo)).astype(np.float32)
    res = rng.normal(0, 1, (m, ldo)).astype(np.float32)
    plain = mm(w, a, ldo=ldo)[0][:, :n]
    got, launches = mm(w, a, ldo=ldo, bias=bias_row, residual=res)
    assert launches == 2
    assert np.array_equal(got[:, :n], (plain + bias_row[:, :n]) + res[:, :n]) and np.isnan(got[:, n:]).all()
    got = mm(w, a, ldo=ldo, bias=bias_b, bcast=True, residual=res)[0][:, :n]
    assert np.array_equal(got, (plain + bias_b) + res[:, :n])
    assert np.array_equal(mm(w, a, ldo=ldo, bias=bias_row)[0][:, :n], plain + bias_row[:, :n])


def gelu_f32(x):
    """the tanh GELU in fp32 (ns_gelu), and the operand scale its ulp bar is measured in"""
    x = np.asarray(x, np.float32)
    t = np.tanh(np.float32(0.7978845834732056) * (x + np.float32(0.044714998453855515) * x * x * x))
    return np.float32(0.5) * x * (np.float32(1) + t), 0.5 * np.abs(x) * (1 + np.abs(t))


def silu_f32(x):
    """x / (1 + exp(-x)) in fp32 (orc_silu; ns_silu), and its operand scale"""
    y = np.array([oracle.lib().orc_silu(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32).reshape(np.shape(x))
    return y, np.abs(y)


def assert_ulps(got, want, scale, ulps=ELT_ULPS):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    bar = np.spacing(np.maximum(np.asarray(scale, np.float32), np.float32(1e-30))).astype(np.float64)
    assert (err <= ulps * bar).all(), (err / bar).max()


def test_gelu_epilogue_and_plain_ffn():
    """ns_ffn_gelu without w3: tmp = gelu(x W1^T + b1) in the matmul epilogue, within ELT_ULPS of the fp32 GELU of the GPU's own
    pre-activation (a plain call with the bias, same m); dst = tmp W2^T + b2 bit-equal to a plain call on the GPU's tmp"""
    E, F, m = 1024, 256, 12
    w1, w2 = IW("int8_s8", F, E, 64, True, "f16", seed=1000), IW("int8_s8", E, F, 64, False, "f32", seed=1001)
    rng = np.random.default_rng(1002)
    a = rng.normal(0, 1, (m, E)).astype(np.float32)
    b1, b2 = rng.normal(0, 1, F).astype(np.float32), rng.normal(0, 1, E).astype(np.float32)
    x, tmp, out = dev(a), torch.full((m, F), float("nan"), device="cuda"), torch.full((m, E), float("nan"), device="cuda")
    d1, d2 = dev(b1), dev(b2)
    torch.cuda.synchronize()
    lc = ns.lib().ns_launch_count()
    ns.ffn_gelu(w1.w, w2.w, None, d1.data_ptr(), d2.data_ptr(), 1, x.data_ptr(), E, tmp.data_ptr(), out.data_ptr(), E, m)
    sync()
    assert ns.lib().ns_launch_count() - lc == 4
    want, scale = gelu_f32(mm(w1, a, bias=b1, bcast=True)[0])
    t = tmp.cpu().numpy()
    assert_ulps(t, want, scale)
    assert np.array_equal(out.cpu().numpy(), mm(w2, t, bias=b2, bcast=True)[0])


def test_qkv_gqa_slabs():
    """ns_mul_qkv with GQA widths (q 1024, k / v 256): bars 1 and 2 on every slab of the [3][m][ldo] output"""
    E, KV, m = 1024, 256, 19
    for exact in (True, False):
        ws = [IW("int8_s8", nn, E, 64, True, "f16", seed=1100 + i, exact=exact) for i, nn in enumerate((E, KV, KV))]
        a = exact_acts(m, E, 64, "int8_s8", 1110) if exact else np.random.default_rng(1111).normal(0, 1, (m, E)).astype(np.float32)
        x = dev(a)
        out = torch.full((3, m, E), float("nan"), device="cuda")
        torch.cuda.synchronize()
        lc = ns.lib().ns_launch_count()
        ns.mul_qkv(ws[0].w, ws[1].w, ws[2].w, x.data_ptr(), E, out.data_ptr(), E, m)
        sync()
        assert ns.lib().ns_launch_count() - lc == 2
        o = out.cpu().numpy()
        for i, w in enumerate(ws):
            model = w.model(a)
            assert np.isnan(o[i, :, w.n:]).all()
            if exact:
                assert_exact_construction(w, a, model[1])
                assert np.array_equal(o[i, :, :w.n], model[0].astype(np.float32)), i
            else:
                check_bound(o[i, :, :w.n], model)


@pytest.mark.parametrize("gelu", [False, True], ids=["silu", "gelu"])
@pytest.mark.parametrize("m", [5, 24])
def test_gate_up_and_down(gelu, m):
    """SiLU / GELU(gate) * up in the gate/up epilogue (64-row tiles of each weight), then the down projection bit-equal to a plain
    call on the GPU's own product.  Exact data: g and u are exact, so the product is within ELT_ULPS of elt(g) * u.  Random data:
    bar 2 on g and u, carried through elt (|elt'| <= 1.13).  fmid is a multiple of 256 here: the down projection takes the
    integer kernel only for k % 256 == 0, and an FFN takes it for both halves or neither."""
    E, F = 1024, 768
    w2 = IW("int8", E, F, 128, True, "bf16", seed=1210)
    elt = gelu_f32 if gelu else silu_f32
    for exact in (True, False):
        w1, w3 = (IW("int8", F, E, 128, True, "bf16", seed=1200 + s + 2 * exact, exact=exact) for s in (0, 1))
        a = exact_acts(m, E, 128, "int8", 1203) if exact else np.random.default_rng(1204).normal(0, 1, (m, E)).astype(np.float32)
        x = dev(a)
        tmp = torch.full((2 * m * F,), float("nan"), device="cuda")
        out = torch.full((m, E), float("nan"), device="cuda")
        torch.cuda.synchronize()
        lc = ns.lib().ns_launch_count()
        if gelu:
            ns.ffn_gelu(w1.w, w2.w, w3.w, None, None, 0, x.data_ptr(), E, tmp.data_ptr(), out.data_ptr(), E, m)
        else:
            ns.ffn_silu(w1.w, w2.w, w3.w, x.data_ptr(), E, tmp.data_ptr(), out.data_ptr(), E, m)
        sync()
        assert ns.lib().ns_launch_count() - lc == 4
        mid = tmp.cpu().numpy()[:m * F].reshape(m, F)
        (g, gmag, nb), (u, umag, _) = w1.model(a), w3.model(a)
        n = nb + 16
        gam = n * 2.0 ** -24 / (1 - n * 2.0 ** -24)
        eg, eu = (0, 0) if exact else (gam * gmag, gam * umag)
        if exact:
            assert_exact_construction(w1, a, gmag)
            assert_exact_construction(w3, a, umag)
        s, scale = elt(g.astype(np.float32))  # the fp32 function (it underflows to 0 below -88 as the kernel's does)
        s = s.astype(np.float64)
        sp = lambda v: np.spacing(np.asarray(v, np.float32)).astype(np.float64)
        bound = 1.13 * eg * (np.abs(u) + eu) + (np.abs(s) + 1.13 * eg) * eu + ELT_ULPS * sp(scale + 1.13 * eg) * (np.abs(u) + eu)
        err = np.abs(mid.astype(np.float64) - s * u)
        assert (err <= bound + sp(np.abs(mid))).all(), (exact, float((err / (bound + sp(np.abs(mid)))).max()))
        assert np.array_equal(out.cpu().numpy(), mm(w2, mid)[0]), exact


def test_graph_replay_two_nodes_share_a_workspace():
    """two integer tensor-core nodes of different plans (16 splits of one tile; 4 splits of 3 tiles) captured into one CUDA graph
    through the queue argument, sharing one caller workspace: every replay equals the eager results (the tickets of each split
    tile are back at zero after every launch)"""
    m, k = 8, 4096
    wa, wb = IW("int8", 8, k, 64, True, "bf16", seed=1300), IW("q4_0", 320, 1024, seed=1301)
    assert (plan_of(8, k, 64, "bf16", True, m), plan_of(320, 1024, 32, "f16", False, m)) == (16, 4)
    rng = np.random.default_rng(1302)
    xa, xb = dev(rng.normal(0, 1, (m, k)).astype(np.float32)), dev(rng.normal(0, 1, (m, 1024)).astype(np.float32))
    ws = torch.zeros(ns.lib().ns_device_workspace_bytes(m, k), dtype=torch.uint8, device="cuda")
    oa, ob = torch.full((m, 8), float("nan"), device="cuda"), torch.full((m, 320), float("nan"), device="cuda")
    s = torch.cuda.Stream()

    def nodes():
        q = C.c_void_p(s.cuda_stream)
        ns.mul_mat(wa.w, xa.data_ptr(), k, oa.data_ptr(), 8, m, ws_ptr=ws.data_ptr(), queue=q)
        ns.mul_mat(wb.w, xb.data_ptr(), 1024, ob.data_ptr(), 320, m, ws_ptr=ws.data_ptr(), queue=q)

    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        nodes()
    s.synchronize()
    want_a, want_b = oa.cpu().numpy(), ob.cpu().numpy()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        nodes()
    for _ in range(3):
        oa.fill_(float("nan"))
        ob.fill_(float("nan"))
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(oa.cpu().numpy(), want_a) and np.array_equal(ob.cpu().numpy(), want_b)
    del g


def test_workspace_bound_leaves_guard_bytes():
    """with exactly ns_device_workspace_bytes(m, k) bytes of workspace, bytes placed after it are never written: the largest image
    (m = 32, k = 14336), the most partial tiles (many tiles x splits) and the largest split of one tile"""
    L = ns.lib()
    for n, k, m in ((4160, 14336, 32), (1024, 4096, 32), (8, 4096, 17), (4160, 256, 9)):
        assert plan_of(n, k, 32, "f32", False, m) > 0
        w = big_random(n, k, 32, ns.S_F32, False)
        nbytes = L.ns_device_workspace_bytes(m, k)
        buf = torch.full((nbytes + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
        a = np.random.default_rng(1400 + m).normal(0, 1, (m, k)).astype(np.float32)
        got, launches = mm(w, a, ws=buf.data_ptr())
        assert launches == 2
        assert (buf[nbytes:].cpu().numpy() == 0xA5).all(), (n, k, m)
        assert np.array_equal(got, mm(w, a)[0])


def test_mul_mat_id_expert_slices():
    """ns_mul_mat_id with shuffled ids: each expert slice of 3..32 rows equals a plain call on that expert's gathered rows"""
    n, k = 320, 2048
    ws = [IW("int8", n, k, 128, True, "bf16", seed=1500 + e) for e in range(4)]
    counts = [3, 17, 9, 32]
    rng = np.random.default_rng(1501)
    ids = rng.permutation(np.repeat(np.arange(4), counts)).astype(np.int32)[:, None]
    m = len(ids)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    x, out = dev(a), torch.full((m, n), float("nan"), device="cuda")
    ns.mul_mat_id([w.w for w in ws], ids, 0, x.data_ptr(), k, out.data_ptr(), n, m)
    sync()
    got = out.cpu().numpy()
    for e, w in enumerate(ws):
        rows = np.flatnonzero(ids[:, 0] == e)
        plain, launches = mm(w, a[rows])
        assert launches == 2
        assert np.array_equal(got[rows], plain), e


# ------------------------------------------------------------------------------------------------ shapes without a plan
def gemv_tile(k):
    """rows of one GEMV tile of int4 weights with an integer compute type (ns_gemv_tile_rows): fewer for long rows"""
    kpad = -(-k // 32) * 32
    per_row, mt = -(-kpad // 1024) * 1024 + -(-(kpad // 32) // 2) * 2 * 8, 4
    while mt > 1 and per_row * mt > 64 * 1024:
        mt //= 2
    return mt


# (n, k) of the nodes the planner cannot fit at some of 3..32 rows with group-32 weights: 7B lm_head, 70B gate/up and down,
# Mistral down, 70B lm_head
NO_PLAN_SHAPES = [(32000, 4096), (28672, 8192), (8192, 28672), (4096, 14336), (32000, 8192)]
WEIGHTS = [("f32", False), ("bf16", True)]


@pytest.mark.parametrize("stype,asym", WEIGHTS, ids=["g32-f32", "g32-bf16-asym"])
@pytest.mark.parametrize("n,k", NO_PLAN_SHAPES)
def test_unplanned_shapes_take_gemv_tiles(n, k, stype, asym):
    """a plain node whose launch has no shared-memory plan runs GEMV tiles (the same exact block sums, never the bf16 GEMM):
    rc 0, one ring launch per tile of <= 4 rows, bit-equal to NS_MM_FORCE_GEMV; a node with a plan keeps the integer tensor cores"""
    w = big_random(n, k, 32, STYPES[stype], asym)
    x = np.random.default_rng(1600).normal(0, 1, (32, k)).astype(np.float32)
    for m in (3, 17, 32):
        got, launches = mm(w, x[:m])
        ref, ref_launches = mm(w, x[:m], flags=ns.MM_FORCE_GEMV)
        assert ref_launches == -(-m // gemv_tile(k))
        if plan_of(n, k, 32, stype, asym, m):
            assert launches == 2, (m, launches)
            assert np.abs(got - ref).max() <= 2e-6 * np.abs(ref).max()
        else:
            assert launches == ref_launches, (m, launches)
            assert np.array_equal(got, ref), m


def test_planner_mirror_matches_the_known_table():
    """the test's planner mirror against shapes worked out by hand from make_plan (m classes 3..8, 9..16, 17..32)"""
    table = {(32000, 4096, "f32", False): (True, True, False), (28672, 8192, "f32", False): (False, False, False),
             (8192, 28672, "f32", False): (False, False, False), (8192, 28672, "bf16", True): (True, True, False),
             (4096, 14336, "f32", True): (True, True, False), (32000, 8192, "f32", False): (False, False, False)}
    for (n, k, st, asym), want in table.items():
        assert tuple(plan_of(n, k, 32, st, asym, m) > 0 for m in (3, 9, 17)) == want, (n, k, st, asym)
    assert not plan_of(28672, 8192, 32, "f32", False, 3, gate_up=True)


def test_ffn_with_unplanned_down_issues_no_imma_launch():
    """a wide FFN on a narrow model (1024 -> 14336 -> 1024), group-32 asym weights at 17 rows: gate/up has a plan, the down
    projection (k = 14336) has none, so both halves run GEMV tiles and nothing reaches the integer tensor cores"""
    E, F, m = 1024, 14336, 17
    assert plan_of(F, E, 32, "f32", True, m, gate_up=True) and not plan_of(E, F, 32, "f32", True, m)
    w1, w3, w2 = (big_random(nn, kk, 32, ns.S_F32, True, seed=s) for nn, kk, s in ((F, E, 1), (F, E, 2), (E, F, 3)))
    x = dev(np.random.default_rng(1700).normal(0, 1, (m, E)).astype(np.float32))
    tmp = torch.zeros(2 * m * F, device="cuda")
    out = torch.full((m, E), float("nan"), device="cuda")
    L = ns.lib()
    torch.cuda.synchronize()
    lc = L.ns_launch_count()
    rc = L.ns_ffn_silu(w1.h, w2.h, w3.h, C.c_void_p(x.data_ptr()), E, C.c_void_p(tmp.data_ptr()), C.c_void_p(out.data_ptr()), E, m,
                       None, None)
    sync()
    assert rc == 0, ns.last_error()
    assert L.ns_launch_count() - lc == -(-m // gemv_tile(E)) + -(-m // gemv_tile(F))  # one ring launch per tile
    assert not np.isnan(out.cpu().numpy()).any()


@pytest.fixture(scope="module", autouse=True)
def _report_ratio():
    yield
    if RATIOS:
        print(f"\nlargest bar-2 ratio: {max(RATIOS):.4g} of gamma_n sum |t_b| over {len(RATIOS)} checks")

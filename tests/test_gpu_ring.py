"""The ring GEMV (csrc/gemv_ring_impl.cuh: gemv_ring_kernel, launched from gemv_ring.cu / gemv_ring_wide.cu) held to its stated
arithmetic bit for bit (DESIGN.md section 4).  For output row n and activation row m: per 32-element chunk c an exact integer
isum_c = sum (a - za)(q - zp) and t_c = fp32(a_scale_c * w_scale_gi); lane L runs acc = fmaf(isum_c, t_c, acc) over
c = L, L + 32, ... from +0; the xor butterfly 16, 8, 4, 2, 1 combines the lanes (oracle.ring_stated).  The fused RMSNorm hands the
quantiser oracle.ring_norm_row's fp32 row.  The epilogue is plain fp32: fl(fl(v + bias) + residual); SiLU and GELU are held within
ELT_ULPS of the fp32 function of the GPU's own pre-activation.

Every case states which plan it runs through ns_gemv_ring_plan, the function the launchers themselves ask (wide = one CTA per SM
with 14 consumer warps, else 7 consumer warps; weight rows per ring stage; stages; stage-owning warps; CTAs per SM), and pins its
launch count: 1 per tile when the kernel quantises its own fp32 activations, 2 with a prepared activation image."""
import ctypes as C

import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
import oracle

pytestmark = pytest.mark.gpu

E_UNSUPPORTED = -4
ELT_ULPS = 6
COMP = {"q8_0": ns.COMP_Q8_0, "int8": ns.COMP_INT8, "int8_s8": ns.COMP_INT8_S8}
STYPES = {"f32": ns.S_F32, "bf16": ns.S_BF16, "f16": ns.S_F16}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def sync():
    torch.cuda.synchronize()
    ns.lib().bestla_device_sync(None)


def launches():
    return ns.lib().ns_launch_count()


def round_scale(sc, stype):
    if stype == ns.S_BF16:
        return oracle.bf16_bits_to_f32(oracle.f32_to_bf16_bits(sc))
    if stype == ns.S_F16:
        return sc.astype(np.float16).astype(np.float32)
    return sc.astype(np.float32)


class RW:
    """a device int4 weight with its host codes q [K, N] (signed), stored scales [ceil(K/g), N] and zero points.
    comp 'q4_0': a ggml Q4_0 weight (fp16 d, groups of 32); otherwise ns_weight_from_unpacked with that compute type."""

    def __init__(self, comp, n, k, g=32, asym=False, stype="f32", seed=0, q=None, zp=None, sc=None):
        rng = np.random.default_rng(seed)
        if comp == "q4_0":
            g, asym, stype = 32, False, "f16"
        self.comp, self.n, self.k, self.g, self.asym, self.stype = comp, n, k, g, asym, STYPES[stype]
        nb = -(-k // g)
        self.q = q if q is not None else rng.integers(-8, 8, (k, n), dtype=np.int8)
        self.zp = zp if zp is not None else (rng.integers(-8, 8, (nb, n), dtype=np.int8) if asym else None)
        if sc is None:
            sc = rng.uniform(0.5, 1.5, (nb, n)).astype(np.float32) / 16
        self.sc = round_scale(np.asarray(sc, np.float32), self.stype)
        if comp == "q4_0":
            nib = (self.q.T.astype(np.int16) + 8).astype(np.uint8).reshape(n, nb, 32)
            rows = np.zeros((n, nb, 18), np.uint8)
            rows[:, :, :2] = np.ascontiguousarray(self.sc.T.astype(np.float16)).view(np.uint8).reshape(n, nb, 2)
            rows[:, :, 2:] = nib[:, :, :16] | (nib[:, :, 16:] << 4)
            self.w = ns.Weight.from_q4_0_host(rows.reshape(n, -1), n, k)
        else:
            self.w = ns.Weight.from_unpacked(self.q, self.sc, self.zp, g, ns.W_S4, self.stype, COMP[comp])

    @property
    def acomp(self):
        return "q8_0" if self.comp == "q4_0" else self.comp

    @property
    def fused(self):
        """the kernel quantises fp32 activations itself (ns_gemv_fused_quant_ok)"""
        qg = 32 if self.acomp == "q8_0" else self.g
        return qg in (32, 64, 128, 256) and self.k % qg == 0

    def model(self, a):
        codes, asc, ab = oracle.imma_act(np.asarray(a, np.float32), self.acomp, self.g)
        return oracle.ring_stated(codes, asc, ab, self.q, self.sc, self.zp, self.g)

    @property
    def tile(self):
        """rows of one GEMV tile (ns_gemv_tile_rows): the largest m the plan entry takes"""
        out = (C.c_int * 5)()
        return max(m for m in (1, 2, 4) if ns.lib().ns_gemv_ring_plan(self.k, self.g, self.stype, 1 if self.asym else 0,
                                                                       COMP[self.acomp], 0, m, 0, 0, out) >= 0)

    def plan(self, m, fused, mode=0, norm=False):
        out = (C.c_int * 5)()
        rc = ns.lib().ns_gemv_ring_plan(self.k, self.g, self.stype, 1 if self.asym else 0, ns.COMP_Q8_0 if self.comp == "q4_0" else
                                        COMP[self.comp], mode, m, 1 if fused else 0, 1 if norm else 0, out)
        assert rc == 1, (rc, ns.last_error())
        return tuple(out)


def mm(w, a, flags=0, lda=None, ldo=None, bias=None, bcast=False, residual=None, engine=False, ws=None):
    """one ns_mul_mat (or ns_mul_mat_engine_image) call into a NaN-filled dst; returns (dst [m][ldo], launches)"""
    m, k = a.shape
    lda, ldo = lda or k, ldo or w.n
    x = torch.zeros((m, lda), device="cuda")
    x[:, :k] = dev(a)
    out = torch.full((m, ldo), float("nan"), device="cuda")
    b = dev(bias) if bias is not None else None
    r = dev(residual) if residual is not None else None
    torch.cuda.synchronize()
    lc = launches()
    if engine:
        rc = ns.lib().ns_mul_mat_engine_image(w.w.h, C.c_void_p(x.data_ptr()), lda, C.c_void_p(out.data_ptr()), ldo, m,
                                              C.c_void_p(r.data_ptr()) if r is not None else None, None, None)
        assert rc == 0, ns.last_error()
    else:
        ns.mul_mat(w.w, x.data_ptr(), lda, out.data_ptr(), ldo, m, b.data_ptr() if b is not None else None,
                   r.data_ptr() if r is not None else None, flags | (ns.MM_BIAS_BCAST if bcast else 0), ws_ptr=ws)
    sync()
    return out.cpu().numpy(), launches() - lc


def prepared(ws_list, a, mode=0, ldo=None, aux=False):
    """ns_prepare_activation + ns_matmul_prepared (the two-CTA kernel on a pre-quantised image); returns (dst, aux, launches)"""
    L = ns.lib()
    m, k = a.shape
    w0 = ws_list[0]
    ldo = ldo or max(w.n for w in ws_list)
    rows = len(ws_list) * m if mode == 1 else m
    x = dev(a)
    wsb = torch.zeros(L.ns_device_workspace_bytes(m, k), dtype=torch.uint8, device="cuda")
    out = torch.full((rows, ldo), float("nan"), device="cuda")
    ax = torch.full((m, ldo), float("nan"), device="cuda") if aux else None
    torch.cuda.synchronize()
    lc = launches()
    assert L.ns_prepare_activation(w0.w.h, C.c_void_p(x.data_ptr()), k, m, C.c_void_p(wsb.data_ptr()), None) == 0, ns.last_error()
    hs = (C.c_void_p * len(ws_list))(*[w.w.h for w in ws_list])
    rc = L.ns_matmul_prepared(hs, len(ws_list), mode, C.c_void_p(wsb.data_ptr()), C.c_void_p(out.data_ptr()), ldo, m, None, 0, None,
                              C.c_void_p(ax.data_ptr()) if aux else None, None)
    assert rc == 0, ns.last_error()
    sync()
    return out.cpu().numpy(), (ax.cpu().numpy() if aux else None), launches() - lc


def check_equal(got, want, what=""):
    if not np.array_equal(got, want):
        bad = got != want
        ulps = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.size} differ, first at {np.argwhere(bad)[0].tolist()}, "
                             f"largest {int(ulps.max())} ulps")


def gelu_f32(x):
    x = np.asarray(x, np.float32)
    t = np.tanh(np.float32(0.7978845834732056) * (x + np.float32(0.044714998453855515) * x * x * x))
    return np.float32(0.5) * x * (np.float32(1) + t), 0.5 * np.abs(x) * (1 + np.abs(t))


def silu_f32(x):
    y = np.array([oracle.lib().orc_silu(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32).reshape(np.shape(x))
    return y, np.abs(y)


def assert_ulps(got, want, scale, ulps=ELT_ULPS):
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    bar = np.spacing(np.maximum(np.asarray(scale, np.float32), np.float32(1e-30))).astype(np.float64)
    assert (err <= ulps * bar).all(), (err / bar).max()


def acts(m, k, seed):
    return np.random.default_rng(seed).normal(0, 1, (m, k)).astype(np.float32)


# ------------------------------------------------------------------------------------------------ formats
FORMATS = [(c, asym, st, g) for c in ("q8_0", "int8", "int8_s8") for asym in (False, True) for st in ("f32", "f16", "bf16")
           for g in (32, 64, 128, 256)]
K_G32 = [1056, 4000, 11008, 4096]      # partial 1024-byte super-blocks of the activation image (1056, 4000, 11008)
K_G = [4096, 11008, 2048, 5120]


def fmt_id(f):
    return f"{f[0]}-{'asym' if f[1] else 'sym'}-{f[2]}-g{f[3]}"


@pytest.mark.parametrize("i", range(len(FORMATS)), ids=[fmt_id(f) for f in FORMATS])
def test_formats_bitwise(i):
    """every compute type x zero points x scale type x group: ns_mul_mat at 1 and 2 rows (fused quantiser), the 4-row template at
    3 and 4 rows (NS_MM_FORCE_GEMV keeps them off the integer tensor cores), and a prepared single row"""
    comp, asym, st, g = FORMATS[i]
    k = (K_G32 if g == 32 else K_G)[i % 4]
    n = 301 + 2 * (i % 5)  # odd: the last row pair has one valid row
    w = RW(comp, n, k, g, asym, st, seed=100 + i)
    a = acts(4, k, 200 + i)
    want = w.model(a)
    for m in (1, 2, 3, 4):
        got, lc = mm(w, a[:m], flags=ns.MM_FORCE_GEMV)
        assert lc == -(-m // w.tile) * (1 if w.fused else 2), (m, lc)
        check_equal(got, want[:m], f"m={m} plan={w.plan(m, w.fused)}")
    got, _, lc = prepared([w], a[:1])
    assert lc == 2
    check_equal(got[:, :n], want[:1], f"prepared plan={w.plan(1, False)}")


@pytest.mark.parametrize("k", [1024, 4096, 11008, 14336])
def test_q4_0_ggml_bitwise(k):
    w = RW("q4_0", 4097, k, seed=k)
    a = acts(4, k, k + 1)
    want = w.model(a)
    for m in (1, 2, 3, 4):
        got, lc = mm(w, a[:m], flags=ns.MM_FORCE_GEMV)
        assert lc == -(-m // w.tile), (m, lc)  # one launch per tile (2 rows at K = 14336)
        check_equal(got, want[:m], f"m={m}")


def test_group_equal_to_k_prepared():
    """one group of K = 1000 (K not a multiple of 32): the prepared path, a partial last chunk, gi = 0 everywhere"""
    for comp, asym in (("int8", True), ("int8_s8", False)):
        w = RW(comp, 77, 1000, 1000, asym, "bf16", seed=7)
        assert not w.fused
        a = acts(2, 1000, 8)
        for m in (1, 2):
            got, lc = mm(w, a[:m], flags=ns.MM_FORCE_GEMV)
            assert lc == 2
            check_equal(got, w.model(a[:m]), comp)


# ------------------------------------------------------------------------------------------------ plan classes
CLASSES = [
    # (label, comp, k, g, stype, m, fused, plan)
    ("wide-pairs", "q4_0", 4096, 32, "f16", 1, True, (1, 2, 42, 14, 1)),
    ("wide-single-rows", "q4_0", 13824, 32, "f16", 1, True, (1, 1, 14, 14, 1)),
    ("wide-refused-odd-ring", "int8", 11008, 32, "f32", 1, True, (0, 2, 7, 7, 2)),
    ("two-cta-pairs", "q4_0", 4096, 32, "f16", 1, False, (0, 2, 21, 7, 2)),
    ("two-cta-single-rows-4-active", "int8", 28672, 32, "f32", 1, True, (0, 1, 4, 4, 2)),
    ("whole-sm-prepared", "int8", 32768, 32, "f32", 1, False, (0, 1, 7, 7, 1)),
    ("whole-sm-fused-wide-refused", "q4_0", 49152, 32, "f16", 1, True, (0, 1, 5, 5, 1)),
    ("m2-pairs", "q4_0", 4096, 32, "f16", 2, True, (0, 2, 21, 7, 2)),
    ("m2-single-rows", "int8", 11008, 32, "f32", 2, True, (0, 1, 7, 7, 2)),
    ("m3-in-m4", "int8", 11008, 128, "bf16", 3, True, (0, 1, 7, 7, 2)),
    ("m4-pairs", "int8_s8", 4096, 64, "f16", 4, True, (0, 2, 21, 7, 2)),
]


@pytest.mark.parametrize("case", CLASSES, ids=[c[0] for c in CLASSES])
def test_plan_classes_bitwise(case):
    label, comp, k, g, st, m, fused, plan = case
    w = RW(comp, 263, k, g, comp == "int8" and g == 128, st, seed=k + m)
    assert w.plan(m, fused) == plan, label
    a = acts(m, k, k + 5)
    if fused:
        got, lc = mm(w, a, flags=ns.MM_FORCE_GEMV)
        assert lc == 1
    else:
        got, _, lc = prepared([w], a)
        got = got[:, :w.n]
        assert lc == 2
    check_equal(got, w.model(a), label)


# ------------------------------------------------------------------------------------------------ n and the ring
@pytest.mark.parametrize("n", [1, 2, 3, 131, 263])
def test_small_n(n):
    """fewer rows (pairs) than CTAs: idle CTAs, one-row weights, odd n"""
    w = RW("int8", n, 4096, 128, True, "f16", seed=n)
    a = acts(2, 4096, n)
    want = w.model(a)
    for m in (1, 2):
        check_equal(mm(w, a[:m])[0], want[:m], f"fused m={m}")
    check_equal(prepared([w], a[:1])[0][:, :n], want[:1], "prepared")


@pytest.mark.parametrize("n", [32000, 32001])
def test_ring_wraps_many_times(n):
    """n = 32000 / 32001 at K = 4096: every CTA runs its ring around many times, on the wide kernel (fused single row) and on the
    two-CTA kernel (prepared image); both equal the model and each other"""
    w = RW("int8_s8", n, 4096, 128, False, "f16", seed=n)
    assert w.plan(1, True)[0] == 1 and w.plan(1, False)[0] == 0
    a = acts(1, 4096, 3)
    want = w.model(a)
    got_w, lc = mm(w, a)
    assert lc == 1
    check_equal(got_w, want, "wide")
    got_p = prepared([w], a)[0]
    check_equal(got_p, want, "two-cta")


# ------------------------------------------------------------------------------------------------ field extremes
def test_field_extremes():
    """u8 codes 0 and 255 (Sa up to 255 * 32 per chunk), s8 codes +-127, nibbles all 0 / all 15, zero points -8 and 7"""
    k, n, g = 2048, 40, 128
    rng = np.random.default_rng(11)
    q = rng.integers(-8, 8, (k, n)).astype(np.int8)
    zp = rng.integers(-8, 8, (k // g, n)).astype(np.int8)
    q[:, 0], zp[:, 0] = -8, 7      # nibble 0, q - zp = -15
    q[:, 1], zp[:, 1] = 7, -8      # nibble 15, q - zp = 15
    q[:, 2], zp[:, 2] = 7, 7
    q[:, 3], zp[:, 3] = -8, -8
    for comp in ("int8", "int8_s8"):
        w = RW(comp, n, k, g, True, "f32", q=q, zp=zp)
        a = acts(2, k, 12)
        a[0, :g] = 1.0                                    # u8: one code (255 or 0) over a block; s8: 127
        a[0, g:2 * g:2], a[0, g + 1:2 * g:2] = 1.0, -1.0  # codes at both ends
        a[1, :g] = -1.0
        codes, _, _ = oracle.imma_act(a, w.acomp, g)
        assert np.abs(codes).max() >= 127
        want = w.model(a)
        for m in (1, 2):
            check_equal(mm(w, a[:m])[0], want[:m], f"{comp} m={m}")
        check_equal(prepared([w], a[:1])[0], want[:1], f"{comp} prepared")


# ------------------------------------------------------------------------------------------------ invariance
def test_invariance_across_kernels_tiles_images_and_slots():
    """the same output row, bit-identical whichever way it is computed: wide vs two-CTA kernel, 1-, 2- and 4-row tiles (pairs vs
    single rows at K = 11008), plain vs the engine's kernel image, plain vs its QKV slot (no model involved)"""
    k = 11008
    w = RW("int8", 515, k, 128, True, "bf16", seed=21)
    a = acts(4, k, 22)
    assert w.plan(1, True)[:2] == (1, 2) and w.plan(1, False)[0] == 0
    assert w.plan(2, True)[1] == 2 and w.plan(4, True)[1] == 1
    one = mm(w, a[:1])[0]
    check_equal(prepared([w], a[:1])[0], one, "wide vs two-cta")
    check_equal(mm(w, a[:2])[0][:1], one, "1 vs 2 rows")
    check_equal(mm(w, a, flags=ns.MM_FORCE_GEMV)[0][:1], one, "1 vs 4 rows")
    eng, lc = mm(w, a[:1], engine=True)
    assert lc == 1
    check_equal(eng, one, "engine image")
    check_equal(mm(w, a[:2], engine=True)[0], mm(w, a[:2])[0], "engine image, 2 rows")
    wq, wk = RW("int8", 128, k, 128, True, "bf16", seed=23), RW("int8", 130, k, 128, True, "bf16", seed=24)
    x = dev(a[:2])
    out = torch.full((3, 2, 515), float("nan"), device="cuda")
    ns.mul_qkv(wq.w, wk.w, w.w, x.data_ptr(), k, out.data_ptr(), 515, 2)  # the odd-n weight in the last slot
    sync()
    o = out.cpu().numpy()
    for i, wi in enumerate((wq, wk, w)):
        check_equal(o[i, :, :wi.n], mm(wi, a[:2])[0], f"qkv slot {i}")
        assert np.isnan(o[i, :, wi.n:]).all()
    check_equal(mm(w, a[:1])[0], w.model(a[:1]), "model")


def test_gate_up_against_plain_gate_and_up():
    """ns_matmul_prepared mode 2: aux = silu(g) within ELT_ULPS of the fp32 SiLU of the plain gate, dst = fp32(aux * up_plain)"""
    E, F = 4096, 1030
    w1, w3 = RW("q4_0", F, E, seed=31), RW("q4_0", F, E, seed=32)
    a = acts(2, E, 33)
    for m in (1, 2):
        g = prepared([w1], a[:m])[0]
        u = prepared([w3], a[:m])[0]
        check_equal(g, w1.model(a[:m]), "gate")
        dst, aux, lc = prepared([w1, w3], a[:m], mode=2, aux=True)
        assert lc == 2
        want, scale = silu_f32(g)
        assert_ulps(aux, want, scale)
        check_equal(dst, aux * u, f"m={m}")


# ------------------------------------------------------------------------------------------------ epilogues and layout
def test_bias_residual_and_layout():
    """broadcast and per-row bias, residual: fl(fl(v + b) + r) on the plain result; lda > k, ldo > n with the columns past n
    left NaN"""
    n, k, ldo = 301, 4096, 320
    w = RW("int8_s8", n, k, 64, True, "f32", seed=41)
    rng = np.random.default_rng(42)
    a = acts(2, k, 43)
    bias_b = rng.normal(0, 1, n).astype(np.float32)
    bias_r = rng.normal(0, 1, (2, ldo)).astype(np.float32)
    res = rng.normal(0, 1, (2, ldo)).astype(np.float32)
    for m in (1, 2):
        plain = w.model(a[:m])
        got, lc = mm(w, a[:m], lda=k + 40, ldo=ldo, bias=bias_r[:m], residual=res[:m])
        assert lc == 1
        check_equal(got[:, :n], (plain + bias_r[:m, :n]) + res[:m, :n], "row bias + residual")
        assert np.isnan(got[:, n:]).all()
        got = mm(w, a[:m], ldo=ldo, bias=bias_b, bcast=True)[0]
        check_equal(got[:, :n], plain + bias_b, "broadcast bias")
        assert np.isnan(got[:, n:]).all()
        check_equal(mm(w, a[:m], engine=True, ldo=ldo, residual=res[:m])[0][:, :n], plain + res[:m, :n], "engine residual")


def test_gelu_plain_ffn():
    """ns_ffn_gelu without w3 at 1 and 2 rows: tmp = gelu(x W1^T + b1) within ELT_ULPS; dst = tmp W2^T + b2 bit-equal"""
    E, F = 1024, 768
    w1, w2 = RW("int8", F, E, 64, True, "f16", seed=51), RW("int8", E, F, 128, False, "f32", seed=52)
    rng = np.random.default_rng(53)
    b1, b2 = rng.normal(0, 1, F).astype(np.float32), rng.normal(0, 1, E).astype(np.float32)
    for m in (1, 2):
        a = acts(m, E, 54 + m)
        x, tmp, out = dev(a), torch.full((m, F), float("nan"), device="cuda"), torch.full((m, E), float("nan"), device="cuda")
        d1, d2 = dev(b1), dev(b2)
        torch.cuda.synchronize()
        lc = launches()
        ns.ffn_gelu(w1.w, w2.w, None, d1.data_ptr(), d2.data_ptr(), 1, x.data_ptr(), E, tmp.data_ptr(), out.data_ptr(), E, m)
        sync()
        assert launches() - lc == 2
        want, scale = gelu_f32(w1.model(a) + b1)
        t = tmp.cpu().numpy()
        assert_ulps(t, want, scale)
        check_equal(out.cpu().numpy(), w2.model(t) + b2, "down")


def test_qkv_gqa_odd_last_weight():
    E = 4096
    ws = [RW("q4_0", nn, E, seed=60 + i) for i, nn in enumerate((4096, 1024, 1023))]
    for m in (1, 2):
        a = acts(m, E, 63 + m)
        x = dev(a)
        out = torch.full((3, m, E), float("nan"), device="cuda")
        torch.cuda.synchronize()
        lc = launches()
        ns.mul_qkv(ws[0].w, ws[1].w, ws[2].w, x.data_ptr(), E, out.data_ptr(), E, m)
        sync()
        assert launches() - lc == 1
        o = out.cpu().numpy()
        for i, w in enumerate(ws):
            check_equal(o[i, :, :w.n], w.model(a), f"slot {i}")
            assert np.isnan(o[i, :, w.n:]).all()


# ------------------------------------------------------------------------------------------------ fused RMSNorm
def norm_model(w, a, nw, eps, nt):
    xn = np.stack([oracle.ring_norm_row(r, nw, eps, nt) for r in a])
    return w.model(xn)


@pytest.mark.parametrize("m,k", [(1, 10752), (1, 10784), (2, 5376), (2, 5408), (1, 4096), (2, 11008)])
@pytest.mark.parametrize("exact", [False, True], ids=["random", "exact"])
def test_fused_rmsnorm_bitwise(m, k, exact):
    """ns_rmsnorm_mul_mat against ring_norm_row + the quantiser + ring_stated, on both sides of the single/multi-pass boundary of
    the wide kernel (448 threads: 10752) and of the two-CTA kernel (224 threads: 5376)"""
    w = RW("q4_0", 515, k, seed=k + m)
    p = w.plan(m, True, norm=True)
    nt = 448 if p[0] else 224
    assert nt == (448 if m == 1 else 224)
    rng = np.random.default_rng(k + 7 * m)
    if exact:
        a = (rng.choice([-1.0, 1.0], (m, k)) * 2.0 ** rng.integers(-4, 4, (m, 1))).astype(np.float32)
        nw, eps = (2.0 ** rng.integers(-2, 3, k)).astype(np.float32), 0.0
        xn = np.stack([oracle.ring_norm_row(r, nw, eps, nt) for r in a])
        assert np.array_equal(xn, np.sign(a) * nw)
    else:
        a = rng.normal(0, 2, (m, k)).astype(np.float32)
        nw, eps = rng.uniform(0.5, 1.5, k).astype(np.float32), 1e-5
    res = rng.normal(0, 1, (m, w.n)).astype(np.float32)
    x, nd, r = dev(a), dev(nw), dev(res)
    out = torch.full((m, w.n), float("nan"), device="cuda")
    torch.cuda.synchronize()
    lc = launches()
    ns.rmsnorm_mul_mat(w.w, x.data_ptr(), k, nd.data_ptr(), eps, out.data_ptr(), w.n, m, r.data_ptr())
    sync()
    assert launches() - lc == 1
    check_equal(out.cpu().numpy(), norm_model(w, a, nw, eps, nt) + res, f"plan={p}")


def test_fused_rmsnorm_qkv_and_ffn():
    """the norm folded into the QKV launch and into the FFN's gate/up launch (1 and 2 rows, multi-pass on both kernels)"""
    E, KV, F = 11008, 512, 1024
    ws = [RW("int8", nn, E, 128, True, "bf16", seed=70 + i) for i, nn in enumerate((1024, KV, KV - 1))]
    w1, w3 = RW("int8", F, E, 128, True, "bf16", seed=74), RW("int8", F, E, 128, True, "bf16", seed=75)
    w2 = RW("int8", E, F, 128, False, "f32", seed=76)
    rng = np.random.default_rng(77)
    nw, eps = rng.uniform(0.5, 1.5, E).astype(np.float32), 1e-6
    for m in (1, 2):
        nt = 448 if ws[0].plan(m, True, mode=1, norm=True)[0] else 224
        a = rng.normal(0, 1, (m, E)).astype(np.float32)
        x, nd = dev(a), dev(nw)
        out = torch.full((3, m, 1024), float("nan"), device="cuda")
        ns.rmsnorm_mul_qkv(ws[0].w, ws[1].w, ws[2].w, x.data_ptr(), E, nd.data_ptr(), eps, out.data_ptr(), 1024, m)
        sync()
        o = out.cpu().numpy()
        for i, w in enumerate(ws):
            check_equal(o[i, :, :w.n], norm_model(w, a, nw, eps, nt), f"qkv m={m} slot {i}")
        nt = 448 if w1.plan(m, True, mode=2, norm=True)[0] else 224
        res = rng.normal(0, 1, (m, E)).astype(np.float32)
        tmp, dst, r = torch.zeros(2 * m * F, device="cuda"), torch.full((m, E), float("nan"), device="cuda"), dev(res)
        torch.cuda.synchronize()
        lc = launches()
        ns.rmsnorm_ffn_silu(w1.w, w2.w, w3.w, x.data_ptr(), E, nd.data_ptr(), eps, tmp.data_ptr(), dst.data_ptr(), E, m, r.data_ptr())
        sync()
        assert launches() - lc == 2
        g, u = norm_model(w1, a, nw, eps, nt), norm_model(w3, a, nw, eps, nt)
        mid = tmp.cpu().numpy()[:m * F].reshape(m, F)
        s, scale = silu_f32(g)
        assert_ulps(mid, s * u, scale * np.abs(u) + np.abs(s * u))
        check_equal(dst.cpu().numpy(), w2.model(mid) + res, f"ffn down m={m}")


# ------------------------------------------------------------------------------------------------ chains, graphs, workspace
def test_chains_under_pdl_and_graphs():
    """square nodes back to back in one stream, each output feeding the next node's activations and residual, fused and prepared
    (one shared workspace), eagerly and replayed from a captured graph: bit-equal to the same nodes with a synchronise between"""
    L = ns.lib()
    k, depth = 4096, 4
    nodes = [RW("q4_0", k, k, seed=80 + i) for i in range(depth)] + [RW("int8", k, k, 128, True, "f16", seed=90 + i)
                                                                     for i in range(depth)]
    x0 = dev(acts(1, k, 85) * 0.05)
    bufs = [torch.zeros((1, k), device="cuda") for _ in range(2 * depth)]
    wsb = torch.zeros(L.ns_device_workspace_bytes(1, k), dtype=torch.uint8, device="cuda")
    s = torch.cuda.Stream()

    def run(between=None, prep=False):
        q = C.c_void_p(s.cuda_stream)
        src = x0
        for i, w in enumerate(nodes):
            dst = bufs[i]
            if prep:
                assert L.ns_prepare_activation(w.w.h, C.c_void_p(src.data_ptr()), k, 1, C.c_void_p(wsb.data_ptr()), q) == 0
                hs = (C.c_void_p * 1)(w.w.h)
                assert L.ns_matmul_prepared(hs, 1, 0, C.c_void_p(wsb.data_ptr()), C.c_void_p(dst.data_ptr()), k, 1, None, 0,
                                            C.c_void_p(src.data_ptr()), None, q) == 0, ns.last_error()
            else:
                ns.mul_mat(w.w, src.data_ptr(), k, dst.data_ptr(), k, 1, None, src.data_ptr(), 0, ws_ptr=wsb.data_ptr(), queue=q)
            if between:
                between()
            src = dst

    s.wait_stream(torch.cuda.current_stream())
    for prep in (False, True):
        with torch.cuda.stream(s):
            run(between=s.synchronize, prep=prep)
        s.synchronize()
        want = [b.cpu().numpy() for b in bufs]
        assert all(np.isfinite(v).all() for v in want)
        for b in bufs:
            b.fill_(float("nan"))
        torch.cuda.synchronize()
        with torch.cuda.stream(s):
            run(prep=prep)
        s.synchronize()
        for i, b in enumerate(bufs):
            check_equal(b.cpu().numpy(), want[i], f"eager prep={prep} node {i}")
        q = C.c_void_p(s.cuda_stream)
        with torch.cuda.stream(s):
            assert L.ns_graph_begin(q) == 0
            run(prep=prep)
            gr = L.ns_graph_end(q)
        assert gr, ns.last_error()
        for _ in range(2):
            for b in bufs:
                b.fill_(float("nan"))
            torch.cuda.synchronize()
            assert L.ns_graph_launch(gr, q) == 0
            s.synchronize()
            for i, b in enumerate(bufs):
                check_equal(b.cpu().numpy(), want[i], f"graph prep={prep} node {i}")
        L.ns_graph_free(gr)
    # the first node on its own against the model: the chain is not trivially self-consistent
    check_equal(want[0], nodes[0].model(x0.cpu().numpy()) + x0.cpu().numpy(), "node 0")


def test_workspace_exact_size_leaves_guard_bytes():
    """prepared tiles of up to 4 rows in exactly ns_device_workspace_bytes(m, k) bytes: the bytes after it are never written"""
    L = ns.lib()
    for comp, k, g in (("int8", 11008, 128), ("q8_0", 14336, 32), ("int8_s8", 1000, 1000)):
        w = RW(comp, 96, k, g, comp != "q8_0", "bf16", seed=k)
        for m in (1, 2, 3, 4):
            if m > (1 if k == 14336 else 4):
                continue
            a = acts(m, k, 100 + m)
            nbytes = L.ns_device_workspace_bytes(m, k)
            buf = torch.full((nbytes + 4096,), 0xA5, dtype=torch.uint8, device="cuda")
            x = dev(a)
            out = torch.full((m, 96), float("nan"), device="cuda")
            assert L.ns_prepare_activation(w.w.h, C.c_void_p(x.data_ptr()), k, m, C.c_void_p(buf.data_ptr()), None) == 0, ns.last_error()
            hs = (C.c_void_p * 1)(w.w.h)
            assert L.ns_matmul_prepared(hs, 1, 0, C.c_void_p(buf.data_ptr()), C.c_void_p(out.data_ptr()), 96, m, None, 0, None, None,
                                        None) == 0
            sync()
            assert (buf[nbytes:].cpu().numpy() == 0xA5).all(), (comp, m)
            check_equal(out.cpu().numpy(), w.model(a), f"{comp} m={m}")


# ------------------------------------------------------------------------------------------------ nodes without a plan
def test_unplannable_plain_node_is_refused_before_any_launch():
    L = ns.lib()
    k = 131072
    for g, stype in ((32, ns.S_F32), (k, ns.S_F32)):   # fused quantiser; one group of K (prepared image: act_prep would run first)
        w = ns.Weight.random(8, k, g, ns.W_S4, stype, ns.COMP_INT8, False, 3)
        out = (C.c_int * 5)()
        assert L.ns_gemv_ring_plan(k, g, stype, 0, ns.COMP_INT8, 0, 1, 1 if g == 32 else 0, 0, out) == 0
        x, y = torch.zeros((1, k), device="cuda"), torch.zeros((1, 8), device="cuda")
        torch.cuda.synchronize()
        lc = launches()
        rc = L.ns_mul_mat(w.h, C.c_void_p(x.data_ptr()), k, C.c_void_p(y.data_ptr()), 8, 1, None, None, 0, None, None)
        sync()
        assert rc == E_UNSUPPORTED and launches() - lc == 0, (rc, launches() - lc)
        assert "ring GEMV" in ns.last_error(), ns.last_error()


def test_ffn_with_unplannable_down_is_refused_before_gate_up_runs():
    L = ns.lib()
    E, F = 256, 131072
    w1, w3 = (ns.Weight.random(F, E, 32, ns.W_S4, ns.S_F32, ns.COMP_INT8, False, s) for s in (1, 2))
    w2 = ns.Weight.random(E, F, 32, ns.W_S4, ns.S_F32, ns.COMP_INT8, False, 3)
    out = (C.c_int * 5)()
    assert L.ns_gemv_ring_plan(E, 32, ns.S_F32, 0, ns.COMP_INT8, 2, 1, 1, 0, out) == 1
    assert L.ns_gemv_ring_plan(F, 32, ns.S_F32, 0, ns.COMP_INT8, 0, 1, 1, 0, out) == 0
    x, tmp, y = torch.zeros((1, E), device="cuda"), torch.zeros(2 * F, device="cuda"), torch.zeros((1, E), device="cuda")
    torch.cuda.synchronize()
    lc = launches()
    rc = L.ns_ffn_silu(w1.h, w2.h, w3.h, C.c_void_p(x.data_ptr()), E, C.c_void_p(tmp.data_ptr()), C.c_void_p(y.data_ptr()), E, 1,
                       None, None)
    sync()
    assert rc == E_UNSUPPORTED and launches() - lc == 0, (rc, launches() - lc)
    assert "ring GEMV" in ns.last_error(), ns.last_error()

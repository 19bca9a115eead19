"""Every activation quantiser that feeds a matmul, held bit-exact against the oracle's quantize_row_q8_0 /
quantize_fp_u8_colblock / quantize_fp_s8_colblock.

The codes are read back through real matmuls with an identity weight: n = k, code 1 on the diagonal, weight scale 1.0 (or the
Q4_0 quantisation of the identity: code -8, scale -1/8).  Output j is then (q_j - za) * a_scale of the block holding j: every
block sum is an exact integer, every other block contributes an exact zero, and the one product is rounded once, as numpy
rounds it.  So the bar is np.array_equal.  Each case also pins its kernel path by its launch count (test_gpu_routing.py).

Paths: the ring GEMV's in-kernel quantiser (one CTA per SM at m = 1, two at m = 2), with and without the fused RMSNorm;
act_quant_kernel in the ring layout (ns_prepare_activation + ns_matmul_prepared, and K with a partial last block) and in
natural rows (8-bit weights); the IMMA kernel's quantiser at m = 3, 8, 32.
"""
import ctypes as C

import numpy as np
import pytest

import oracle
import neural_speed_b200 as ns

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

EPS = 1e-6
COMPS = {"q8_0": ns.COMP_Q8_0, "int8": ns.COMP_INT8, "int8_s8": ns.COMP_INT8_S8}


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def counted(fn):
    torch.cuda.synchronize()
    lc = ns.lib().ns_launch_count()
    fn()
    ns.lib().bestla_device_sync(None)
    return ns.lib().ns_launch_count() - lc


def block_of(comp, g):
    return 32 if comp == "q8_0" else g  # ggml's Q8_0 block is always 32


def acts(m, k, qb, seed, grid=None):
    """Per row: a zero block, an all-positive block, an all-negative block, a block on a 1/8 grid; row 1 is all positive.
    grid: every value on that dyadic grid (the fused-norm case)."""
    rng = np.random.default_rng(seed)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    if grid:
        a = np.round(a * grid) / grid
    a[:, :qb] = 0
    a[:, qb:2 * qb] = np.abs(a[:, qb:2 * qb])
    a[:, 2 * qb:3 * qb] = -np.abs(a[:, 2 * qb:3 * qb])
    a[:, 3 * qb:4 * qb] = np.round(a[:, 3 * qb:4 * qb] * 8) / 8
    if m > 1:
        a[1] = np.abs(a[1])
    return a.astype(np.float32)


def want(a, comp, g):
    """(q - za) * a_scale per element, float32, from the oracle's quantiser"""
    m, k = a.shape
    if comp == "q8_0":
        blocks = oracle.quantize_q8_0(a).reshape(m, k // 32, 34)
        q = blocks[:, :, 2:].copy().view(np.int8).reshape(m, k).astype(np.float32)
        d = blocks[:, :, :2].copy().view(np.float16).reshape(m, k // 32).astype(np.float32)
        return q * np.repeat(d, 32, axis=1)
    if comp == "int8":
        q, sc, zp = oracle.btla_quantize_act_u8(a, g)
        qa = q.astype(np.float32) - np.repeat(zp.astype(np.float32), g, axis=1)[:, :k]
    else:
        q, sc = oracle.btla_quantize_act_s8(a, g)
        qa = q.astype(np.float32)
    return qa * np.repeat(sc.astype(np.float32), g, axis=1)[:, :k]


_W = {}


def identity(k, g, comp, wfmt=ns.W_S4):
    key = (k, g, comp, wfmt)
    if key not in _W:
        if g is None:  # ggml Q4_0 of the identity
            _W[key] = ns.Weight.from_q4_0_host(oracle.quantize_q4_0(np.eye(k, dtype=np.float32)), k, k)
        else:
            _W[key] = ns.Weight.from_unpacked(np.eye(k, dtype=np.int8), np.ones((-(-k // g), k), np.float32), None, g, wfmt,
                                              ns.S_F32, COMPS[comp])
    return _W[key]


def mul_mat(w, a):
    m, k = a.shape
    x = dev(a)
    out = torch.full((m, w.n), float("nan"), device="cuda")
    n = counted(lambda: ns.mul_mat(w, x.data_ptr(), k, out.data_ptr(), w.n, m))
    return out.cpu().numpy(), n


def check(got, a, comp, g):
    exp = want(a, comp, g)
    bad = np.argwhere(got != exp)
    assert bad.size == 0, (len(bad), bad[:4].tolist(), got[tuple(bad[0])], exp[tuple(bad[0])])


CASES = [(c, g) for c in ("q8_0", "int8", "int8_s8") for g in (32, 128)]


@pytest.mark.parametrize("comp,g", CASES)
@pytest.mark.parametrize("m", [1, 2])
def test_ring_in_kernel_quantiser(comp, g, m):
    k = 2048
    a = acts(m, k, block_of(comp, g), 10 + m)
    got, n = mul_mat(identity(k, g, comp), a)
    assert n == 1  # the ring GEMV quantises its own activations
    check(got, a, comp, g)


@pytest.mark.parametrize("m", [1, 2])
def test_ring_in_kernel_quantiser_q4_0(m):
    k = 2048
    a = acts(m, k, 32, 20 + m)
    got, n = mul_mat(identity(k, None, "q8_0"), a)
    assert n == 1
    check(got, a, "q8_0", 32)


@pytest.mark.parametrize("comp,g", CASES)
def test_ring_norm_fused_quantiser(comp, g):
    """k a power of two and dyadic inputs: the sum of squares is exact in any order, so 1/rms is the numpy float32 value"""
    k = 2048
    rng = np.random.default_rng(30)
    x = acts(1, k, block_of(comp, g), 31, grid=8)
    nw = (rng.integers(1, 24, k) / 8).astype(np.float32)
    w = identity(k, g, comp)
    assert ns.rmsnorm_fusable([w], 1)
    xd, nwd = dev(x), dev(nw)
    out = torch.full((1, k), float("nan"), device="cuda")
    n = counted(lambda: ns.rmsnorm_mul_mat(w, xd.data_ptr(), k, nwd.data_ptr(), EPS, out.data_ptr(), k, 1))
    assert n == 1
    ss = np.float32((x.astype(np.float64) ** 2).sum())
    assert float(ss) == (x.astype(np.float64) ** 2).sum()
    inv = np.float32(1) / np.sqrt(ss / np.float32(k) + np.float32(EPS))
    y = ((x * inv) * nw).astype(np.float32)
    check(out.cpu().numpy(), y, comp, g)


@pytest.mark.parametrize("comp,g", CASES)
def test_act_prep_ring_layout_prepared(comp, g):
    L = ns.lib()
    k, m = 2048, 3
    a = acts(m, k, block_of(comp, g), 40)
    w = identity(k, g, comp)
    x = dev(a)
    ws = torch.zeros(L.ns_device_workspace_bytes(m, k), dtype=torch.uint8, device="cuda")
    out = torch.full((m, k), float("nan"), device="cuda")
    wl = (C.c_void_p * 1)(w.h.value)

    def run():
        assert L.ns_prepare_activation(w.h, C.c_void_p(x.data_ptr()), k, m, C.c_void_p(ws.data_ptr()), None) == 0, ns.last_error()
        assert L.ns_matmul_prepared(wl, 1, 0, C.c_void_p(ws.data_ptr()), C.c_void_p(out.data_ptr()), k, m, None, 0, None, None,
                                    None) == 0, ns.last_error()
    assert counted(run) == 2
    check(out.cpu().numpy(), a, comp, g)


@pytest.mark.parametrize("comp", ["int8", "int8_s8"])
@pytest.mark.parametrize("wfmt", [ns.W_S4, ns.W_S8])
@pytest.mark.parametrize("m", [1, 2])
def test_act_prep_partial_last_block(comp, wfmt, m):
    """k = 1500, blocks of 128: the last block holds 92 values (quantize_fp_u8_colblock starts its range at 0).  The ring's
    in-kernel quantiser takes whole blocks only, so both weight formats run act_quant_kernel: ring layout for 4-bit weights,
    natural rows for 8-bit ones."""
    k, g = 1500, 128
    a = acts(m, k, g, 50 + m)
    a[:, 1408:] = -np.abs(a[:, 1408:]) - 0.25  # all-negative tail: vmax stays at its start value (0, not FLT_MIN)
    got, n = mul_mat(identity(k, g, comp, wfmt), a)
    assert n == 2  # act_prep + GEMV
    check(got, a, comp, g)


@pytest.mark.parametrize("comp,g", CASES)
def test_act_prep_natural_rows(comp, g):
    k, m = 2048, 2
    a = acts(m, k, block_of(comp, g), 60)
    got, n = mul_mat(identity(k, g, comp, ns.W_S8), a)
    assert n == 2
    check(got, a, comp, g)


@pytest.mark.parametrize("comp,g", CASES)
@pytest.mark.parametrize("m", [3, 8, 32])
def test_imma_quantiser(comp, g, m):
    k = 2048
    a = acts(m, k, block_of(comp, g), 70 + m)
    got, n = mul_mat(identity(k, g, comp), a)
    assert n == 2  # activation image + IMMA GEMM (the bf16 GEMM would not be exact)
    check(got, a, comp, g)

"""Which kernel path every public matmul node takes, pinned by launch counts (DESIGN.md section 4).

The path fixes the numerics class of a call, so it must be a function of (format, m, flags) only:
  Q6_K weights (plain nodes)                      Q6_K kernel, tiles of <= 4 rows (2 launches per tile)
  3 <= m <= 32, int4 weights, integer compute     integer tensor cores (IMMA): 2 launches per launch set; FFN: both halves or neither
                                                  (GEMV tiles when its shared-memory planner cannot fit a launch of the node)
  m > 16 or NS_MM_FORCE_TC                        wgmma GEMM (bf16): activation image + one GEMM per weight
  otherwise, or NS_MM_FORCE_GEMV                  GEMV tiles of <= 4 rows: 1 launch per tile on the ring (int4 weights with an
                                                  integer compute type quantise their own activations), else act_prep + GEMV
A plain IMMA node and a plain wgmma node both issue two launches; there the numerics class tells them apart: the integer paths
agree with the forced GEMV to fp32 summation order (2e-6), the bf16 GEMM does not.  An RMSNorm folds into the ring GEMV only.
"""
import ctypes as C
import functools

import numpy as np
import pytest

import neural_speed_b200 as ns
import oracle

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

N, K, FMID = 256, 1024, 512
MS = [1, 2, 3, 4, 5, 16, 17, 32, 33, 64]
FLAGS = [0, ns.MM_FORCE_GEMV, ns.MM_FORCE_TC]
FMTS = ["q4_0", "int4_g128_asym", "nf4_bf16", "int8_f32", "q6_K"]
RING = {"q4_0", "int4_g128_asym"}  # int4 weights with an integer compute type: the ring GEMV and the integer tensor cores
E_UNSUPPORTED = -4


@pytest.fixture(scope="module", autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


@functools.lru_cache(maxsize=None)
def weight(fmt, n, k, seed):
    w = np.random.default_rng(seed).normal(0, 0.05, (n, k)).astype(np.float32)
    if fmt == "q4_0":
        return ns.Weight.from_q4_0_host(oracle.quantize_q4_0(w), n, k)
    if fmt == "q6_K":
        return ns.Weight.from_q6_K_host(oracle.quantize_q6_K(w), n, k)
    args = {"int4_g128_asym": ("int4", 128, "asym", "fp32", "int8"), "nf4_bf16": ("nf4", 32, "sym", "fp32", "bf16"),
            "int8_f32": ("int8", 32, "sym", "fp32", "fp32")}[fmt]
    return ns.Weight.from_blob(ns.np_bestla_quantize(w, *args))


def route(fmt, m, flags=0):
    if fmt == "q6_K":
        return "q6k"
    if flags == 0 and fmt in RING and 3 <= m <= 32:
        return "imma"
    if not flags & ns.MM_FORCE_GEMV and (m > 16 or flags & ns.MM_FORCE_TC):
        return "tc"
    return "gemv"


def gemv_launches(fmt, m):
    return -(-m // 4) * (1 if fmt in RING else 2)


def plain_launches(fmt, m, flags=0):
    return {"q6k": 2 * -(-m // 4), "imma": 2, "tc": 2, "gemv": gemv_launches(fmt, m)}[route(fmt, m, flags)]


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def counted(fn):
    torch.cuda.synchronize()
    lc = ns.lib().ns_launch_count()
    rc = fn()
    ns.lib().bestla_device_sync(None)
    return rc, ns.lib().ns_launch_count() - lc


def act(m, k=K, seed=0):
    return dev(np.random.default_rng(1000 + m + seed).normal(0, 1, (m, k)))


def rel_diff(a, b):
    return float(np.abs(a - b).max()) / (float(np.abs(b).max()) + 1e-30)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("m", MS)
def test_mul_mat_route(fmt, m):
    w, x = weight(fmt, N, K, 1), act(m)
    outs = {}
    for flags in FLAGS:
        out = torch.full((m, N), float("nan"), device="cuda")
        _, n = counted(lambda: ns.mul_mat(w, x.data_ptr(), K, out.data_ptr(), N, m, flags=flags))
        assert n == plain_launches(fmt, m, flags), (flags, n)
        outs[flags] = out.cpu().numpy()
    ref = outs[ns.MM_FORCE_GEMV]
    for flags in (0, ns.MM_FORCE_TC):
        r = route(fmt, m, flags)
        if r == "q6k":
            assert np.array_equal(outs[flags], ref)
        elif r == "imma":
            assert rel_diff(outs[flags], ref) <= 2e-6
        elif r == "tc" and fmt in RING:
            assert rel_diff(outs[flags], ref) > 2e-6  # bf16 numerics, not the integer block sums


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("m", MS)
def test_mul_mat_id_route(fmt, m):
    """two experts, tokens already grouped (no gather / scatter): each expert's slice is routed by its own height"""
    experts = [weight(fmt, N, K, 1), weight(fmt, N, K, 2)]
    c0 = (m + 1) // 2
    ids = np.array([[0]] * c0 + [[1]] * (m - c0), np.int32)
    x = act(m)
    for flags in FLAGS:
        out = torch.full((m, N), float("nan"), device="cuda")
        _, n = counted(lambda: ns.mul_mat_id(experts, ids, 0, x.data_ptr(), K, out.data_ptr(), N, m, flags=flags))
        want = plain_launches(fmt, c0, flags) + (plain_launches(fmt, m - c0, flags) if m > c0 else 0)
        assert n == want, (flags, n)


@pytest.mark.parametrize("fmt", FMTS[:4])
@pytest.mark.parametrize("m", MS)
def test_mul_qkv_route(fmt, m):
    ws, x = [weight(fmt, N, K, s) for s in (1, 2, 3)], act(m)
    out = torch.full((3, m, N), float("nan"), device="cuda")
    _, n = counted(lambda: ns.mul_qkv(*ws, x.data_ptr(), K, out.data_ptr(), N, m))
    assert n == {"imma": 2, "tc": 4, "gemv": gemv_launches(fmt, m)}[route(fmt, m)], n


def ffn_launches(fmt, m, w3):
    # TC: activation image, gate (and up) GEMMs, SiLU*mul or GELU, down activation image, down GEMM
    return {"imma": 4, "tc": 6 if w3 else 5, "gemv": 2 * gemv_launches(fmt, m)}[route(fmt, m)]


@pytest.mark.parametrize("fmt", FMTS[:4])
@pytest.mark.parametrize("m", MS)
def test_ffn_route(fmt, m):
    w1, w3, w2 = weight(fmt, FMID, K, 4), weight(fmt, FMID, K, 5), weight(fmt, K, FMID, 6)
    x = act(m)
    tmp = torch.zeros(2 * m * FMID, device="cuda")
    b1, b2 = dev(np.linspace(-1, 1, FMID)), dev(np.linspace(-1, 1, K))
    cases = [("silu", lambda out: ns.ffn_silu(w1, w2, w3, x.data_ptr(), K, tmp.data_ptr(), out.data_ptr(), K, m), True),
             ("gelu_mul", lambda out: ns.ffn_gelu(w1, w2, w3, None, None, 0, x.data_ptr(), K, tmp.data_ptr(), out.data_ptr(), K, m), True),
             ("gelu", lambda out: ns.ffn_gelu(w1, w2, None, None, None, 0, x.data_ptr(), K, tmp.data_ptr(), out.data_ptr(), K, m), False),
             ("add_gelu", lambda out: ns.ffn_gelu(w1, w2, None, b1.data_ptr(), b2.data_ptr(), 1, x.data_ptr(), K, tmp.data_ptr(),
                                                  out.data_ptr(), K, m), False)]
    for name, fn, has_w3 in cases:
        out = torch.full((m, K), float("nan"), device="cuda")
        _, n = counted(lambda: fn(out))
        assert n == ffn_launches(fmt, m, has_w3), (name, n)


@pytest.mark.parametrize("fmt", FMTS)
@pytest.mark.parametrize("m", MS)
def test_rmsnorm_route(fmt, m):
    """the norm folds into the ring GEMV (decode rows the integer tensor cores do not take); elsewhere the entries fail loudly"""
    L = ns.lib()
    fold = fmt in RING and m <= 2
    w = weight(fmt, N, K, 1)
    assert ns.rmsnorm_fusable([w], m) == fold
    x, nw = act(m), dev(np.ones(K))
    p = lambda t: C.c_void_p(t.data_ptr())
    out = torch.zeros(3 * m * K, device="cuda")
    rc, n = counted(lambda: L.ns_rmsnorm_mul_mat(w.h, p(x), K, p(nw), 1e-6, p(out), N, m, None, None, None))
    assert (rc, n) == ((0, 1) if fold else (E_UNSUPPORTED, 0))
    if fmt == "q6_K":
        return
    qkv = [weight(fmt, N, K, s) for s in (1, 2, 3)]
    assert ns.rmsnorm_fusable(qkv, m) == fold
    rc, n = counted(lambda: L.ns_rmsnorm_mul_qkv(*[w.h for w in qkv], p(x), K, p(nw), 1e-6, p(out), N, m, None, None))
    assert (rc, n) == ((0, 1) if fold else (E_UNSUPPORTED, 0))
    w1, w3, w2 = weight(fmt, FMID, K, 4), weight(fmt, FMID, K, 5), weight(fmt, K, FMID, 6)
    assert ns.rmsnorm_fusable([w1, w3], m) == fold
    tmp = torch.zeros(2 * m * FMID, device="cuda")
    rc, n = counted(lambda: L.ns_rmsnorm_ffn_silu(w1.h, w2.h, w3.h, p(x), K, p(nw), 1e-6, p(tmp), p(out), K, m, None, None, None))
    assert (rc, n) == ((0, 2) if fold else (E_UNSUPPORTED, 0))

"""ggml Q8_0 weights on the device: load, the ring GEMV, the integer tensor cores, the wgmma GEMM, the host drop-in and the eval step.

Arithmetic (DESIGN.md section 4, tests/q8_0_model.py):
  ring GEMV   per 32-chunk an exact isum_c = sum a*q, t_c = fp32(a_d * w_d), lane L: acc = fmaf(isum_c, t_c, acc) over
              c = L, L + 32, ...; the xor butterfly combines the lanes -- bit for bit (q8.ring_stated).
  IMMA        the same exact block sums, summed per split in block order: bit for bit on exact constructions, within
              gamma_n sum |t_b| on random data (oracle.imma_bound_ratio).
  wgmma       code exact in bf16 times the bf16-rounded d: within the bf16 bar the int4 GEMM is held to.
Where every fp32 partial sum is exact (power-of-two scales, small codes), every path equals the reference's ne_vec_dot_q8_0_q8_0
bit for bit.  The eval step is held to the running bar of tests/llama_models.py against the Q8_0 CPU graph, and at Llama-2-7B
shapes against the reference's own engine."""
import ctypes as C

import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
import oracle
import q8_0_model as q8
from llama_models import RunningBar, check_logits, close, distance, scale, toy, unambiguous
from oracle.llama_model import greedy

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


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def rand_rows(rng, n, k, sd=0.02):
    return q8.quantize_weights(rng.normal(0, sd, (n, k)).astype(np.float32))


def run(w, a, flags=0):
    """ns_mul_mat -> (out, launches)"""
    x = dev(a.astype(np.float32))
    m = a.shape[0]
    out = torch.full((m, w.n), float("nan"), device="cuda")
    torch.cuda.synchronize()
    lc = ns.lib().ns_launch_count()
    ns.mul_mat(w, x.data_ptr(), w.k, out.data_ptr(), w.n, m, flags=flags)
    sync()
    return out.cpu().numpy(), ns.lib().ns_launch_count() - lc


def exact_case(rng, n, k, m):
    """power-of-two scales and codes whose Q8_0 quantisation is exact; sum |t_b| stays below 2^24 units, so every fp32 sum is exact"""
    q = rng.integers(-7, 8, (n, k))
    d = np.full((n, k // 32), 2.0 ** -8, np.float32)
    rows = q8.join(q, d)
    codes = rng.integers(-127, 128, (m, k)).astype(np.float32)
    codes.reshape(m, k // 32, 32)[:, :, 0] = 127.0          # amax = 127 units in every block: d_a = 2^-6, id = 2^6
    a = codes * np.float32(2.0 ** -6)
    assert np.abs(q).sum(axis=1).max() * 127 < 2 ** 24
    return rows, a


# ------------------------------------------------------------------------------------------------------------- load
@pytest.mark.parametrize("n,k,pad", [(64, 4096, 0), (33, 352, 0), (7, 1056, 34), (130, 11008, 6)])
def test_load_dequant_exact(n, k, pad):
    rng = np.random.default_rng(n + k)
    rows = rand_rows(rng, n, k, 0.05)
    q, d = q8.split(rows, k)
    q[0, :32] = -128
    d[1, 0] = np.float32(np.float16(2.0 ** -24))             # subnormal fp16 d
    d[2 % n, 1] = 0.0
    rows = q8.join(q, d)
    nb01 = rows.shape[1] + pad
    padded = np.zeros((n, nb01), np.uint8)
    padded[:, :rows.shape[1]] = rows
    want = q8.dequantize(rows, k)
    host = ns.Weight.from_q8_0_host(padded, n, k)          # the row stride is the array's: nb01 > the row's 34 * k / 32 bytes
    rdev = dev(padded)
    wdev = ns.Weight.from_q8_0_device(rdev.data_ptr(), n, k, nb01)
    for w in (host, wdev):
        assert (w.n, w.k, w.group, w.wfmt, w.stype, w.comp, w.asym) == (n, k, 32, ns.W_Q8_0, ns.S_F16, ns.COMP_Q8_0, 0)
        assert w.algorithmic_bytes == n * k + n * k // 32 * 2
        out = torch.full((n, k), float("nan"), device="cuda")
        assert ns.lib().ns_weight_dequant_f32(w.h, C.c_void_p(out.data_ptr()), k, None) == 0
        sync()
        assert np.array_equal(bits(out.cpu().numpy()), bits(want))
    assert ns.lib().ns_weight_set_comp(host.h, ns.COMP_INT8) == -4
    assert not ns.lib().ns_weight_from_q8_0(rows.ctypes.data_as(C.c_void_p), n, k + 16, rows.shape[1], 0, None)
    # the repack reads 16-bit words: an odd row stride or an odd device address is refused before anything launches
    odd = np.zeros((n, rows.shape[1] + 1), np.uint8)
    odd[:, :rows.shape[1]] = rows
    assert not ns.lib().ns_weight_from_q8_0(odd.ctypes.data_as(C.c_void_p), n, k, odd.shape[1], 0, None)
    assert "aligned" in ns.last_error()
    assert not ns.lib().ns_weight_from_q8_0(C.c_void_p(rdev.data_ptr() + 1), n, k, nb01, 1, None)
    assert not ns.lib().ns_weight_from_q4_0(C.c_void_p(rdev.data_ptr() + 1), n, k, nb01, 1, None)


# ------------------------------------------------------------------------------------------------------------- ring GEMV
@pytest.mark.parametrize("k", [4096, 11008, 352])
@pytest.mark.parametrize("m", [1, 2, 3, 4])
def test_ring_plain_bitwise(k, m):
    """ns_mul_mat of <= 4 rows (FORCE_GEMV keeps 3 and 4 rows off the integer tensor cores): one launch per tile, the kernel
    quantises its own activations; m = 1 runs the one-CTA-per-SM kernel, 2..4 rows the two-CTA kernel"""
    rng = np.random.default_rng(k + m)
    n = 300 if k != 11008 else 4096
    rows = rand_rows(rng, n, k)
    w = ns.Weight.from_q8_0_host(rows, n, k)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    got, launches = run(w, a, ns.MM_FORCE_GEMV)
    assert launches == 1
    assert np.array_equal(bits(got), bits(q8.ring_stated(a, rows)))


def prepared(ws, mode, a, ldo, aux=False):
    """ns_prepare_activation + ns_matmul_prepared: the two-CTA kernel on a pre-quantised image"""
    L = ns.lib()
    m, k = a.shape
    x = dev(a)
    wsb = torch.zeros(int(L.ns_device_workspace_bytes(4, k)) // 4 + 64, device="cuda")
    assert L.ns_prepare_activation(ws[0].h, C.c_void_p(x.data_ptr()), k, m, C.c_void_p(wsb.data_ptr()), None) == 0, ns.last_error()
    rows_out = len(ws) * m if mode == 1 else m
    out = torch.full((rows_out, ldo), float("nan"), device="cuda")
    ax = torch.full((m, ldo), float("nan"), device="cuda") if aux else None
    hs = (C.c_void_p * len(ws))(*[w.h for w in ws])
    rc = L.ns_matmul_prepared(hs, len(ws), mode, C.c_void_p(wsb.data_ptr()), C.c_void_p(out.data_ptr()), ldo, m, None, 0, None,
                              C.c_void_p(ax.data_ptr()) if aux else None, None)
    assert rc == 0, ns.last_error()
    sync()
    return out.cpu().numpy(), (ax.cpu().numpy() if aux else None)


@pytest.mark.parametrize("m", [1, 2, 4])
def test_ring_prepared_image_all_modes(m):
    """plain, QKV concat ([3][m][ldo]) and gate/up + SiLU on the pre-quantised image: every weight row bit for bit; the gate/up
    epilogue is fp32(silu(g) * up) on the same g and up"""
    rng = np.random.default_rng(40 + m)
    k = 4096
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    rq, rk, rv = rand_rows(rng, 256, k), rand_rows(rng, 128, k), rand_rows(rng, 97, k)
    wq, wk, wv = (ns.Weight.from_q8_0_host(r, r.shape[0], k) for r in (rq, rk, rv))
    got, _ = prepared([wq], 0, a, 256)
    assert np.array_equal(bits(got), bits(q8.ring_stated(a, rq)))
    got, _ = prepared([wq, wk, wv], 1, a, 256)
    for i, r in enumerate((rq, rk, rv)):
        assert np.array_equal(bits(got[i * m:(i + 1) * m, :r.shape[0]]), bits(q8.ring_stated(a, r)))
    rg, ru = rand_rows(rng, 200, k), rand_rows(rng, 200, k)
    wg, wu = ns.Weight.from_q8_0_host(rg, 200, k), ns.Weight.from_q8_0_host(ru, 200, k)
    got, aux = prepared([wg, wu], 2, a, 200, aux=True)
    g, up = q8.ring_stated(a, rg), q8.ring_stated(a, ru)
    silu = g / (np.float32(1) + np.exp(-g.astype(np.float64)).astype(np.float32))
    assert np.abs(aux.astype(np.float64) - silu).max() <= 4 * np.spacing(np.abs(silu).astype(np.float32)).max() + 1e-30
    assert np.array_equal(bits(got), bits((aux * up).astype(np.float32)))


@pytest.mark.parametrize("m", [1, 2])
def test_fused_qkv_and_ffn_engine_nodes(m):
    """ns_mul_qkv and ns_ffn_silu at decode rows: each q/k/v row and the down projection of the gate/up product bit for bit"""
    rng = np.random.default_rng(50 + m)
    E, FF = 512, 1024
    a = rng.normal(0, 1, (m, E)).astype(np.float32)
    rq, rk, rv = rand_rows(rng, E, E), rand_rows(rng, 256, E), rand_rows(rng, 256, E)
    wq, wk, wv = (ns.Weight.from_q8_0_host(r, r.shape[0], E) for r in (rq, rk, rv))
    x = dev(a)
    out = torch.full((3, m, E), float("nan"), device="cuda")
    lc = ns.lib().ns_launch_count()
    ns.mul_qkv(wq, wk, wv, x.data_ptr(), E, out.data_ptr(), E, m)
    sync()
    assert ns.lib().ns_launch_count() - lc == 1
    o = out.cpu().numpy()
    for i, r in enumerate((rq, rk, rv)):
        assert np.array_equal(bits(o[i][:, :r.shape[0]]), bits(q8.ring_stated(a, r)))
    r1, r3, r2 = rand_rows(rng, FF, E), rand_rows(rng, FF, E), rand_rows(rng, E, FF)
    w1, w3, w2 = ns.Weight.from_q8_0_host(r1, FF, E), ns.Weight.from_q8_0_host(r3, FF, E), ns.Weight.from_q8_0_host(r2, E, FF)
    tmp = torch.zeros((2, m, FF), device="cuda")
    dst = torch.full((m, E), float("nan"), device="cuda")
    lc = ns.lib().ns_launch_count()
    ns.ffn_silu(w1, w2, w3, x.data_ptr(), E, tmp.data_ptr(), dst.data_ptr(), E, m)
    sync()
    assert ns.lib().ns_launch_count() - lc == 2
    mid = tmp.cpu().numpy()[0]
    assert np.array_equal(bits(dst.cpu().numpy()), bits(q8.ring_stated(mid, r2)))


@pytest.mark.parametrize("m,k", [(1, 4096), (2, 4096), (1, 11008), (2, 352)])
def test_fused_rmsnorm_bitwise(m, k):
    """ns_rmsnorm_mul_mat: oracle.ring_norm_row (224 consumer threads on the two-CTA kernel, 448 on the wide one) + the quantiser
    + the ring's block sums, in one launch"""
    rng = np.random.default_rng(60 + m + k)
    n = 384
    rows = rand_rows(rng, n, k)
    w = ns.Weight.from_q8_0_host(rows, n, k)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    nw = rng.uniform(0.5, 1.5, k).astype(np.float32)
    eps = 1e-5
    hs = (C.c_void_p * 1)(w.h)
    assert ns.lib().ns_rmsnorm_fusable(hs, 1, m) == 1
    x, g = dev(a), dev(nw)
    out = torch.full((m, n), float("nan"), device="cuda")
    lc = ns.lib().ns_launch_count()
    rc = ns.lib().ns_rmsnorm_mul_mat(w.h, C.c_void_p(x.data_ptr()), k, C.c_void_p(g.data_ptr()), C.c_float(eps),
                                     C.c_void_p(out.data_ptr()), n, m, None, None, None)
    assert rc == 0, ns.last_error()
    sync()
    assert ns.lib().ns_launch_count() - lc == 1
    nt = 448 if m == 1 else 224
    xn = np.stack([oracle.ring_norm_row(a[i], nw, eps, nt) for i in range(m)])
    assert np.array_equal(bits(out.cpu().numpy()), bits(q8.ring_stated(xn, rows)))


# ------------------------------------------------------------------------------------------------------------- integer tensor cores
def sample_cols(rng, n, count=160):
    """weight rows to restate: the first and last tile's edges and a random spread"""
    return np.unique(np.concatenate([[0, 1, 127, 128, n - 1], rng.choice(n, min(count, n), replace=False)]))


@pytest.mark.parametrize("m", [3, 8, 13, 32])
@pytest.mark.parametrize("n,k", [(384, 4096), (4096, 11008)])
def test_imma_exact_bitwise_and_random_within_bound(m, n, k):
    """exact construction: the reference dot bit for bit; random data: the split-order restatement (q8.imma_stated) bit for bit
    for the split count the planner chose, and within gamma_n sum |t_b|"""
    rng = np.random.default_rng(m * 7 + k)
    rows, a = exact_case(rng, n, k, m)
    w = ns.Weight.from_q8_0_host(rows, n, k)
    got, launches = run(w, a)
    assert launches == 2                                   # activation image + the integer tensor-core matmul
    assert np.array_equal(bits(got), bits(q8.mul_mat(rows, a)))
    rows = rand_rows(rng, n, k)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    w = ns.Weight.from_q8_0_host(rows, n, k)
    got, launches = run(w, a)
    assert launches == 2
    cols = sample_cols(rng, n)
    assert q8.imma_split_of(got[:, cols], a, rows, cols) is not None
    codes, asc = q8.quantize_act(a)
    wq, wd = q8.split(rows, k)
    tot, mag, nb = oracle.imma_stated(codes, asc, 32, wq.T, wd.T, None, 32)
    assert oracle.imma_bound_ratio(got, tot, mag, nb) <= 1.0


@pytest.mark.parametrize("m", [3, 8, 32])
def test_imma_qkv_and_gate_up(m):
    """QKV concat: every weight's rows bit for bit against the split-order restatement, one split count for the launch; gate/up:
    fp32(silu(g) * up) on the restated g and up (the device expf within 4 ulp); the down projection bit for bit on the product"""
    rng = np.random.default_rng(70 + m)
    E, FF = 1024, 2048
    a = rng.normal(0, 1, (m, E)).astype(np.float32)
    rq, rk, rv = rand_rows(rng, E, E), rand_rows(rng, 256, E), rand_rows(rng, 256, E)
    wq, wk, wv = (ns.Weight.from_q8_0_host(r, r.shape[0], E) for r in (rq, rk, rv))
    x = dev(a)
    out = torch.full((3, m, E), float("nan"), device="cuda")
    lc = ns.lib().ns_launch_count()
    ns.mul_qkv(wq, wk, wv, x.data_ptr(), E, out.data_ptr(), E, m)
    sync()
    assert ns.lib().ns_launch_count() - lc == 2
    o = out.cpu().numpy()
    splits = set()
    for i, r in enumerate((rq, rk, rv)):
        cols = sample_cols(rng, r.shape[0])
        ks = q8.imma_split_of(o[i][:, cols], a, r, cols)
        assert ks is not None, i
        splits.add(ks)
    assert len(splits) == 1, splits
    r1, r3, r2 = rand_rows(rng, FF, E), rand_rows(rng, FF, E), rand_rows(rng, E, FF)
    w1, w3, w2 = ns.Weight.from_q8_0_host(r1, FF, E), ns.Weight.from_q8_0_host(r3, FF, E), ns.Weight.from_q8_0_host(r2, E, FF)
    tmp = torch.zeros((2, m, FF), device="cuda")
    dst = torch.full((m, E), float("nan"), device="cuda")
    lc = ns.lib().ns_launch_count()
    ns.ffn_silu(w1, w2, w3, x.data_ptr(), E, tmp.data_ptr(), dst.data_ptr(), E, m)
    sync()
    assert ns.lib().ns_launch_count() - lc == 4           # two integer tensor-core launches, each with its activation image
    mid = tmp.cpu().numpy()[0]                             # the gate/up product
    cols = sample_cols(rng, FF)
    best = None
    for ks in range(1, 17):
        g, u = q8.imma_stated(a, r1, ks, cols), q8.imma_stated(a, r3, ks, cols)
        want = ((g / (1 + np.exp(-g.astype(np.float64)))) * u).astype(np.float32)
        err = float((np.abs(mid[:, cols] - want) / np.spacing(np.maximum(np.abs(want), np.float32(1e-30)))).max())
        best = err if best is None else min(best, err)
    assert best <= 4, best
    cols = sample_cols(rng, E)
    assert q8.imma_split_of(dst.cpu().numpy()[:, cols], mid, r2, cols) is not None


# ------------------------------------------------------------------------------------------------------------- exact-integer case
def test_exact_case_every_path_equals_the_reference_dot():
    """ring (1, 2 rows), IMMA (8 rows) and the host drop-in, on a problem whose every fp32 sum is exact: each equals
    ne_vec_dot_q8_0_q8_0 (q8.mul_mat; the reference build itself where it is present) bit for bit"""
    rng = np.random.default_rng(80)
    n, k = 256, 4096
    for m in (1, 2, 8):
        rows, a = exact_case(rng, n, k, m)
        want = q8.mul_mat(rows, a)
        if oracle.ref_ggml() is not None:
            aq = oracle.quantize_q8_0(a, "ref", "runtime")
            s = C.c_float()
            for i in range(m):
                for j in range(0, n, 17):
                    oracle.ref_ggml().ref_vec_dot_q8_0_q8_0(C.c_int(k), C.byref(s), rows[j].ctypes.data_as(C.c_void_p),
                                                           aq[i].ctypes.data_as(C.c_void_p))
                    assert bits(np.float32(s.value)) == bits(want[i, j])
        w = ns.Weight.from_q8_0_host(rows, n, k)
        got, launches = run(w, a)
        assert launches == (1 if m <= 2 else 2)
        assert np.array_equal(bits(got), bits(want))
        host = np.zeros((m, n), np.float32)
        assert ns.lib().ns_mul_mat_q8_0_f32_host(rows.ctypes.data_as(C.c_void_p), rows.shape[1], a.ctypes.data_as(C.c_void_p),
                                                 host.ctypes.data_as(C.c_void_p), k, n, m) == 0, ns.last_error()
        assert np.array_equal(bits(host), bits(want))
    ns.lib().ns_host_cache_clear()


# ------------------------------------------------------------------------------------------------------------- wgmma and host drop-in
@pytest.mark.parametrize("m", [33, 64, 200])
def test_wgmma_prompt_within_bf16_bar(m):
    """m > 32 takes the bf16 wgmma GEMM: code exact in bf16, times the bf16-rounded d, fp32 accumulation"""
    rng = np.random.default_rng(90 + m)
    n, k = 512, 4096
    rows = rand_rows(rng, n, k)
    w = ns.Weight.from_q8_0_host(rows, n, k)
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    got, launches = run(w, a)
    assert launches == 2                                   # bf16 activation image + GEMM
    want = q8.mul_mat(rows, a)
    assert np.abs(got - want).max() <= 1e-2 * np.abs(want).max()


def test_host_drop_in_against_the_golden_fixture():
    """ns_mul_mat_q8_0_f32_host on the fixture the reference wrote: within the fp32 summation-order bound gamma_n sum |t_b|"""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ggml_q8_0.npz"))
    wq, a, want = g["wq"], g["a"], g["out"]
    m, k = a.shape
    n = wq.shape[0]
    got = np.zeros((m, n), np.float32)
    assert ns.lib().ns_mul_mat_q8_0_f32_host(wq.ctypes.data_as(C.c_void_p), wq.shape[1], np.ascontiguousarray(a).ctypes.data_as(C.c_void_p),
                                             got.ctypes.data_as(C.c_void_p), k, n, m) == 0, ns.last_error()
    codes, asc = q8.quantize_act(a)
    q, d = q8.split(wq, k)
    _, mag, nb = oracle.imma_stated(codes, asc, 32, q.T, d.T, None, 32)
    nn = nb + 32
    bound = nn * 2.0 ** -24 / (1 - nn * 2.0 ** -24) * mag
    assert (np.abs(got.astype(np.float64) - want) <= 2 * bound + 1e-30).all()
    ns.lib().ns_host_cache_clear()


# ------------------------------------------------------------------------------------------------------------- eval step
def test_toy_engine_eval_generate_against_the_cpu_graph():
    m, _ = q8.toy(seed=5)
    orc, jig, eng = m.graph(), m.graph(jig=True), m.engine()
    running = RunningBar()
    prompt = [1, 200, 31, 7, 99]
    want = orc.eval(prompt, 0)
    tol = running(want, jig.eval(prompt, 0))
    got, nxt = eng.eval(prompt, 0)
    check_logits(got, want, tol)
    t, pos = nxt, len(prompt)
    for _ in range(6):
        want = orc.eval([t], pos)
        tol = running(want, jig.eval([t], pos))
        got, nxt = eng.eval([t], pos)
        check_logits(got, want, tol)
        t, pos = greedy(want), pos + 1
    # generate: picks fed back on the device, against the CPU graph's greedy chain where it is unambiguous
    g2, g2j, eng2 = m.graph(), m.graph(jig=True), m.engine()
    eng2.eval(prompt, 0)
    want0 = g2.eval(prompt, 0)
    g2j.eval(prompt, 0)
    first = greedy(want0)
    picks = eng2.generate(first, len(prompt), 6)
    t, pos = first, len(prompt)
    for p in picks:
        want = g2.eval([t], pos)
        tol = running(want, g2j.eval([t], pos))
        if unambiguous(want, 2 * tol):
            assert p == greedy(want)
        t, pos = int(p), pos + 1
    eng.close()
    eng2.close()


def test_toy_engine_batches_and_eval_all():
    m, _ = q8.toy(seed=6, n_head=4, n_head_kv=2)
    running = RunningBar()
    eng = m.engine(n_seq=4)
    graphs = [(m.graph(), m.graph(jig=True)) for _ in range(4)]
    prompts = [[1, 5, 9], [2, 44, 100, 7, 8], [3], [4, 250, 17, 18, 19, 20, 21, 22, 23]]
    logits, picks = eng.eval_batch([0, 1, 2, 3], prompts, [0, 0, 0, 0])
    for i, p in enumerate(prompts):
        want = graphs[i][0].eval(p, 0)
        tol = running(want, graphs[i][1].eval(p, 0))
        check_logits(logits[i], want, tol)
    toks, past = [int(np.argmax(l)) for l in logits], [len(p) for p in prompts]
    for _ in range(3):
        logits, picks = eng.decode_batch([0, 1, 2, 3], toks, past)
        for i in range(4):
            want = graphs[i][0].eval([toks[i]], past[i])
            tol = running(want, graphs[i][1].eval([toks[i]], past[i]))
            check_logits(logits[i], want, tol)
        toks, past = [int(p) for p in picks], [p + 1 for p in past]
    # eval_all: every row of a fresh prompt against the CPU graph run token by token
    eng2 = m.engine(n_seq=1)
    seg = [1, 17, 300, 5, 123, 77, 9, 40]
    _, am, lg = eng2.eval_all([0], [seg], [0], want_logits=True)
    g, gj = m.graph(), m.graph(jig=True)
    for r, t in enumerate(seg):
        want = g.eval([t], r)
        tol = running(want, gj.eval([t], r))
        check_logits(lg[0][r], want, tol)
        assert am[0][r] == int(np.flatnonzero(lg[0][r] == lg[0][r].max())[0])
    eng.close()
    eng2.close()


def test_decode_launches_equal_a_q4_0_engine():
    """a Q8_0 token launches as many kernels as a Q4_0 token of the same shape (fused QKV, gate/up SiLU, the folded RMSNorms),
    counted with ns_launch_count on passes that launch kernels: an eager one-token step on block 1 of a two-block context, and
    the capturing step on block 0 (one eager pass and the captured one).  A replay of the captured step adds no launch: every
    later token of block 0 is one CUDA graph."""
    mq8, _ = q8.toy(seed=7)
    mq4 = toy(seed=7)
    L = ns.lib()
    counts = {}
    for name, mdl in (("q4_0", mq4), ("q8_0", mq8)):
        eng = mdl.engine(n_seq=2)
        eng.eval_seq(0, [1, 2, 3], 0)
        eng.eval_seq(1, [1, 2, 3], 0)
        lc = L.ns_launch_count()
        eng.eval_seq(1, [4], 3)                            # eager: block 1 never takes the captured graph
        eager = L.ns_launch_count() - lc
        lc = L.ns_launch_count()
        eng.eval([4], 3)                                   # block 0: eager warm-up pass + the captured pass
        capturing = L.ns_launch_count() - lc
        lc = L.ns_launch_count()
        eng.eval([5], 4)                                   # replay
        replay = L.ns_launch_count() - lc
        counts[name] = (eager, capturing, replay)
        eng.close()
    assert counts["q8_0"] == counts["q4_0"], counts
    eager, capturing, replay = counts["q8_0"]
    assert eager > 0 and capturing > 0 and replay == 0, counts


def test_gguf_file_loads_and_matches_the_in_memory_model(tmp_path):
    pytest.importorskip("gguf")
    from neural_speed_b200 import gguf_loader
    m, tok_rows = q8.toy(seed=8, n_head=4, n_head_kv=2)
    path = str(tmp_path / "q8.gguf")
    q8.write_gguf(path, m.hp, tok_rows, m.out_norm, m.out_rows, m.layers)
    eng_file = gguf_loader.load_into_engine(gguf_loader.parse(path))
    eng_mem = m.engine()
    prompt = [1, 9, 250, 33]
    a, na = eng_file.eval(prompt, 0)
    b, nb_ = eng_mem.eval(prompt, 0)
    assert np.array_equal(bits(a), bits(b)) and na == nb_
    ga, gb = eng_file.generate(na, 4, 8), eng_mem.generate(nb_, 4, 8)
    assert np.array_equal(ga, gb)
    eng_file.close()
    eng_mem.close()


def test_llama2_7b_shaped_q8_0_greedy_decode_matches_the_reference_engine():
    """tests/test_gpu_llama.py's 7B-shape check on Q8_0 weights: a 12-token prompt token by token, then 16 greedy steps against
    the reference's own engine (NE_TYPE_Q8_0 tensors; the Q8_0 CPU graph where the reference build is absent).  Ids equal where
    the margin is unambiguous; logits within max(1e-2, 1.5 x floor) <= 2.5e-2 of max|logit|."""
    rng = np.random.default_rng(2026)
    m = q8.llama2_7b_shaped(rng, n_ctx=64)
    m.draw_jig(rng)
    ref, ref_jig = m.reference(), m.reference(jig=True)
    eng = m.engine()
    prompt = [1] + [int(t) for t in rng.integers(3, m.hp["n_vocab"], 11)]
    pos, agree, checked, worst, running = 0, 0, 0, 0.0, RunningBar()
    t = prompt[0]
    for step in range(len(prompt) + 16):
        want = ref.eval([t], pos)
        tol = running(want, ref_jig.eval([t], pos))
        got, nxt = eng.eval([t], pos)
        s, err = scale(want), float(np.abs(got - want).max())
        assert err <= tol * s, (step, err / s, running.floor)
        worst = max(worst, err / s)
        if unambiguous(want, 2 * tol):
            checked += 1
            agree += int(nxt == greedy(want))
        pos += 1
        t = prompt[pos] if pos < len(prompt) else greedy(want)
    print(f"7B-shape Q8_0 decode: worst |dlogit|/max|logit| {worst:.2e}; reference against itself {running.floor:.2e}; "
          f"ids {agree}/{checked}; distance helper {distance(got, want):.2e}")
    assert checked >= 8 and agree == checked, (agree, checked)
    eng.close()
    close(ref, ref_jig)

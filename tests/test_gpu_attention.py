"""Each attention kernel of the eval step on its own (ns_llama_attention) against the CPU attention model (oracle/llama_model.py).

Every case runs RoPE of q and of the new k rows, the fp16 KV append and the causal attention of one layer with seeded inputs
and a fresh workspace, and checks
* the KV cache: V rows bit-identical to the oracle's, K rows within 1 fp16 ulp (CUDA sincosf is not glibc's); for the prompt
  paths also the rotated q left in place, within 2 fp32 ulp of the pair's magnitude;
* the output of the exact-order kernels (generic, rows, split decode over one range) against attention_reference, and of the
  deviating ones (tensor-core prompt kernel, split decode over >= 2 ranges) against attention_stated -- max|d| and mean|d|
  relative to max|V| -- and against attention_reference at the 1e-3 bound of tests/test_attention_numerics_cpu.py;
* poisoned memory: cache rows from position n_past on are NaN before the call (the new rows must overwrite them, later ones
  must never be read), the split partials are NaN, and the output must be finite;
* the per-head tickets read zero after every call.
Errors measured on an H100 80GB HBM3 (400 W power limit) over every case of this file, as max|d| / mean|d| relative to max|V|:
split decode 1.3e-5 / 2.9e-7 (one range: 7.0e-6 / 8.4e-8), rows 1.1e-5 / 1.5e-7, tensor-core prompt 1.5e-4 / 2.4e-7, generic
3.8e-5 / 2.8e-7; new K elements not bit-identical to the oracle's: at most 0.4 %.  Each bar in BARS is about 4x its measurement,
never looser than 5e-4 / 1e-6.  The file takes 50 to 75 s on that GPU."""
import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
from oracle import llama_model as lm

pytestmark = pytest.mark.gpu

SPLIT, ROWS, MMA, GENERIC = ns.ATTN_SPLIT_DECODE, ns.ATTN_ROWS, ns.ATTN_MMA, ns.ATTN_GENERIC
NAME = {SPLIT: "split", ROWS: "rows", MMA: "mma", GENERIC: "generic"}
# two-level bars relative to max|V|: any element, and the mean over the output (measurements in the module docstring)
BARS = {SPLIT: (5e-5, 1e-6), ROWS: (5e-5, 6e-7), MMA: (5e-4, 1e-6), GENERIC: (1.5e-4, 1e-6)}


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


class Case:
    """host inputs of one call: q [m][H][hd], k / v [m][HK][hd] fp32, caches [HK][n_ctx][hd] fp16 (NaN from n_past on)"""

    def __init__(self, n_head, n_head_kv, hd, n_ctx, n_past, m, seed=0, theta=10000.0, scale=1.0, q_std=2.0):
        self.H, self.HK, self.hd, self.n_ctx, self.n_past, self.m, self.theta, self.scale = n_head, n_head_kv, hd, n_ctx, n_past, m, theta, scale
        r = np.random.default_rng(seed)
        self.q = r.normal(0, q_std, (m, n_head, hd)).astype(np.float32)
        self.k = r.normal(0, 1, (m, n_head_kv, hd)).astype(np.float32)
        self.v = r.normal(0, 1, (m, n_head_kv, hd)).astype(np.float32)
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.kc = torch.full((n_head_kv, n_ctx, hd), float("nan"), dtype=torch.float16, device="cuda")
        self.vc = torch.full_like(self.kc, float("nan"))
        if n_past:
            self.kc[:, :n_past] = torch.randn((n_head_kv, n_past, hd), generator=g, device="cuda").half()
            self.vc[:, :n_past] = torch.randn((n_head_kv, n_past, hd), generator=g, device="cuda").half()

    @property
    def pos(self):
        return self.n_past + np.arange(self.m)


def _ws(case):
    nbytes = ns.lib().ns_llama_attention_workspace_bytes(case.H, case.hd, case.n_ctx)
    return torch.zeros(nbytes, dtype=torch.uint8, device="cuda")


def _tickets(case, ws):
    return ws[16:16 + 4 * case.H].view(torch.int32).cpu().numpy()


def _poison_partials(case, ws):
    ws[16 + (4 * case.H + 15) // 16 * 16:] = 0xFF  # every float NaN


def run(kernel, case, ws=None, kc=None, vc=None):
    """one ns_llama_attention call on copies of the case's buffers; returns (out, q after the call, kc, vc, tickets) on the host"""
    ws = _ws(case) if ws is None else ws
    _poison_partials(case, ws)
    q = torch.from_numpy(case.q.reshape(case.m, -1)).cuda()
    k = torch.from_numpy(case.k.reshape(case.m, -1)).cuda()
    v = torch.from_numpy(case.v.reshape(case.m, -1)).cuda()
    kc = case.kc.clone() if kc is None else kc
    vc = case.vc.clone() if vc is None else vc
    out = torch.full((case.m, case.H * case.hd), float("nan"), device="cuda")
    torch.cuda.synchronize()
    rc = ns.lib().ns_llama_attention(kernel, q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), case.H, case.HK,
                                     case.hd, case.n_ctx, case.n_past, case.m, case.theta, case.scale, out.data_ptr(), ws.data_ptr(), None)
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    return (out.cpu().numpy().reshape(case.m, case.H, case.hd), q.cpu().numpy().reshape(case.m, case.H, case.hd), kc, vc,
            _tickets(case, ws))


def check_cache_and_q(case, kernel, q_after, kc, vc):
    """V rows bit-identical, K rows within 1 fp16 ulp, every other cache row untouched, q rotated in place within 2 fp32 ulp
    (rope_kv_kernel) or left as it was (the fused kernels).  Ulps are taken of the rotated pair's magnitude where a rotation
    cancels (a 1-ulp difference of sin or cos there moves the result by an ulp of the inputs, not of the result).  Returns the
    fraction of new K elements that are not bit-identical and the oracle's rotated q."""
    pos = case.pos
    q_rot = lm.rope_mode0_rows(case.q, pos, case.hd, case.theta, case.scale)
    k_rot = lm.rope_mode0_rows(case.k, pos, case.hd, case.theta, case.scale)
    want_k, want_v = case.kc.cpu().numpy(), case.vc.cpu().numpy()
    want_k[:, pos] = k_rot.astype(np.float16).transpose(1, 0, 2)
    want_v[:, pos] = case.v.astype(np.float16).transpose(1, 0, 2)
    got_k, got_v = kc.cpu().numpy(), vc.cpu().numpy()
    assert np.array_equal(got_v.view(np.uint16), want_v.view(np.uint16)), "V cache"
    old = np.ones(case.n_ctx, bool)
    old[pos] = False
    assert np.array_equal(got_k[:, old].view(np.uint16), want_k[:, old].view(np.uint16)), "K cache rows other than the new ones"
    g, w = got_k[:, pos].astype(np.float32), want_k[:, pos].astype(np.float32)
    pair = np.sqrt(case.k[..., 0::2] ** 2 + case.k[..., 1::2] ** 2).repeat(2, axis=-1).transpose(1, 0, 2)
    tol = np.maximum(np.spacing(np.abs(w).astype(np.float16)).astype(np.float32), 4 * 2.0 ** -24 * pair)
    assert (np.abs(g - w) <= tol).all(), ("K rows beyond 1 fp16 ulp", float(np.abs(g - w).max()))
    if kernel in (MMA, GENERIC) or (kernel == ROWS and case.m > 1):  # rope_kv_kernel rotates q in place
        qpair = np.sqrt(case.q[..., 0::2] ** 2 + case.q[..., 1::2] ** 2).repeat(2, axis=-1)
        assert (np.abs(q_after - q_rot) <= 2 * np.spacing(qpair)).all(), "rotated q beyond 2 fp32 ulp"
    else:
        assert np.array_equal(q_after, case.q), "the fused kernels rotate q in registers only"
    return float((g != w).mean()), q_rot


def errors(got, want, vmax):
    d = np.abs(got.astype(np.float64) - want)
    return float(d.max()) / vmax, float(d.mean()) / vmax


def check_output(case, kernel, out, kc, vc, q_rot):
    """out against the model the kernel states, computed from the cache the kernel left (K within 1 ulp of the oracle's)"""
    assert np.isfinite(out).all(), "non-finite output"
    L = case.n_past + case.m
    kch, vch = kc[:, :L].cpu().numpy(), vc[:, :L].cpu().numpy()
    vmax = float(np.abs(vch.astype(np.float32)).max())
    ref = lm.attention_reference(q_rot, kch, vch, case.n_past)
    nact = (L + lm.SPLIT_KEYS - 1) // lm.SPLIT_KEYS
    if kernel == MMA or (kernel == SPLIT and nact > 1):
        stated = lm.attention_stated(q_rot, kch, vch, case.n_past, "mma" if kernel == MMA else "split")
        emax, emean = errors(out, stated, vmax)
        rel_ref = float(np.abs(out - ref).max()) / float(np.abs(ref).max())
        assert rel_ref <= 1e-3, (NAME[kernel], "vs reference order", rel_ref)
    else:
        emax, emean = errors(out, ref, vmax)
    bar_max, bar_mean = BARS[kernel]
    assert emax <= bar_max and emean <= bar_mean, (NAME[kernel], emax, emean)
    return emax, emean


def run_and_check(kernel, case):
    out, q_after, kc, vc, tickets = run(kernel, case)
    assert (tickets == 0).all(), tickets
    kfrac, q_rot = check_cache_and_q(case, kernel, q_after, kc, vc)
    if kernel == SPLIT or (kernel == ROWS and case.m == 1):
        # the fused kernels rotate q with the same sincosf arithmetic as rope_kv_kernel, but keep it in registers: take the q the
        # latter leaves (checked against the oracle above) so that the comparison measures the attention, not sincosf vs libm
        q_rot = run(GENERIC, case)[1]
    emax, emean = check_output(case, kernel, out, kc, vc, q_rot)
    print(f"{NAME[kernel]} H{case.H}/{case.HK} hd{case.hd} ctx{case.n_ctx} past{case.n_past} m{case.m}: max {emax:.2e} "
          f"mean {emean:.2e} (x max|V|), K rows not bit-identical {kfrac:.3%}")
    return out


# ------------------------------------------------------------------------------------------------------------- decode
DECODE_PAST = (0, 1, 255, 256, 257, 511, 1023, 2047, 4095, 8191)
DECODE_CASES = ([(128, h, hk, 8192, p) for h, hk in ((8, 1), (4, 2)) for p in DECODE_PAST] +
                [(64, h, hk, 8192, p) for h, hk in ((8, 1), (4, 2)) for p in DECODE_PAST] +
                [(hd, h, hk, 8192, p) for hd in (64, 128) for h, hk in ((32, 32), (32, 8)) for p in (0, 257, 2047, 8191)] +
                [(hd, 32, 8, n_ctx, p) for hd in (64, 128) for n_ctx in (300, 1000) for p in (0, 255, 256, n_ctx - 1)])


@pytest.mark.parametrize("hd,n_head,n_head_kv,n_ctx,n_past", DECODE_CASES)
def test_decode_kernels_against_the_reference(hd, n_head, n_head_kv, n_ctx, n_past):
    """split decode (1 .. 32 ranges) and the fused rows kernel, one new token."""
    case = Case(n_head, n_head_kv, hd, n_ctx, n_past, 1, seed=n_past + hd + n_head_kv)
    for kernel in (SPLIT, ROWS):
        run_and_check(kernel, case)


# ------------------------------------------------------------------------------------------------------------- prompts
MMA_CASES = [(hd, m, p) for hd in (64, 128) for m in (8, 9, 63, 64, 65, 127, 200) for p in (0, 1, 37, 64, 1000)] + \
            [(hd, 2048, p) for hd in (64, 128) for p in (0, 1000)]


@pytest.mark.parametrize("hd,m,n_past", MMA_CASES)
def test_tensor_core_prompt_kernel_against_its_stated_arithmetic(hd, m, n_past):
    """GQA 4:1; n_past + m == n_ctx whenever n_past is even (the prompt fills the context)."""
    n_ctx = n_past + m + (0 if n_past % 2 == 0 else 7)
    run_and_check(MMA, Case(8, 2, hd, n_ctx, n_past, m, seed=m + n_past))


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("m", [2, 3, 7])
@pytest.mark.parametrize("n_past", [0, 300])
def test_rows_kernel_for_short_prompts(hd, m, n_past):
    run_and_check(ROWS, Case(8, 2, hd, n_past + m + 1, n_past, m, seed=hd + m))


@pytest.mark.parametrize("hd", [32, 80, 96])
@pytest.mark.parametrize("m,n_past", [(1, 0), (1, 700), (5, 0), (40, 300)])
def test_generic_kernel_for_other_head_sizes(hd, m, n_past):
    run_and_check(GENERIC, Case(6, 3, hd, n_past + m, n_past, m, seed=hd + n_past))


# ------------------------------------------------------------------------------------------------------------- RoPE
@pytest.mark.parametrize("theta", [10000.0, 500000.0])
@pytest.mark.parametrize("scale", [1.0, 0.25, 4.0])
def test_rope_settings_out_to_position_8191(theta, scale):
    """every RoPE implementation (rope_kv_kernel, and the fused ones in attn_fast_kernel / attn_decode_kernel) at Llama-3's base
    and both directions of the scale: K rows within 1 fp16 ulp, q within 2 fp32 ulp, outputs within the bars"""
    for kernel, m, n_past in ((MMA, 64, 8128), (GENERIC, 3, 8189), (ROWS, 1, 8191), (SPLIT, 1, 8191), (SPLIT, 1, 4000)):
        run_and_check(kernel, Case(4, 2, 128, 8192, n_past, m, seed=m, theta=theta, scale=scale))


# ------------------------------------------------------------------------------------------------------------- edges
def _positions_case(hd, n_ctx, n_past, m):
    """K = 0 (every score exactly 0) and V encoding the position: channel d is 1 before (even d) or from (odd d) position
    c_d = d * n_ctx / hd and 0 elsewhere, so the output is the fraction of the attended window on that side of c_d.  Every sum
    of these values is exact in fp32, and one key too many or too few moves some channel by at least 1 / n_ctx."""
    case = Case(4, 2, hd, n_ctx, n_past, m)
    case.k[:] = 0
    pos = np.arange(n_ctx)[:, None]
    c = np.arange(hd)[None, :] * n_ctx // hd
    enc = np.where(np.arange(hd)[None, :] % 2 == 0, pos < c, pos >= c).astype(np.float32)  # [n_ctx][hd]
    enc16 = torch.from_numpy(enc.astype(np.float16)).cuda()
    case.kc[:, :n_past] = 0
    case.vc[:, :n_past] = enc16[:n_past]
    case.v[:] = enc[n_past:n_past + m][:, None, :]
    return case


@pytest.mark.parametrize("kernel,hd,n_ctx,n_past,m", [(SPLIT, 128, 8192, 8191, 1), (SPLIT, 64, 8192, 4096, 1), (SPLIT, 128, 1000, 255, 1),
                                                      (ROWS, 128, 8192, 8191, 1), (ROWS, 64, 8192, 8185, 7),
                                                      (MMA, 128, 8192, 6144, 2048), (MMA, 64, 4200, 4000, 200),
                                                      (GENERIC, 96, 8192, 8000, 192), (GENERIC, 80, 2048, 2047, 1)])
def test_equal_scores_give_the_mean_over_exactly_the_attended_window(kernel, hd, n_ctx, n_past, m):
    """one key too many or too few moves some channel by >= 1 / n_ctx (1.2e-4 at 8192 positions); measured at most 6.8e-8 (the
    sums are exact, only the final division or p = fp16(1 / L) rounds), bar 3e-7"""
    case = _positions_case(hd, n_ctx, n_past, m)
    out, _, kc, vc, tickets = run(kernel, case)
    assert np.isfinite(out).all() and (tickets == 0).all()
    v = vc.cpu().numpy().astype(np.float64)
    for t in (0, m // 2, m - 1):
        L = n_past + t + 1
        want = np.repeat(v[:, :L].mean(axis=1), case.H // case.HK, axis=0)  # [H][hd]: heads share their kv head's window
        if kernel in (ROWS, GENERIC) or (kernel == SPLIT and L <= lm.SPLIT_KEYS):
            want = want * (float(np.float16(np.float32(1.0 / L))) * L)  # the reference order: every p = fp16(1 / L)
        rel = float(np.abs(out[t] - want).max())  # max|V| = 1
        print(f"{NAME[kernel]} hd{hd} window {L}: {rel:.2e}")
        assert rel <= 3e-7, (NAME[kernel], t, rel)


@pytest.mark.parametrize("hd,n_head,n_head_kv,n_past", [(128, 8, 2, 8191), (64, 4, 4, 1000), (128, 32, 8, 300)])
def test_decode_needles(hd, n_head, n_head_kv, n_past):
    """one cached key of each kv head set to 4 rope(q) of the group's first head at positions 0, 63, 64, 255, 256, 257, pos - 1:
    that key takes all the weight (the others' e underflow to 0), so the head's output is that position's V row"""
    base = Case(n_head, n_head_kv, hd, n_past + 1, n_past, 1, seed=hd + n_past, q_std=1.0)
    q_rot = lm.rope_mode0_rows(base.q, base.pos, hd)[0]
    group = n_head // n_head_kv
    for j in (0, 63, 64, 255, 256, 257, n_past - 1):
        case = Case(n_head, n_head_kv, hd, n_past + 1, n_past, 1, seed=hd + n_past, q_std=1.0)
        case.kc[:, j] = torch.from_numpy((4 * q_rot[::group]).astype(np.float16)).cuda()
        for kernel in (SPLIT, ROWS):
            out = run_and_check(kernel, case)
            want = case.vc[:, j].cpu().numpy().astype(np.float32)
            # exactly V[j] in the reference order; the split merge adds the other ranges at weight exp(-28) or less
            assert np.abs(out[0, ::group] - want).max() <= 1e-6 * np.abs(want).max(), (NAME[kernel], j)


@pytest.mark.parametrize("kernel,hd,m,n_past", [(MMA, 128, 200, 37), (MMA, 64, 65, 0), (ROWS, 128, 7, 100), (GENERIC, 96, 33, 10)])
def test_prompt_diagonal_needle(kernel, hd, m, n_past):
    """k_new = 4 q: at its own position RoPE preserves the dot product, so each row's own key dominates and its output is its
    own V row -- a row that misses its diagonal key (a strict causal mask) gives something else entirely"""
    case = Case(8, 2, hd, n_past + m, n_past, m, seed=m, q_std=1.0)
    case.k[:] = 4 * case.q[:, ::4]
    out = run_and_check(kernel, case)
    want = case.v.astype(np.float16).astype(np.float32)
    assert np.abs(out[:, ::4] - want).max() <= 1e-3 * np.abs(want).max(), NAME[kernel]


# ------------------------------------------------------------------------------------------------------------- reuse
def test_workspace_reuse_and_determinism():
    """identical calls give identical bits; a 32-range call then a 1-range call at another position on the same workspace are
    both right (the tickets were reset); the tickets read zero after every call"""
    a = Case(32, 8, 128, 8192, 8191, 1, seed=3)
    b = Case(32, 8, 128, 8192, 100, 1, seed=4)
    ws = _ws(a)
    for kernel in (SPLIT, ROWS, GENERIC):
        o1 = run(kernel, a, ws=ws)
        o2 = run(kernel, a, ws=ws)
        assert o1[0].tobytes() == o2[0].tobytes(), NAME[kernel]
        assert (o1[4] == 0).all() and (o2[4] == 0).all()
    for c in (a, b, a, b):
        out, q_after, kc, vc, tickets = run(SPLIT, c, ws=ws)
        assert (tickets == 0).all()
        _, q_rot = check_cache_and_q(c, SPLIT, q_after, kc, vc)
        check_output(c, SPLIT, out, kc, vc, q_rot)
    p = Case(8, 2, 64, 300, 37, 200, seed=5)
    o1, o2 = run(MMA, p, ws=_ws(p)), run(MMA, p, ws=_ws(p))
    assert o1[0].tobytes() == o2[0].tobytes()


def test_unsupported_shapes_launch_nothing():
    """a forced kernel that cannot take the shape, or arguments ns_llama_eval would refuse: an error code and no launch"""
    L = ns.lib()
    before = L.ns_launch_count()
    for kernel, hd, m in ((MMA, 80, 9), (ROWS, 96, 3), (SPLIT, 80, 1), (SPLIT, 128, 2)):
        rc = L.ns_llama_attention(kernel, 1, 1, 1, 1, 1, 4, 2, hd, 64, 10, m, 10000.0, 1.0, 1, 1, None)
        assert rc == -4, (kernel, hd, m, rc)  # NS_E_UNSUPPORTED
    for args in ((4, 3, 64, 64, 10, 1), (4, 2, 63, 64, 10, 1), (4, 2, 64, 64, 60, 5)):  # n_head % n_head_kv, odd hd, n_past + m > n_ctx
        rc = L.ns_llama_attention(ns.ATTN_AUTO, 1, 1, 1, 1, 1, *args, 10000.0, 1.0, 1, 1, None)
        assert rc == -1, (args, rc)  # NS_E_INVALID
    assert L.ns_launch_count() == before

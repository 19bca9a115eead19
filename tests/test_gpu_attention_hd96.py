"""The split decode and tensor-core prompt attention at head size 96 (Phi-3-mini), each on its own through ns_llama_attention, against
the CPU attention model under the bars tests/test_gpu_attention.py applies at 64 / 128 (its BARS, checks and inputs): K / V rows,
q left in place or rotated, outputs against attention_reference or attention_stated, poisoned cache rows and partials, the
tickets.  Also: NS_ATTN_AUTO takes these two kernels at 96, and the batched decode and ragged prompt entries give each row and
segment the bits of its single-sequence call."""
import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
import test_gpu_attention as ga
from oracle import llama_model as lm

pytestmark = pytest.mark.gpu

SPLIT, MMA, AUTO = ns.ATTN_SPLIT_DECODE, ns.ATTN_MMA, ns.ATTN_AUTO
HD = 96


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


# ------------------------------------------------------------------------------------------------------------- decode
DECODE_CASES = ([(h, hk, 8192, p) for h, hk in ((8, 1), (4, 2)) for p in ga.DECODE_PAST] +
                [(32, hk, 8192, p) for hk in (32, 8) for p in (0, 257, 2047, 8191)] +
                [(32, 8, n_ctx, p) for n_ctx in (300, 1000) for p in (0, 255, 256, n_ctx - 1)])


@pytest.mark.parametrize("n_head,n_head_kv,n_ctx,n_past", DECODE_CASES)
def test_split_decode_against_the_reference(n_head, n_head_kv, n_ctx, n_past):
    """one new token over 1 .. 32 ranges; NS_ATTN_AUTO runs the same kernel (same bits)"""
    case = ga.Case(n_head, n_head_kv, HD, n_ctx, n_past, 1, seed=n_past + HD + n_head_kv)
    out = ga.run_and_check(SPLIT, case)
    assert ga.run(AUTO, case)[0].tobytes() == out.tobytes()


# ------------------------------------------------------------------------------------------------------------- prompts
MMA_CASES = [(m, p) for m in (2, 3, 7, 8, 9, 63, 64, 65, 127, 200) for p in (0, 1, 37, 64, 1000)] + [(2048, 0), (2048, 1000)]


@pytest.mark.parametrize("m,n_past", MMA_CASES)
def test_tensor_core_prompt_kernel_against_its_stated_arithmetic(m, n_past):
    """GQA 4:1; n_past + m == n_ctx whenever n_past is even (the prompt fills the context); 2 .. 7 rows too, which NS_ATTN_AUTO
    gives this kernel at head size 96 (same bits)"""
    n_ctx = n_past + m + (0 if n_past % 2 == 0 else 7)
    case = ga.Case(8, 2, HD, n_ctx, n_past, m, seed=m + n_past)
    out = ga.run_and_check(MMA, case)
    if m < 8 or m == 2048:
        assert ga.run(AUTO, case)[0].tobytes() == out.tobytes()


@pytest.mark.parametrize("n_head,n_head_kv", [(4, 4), (8, 1), (32, 32)])
def test_tensor_core_prompt_kernel_mha_and_gqa(n_head, n_head_kv):
    ga.run_and_check(MMA, ga.Case(n_head, n_head_kv, HD, 300, 100, 129, seed=n_head + n_head_kv))


# ------------------------------------------------------------------------------------------------------------- RoPE
@pytest.mark.parametrize("theta", [10000.0, 500000.0])
@pytest.mark.parametrize("scale", [1.0, 0.25, 4.0])
def test_rope_settings_out_to_position_8191(theta, scale):
    """the fused RoPE of attn_decode_kernel and rope_kv_kernel's at head size 96: K rows within 1 fp16 ulp, q within 2 fp32 ulp,
    outputs within the bars"""
    for kernel, m, n_past in ((MMA, 64, 8128), (SPLIT, 1, 8191), (SPLIT, 1, 4000)):
        ga.run_and_check(kernel, ga.Case(4, 2, HD, 8192, n_past, m, seed=m, theta=theta, scale=scale))


# ------------------------------------------------------------------------------------------------------------- edges
@pytest.mark.parametrize("kernel,n_ctx,n_past,m", [(SPLIT, 8192, 8191, 1), (SPLIT, 8192, 4096, 1), (SPLIT, 1000, 255, 1),
                                                   (MMA, 8192, 6144, 2048), (MMA, 4200, 4000, 200)])
def test_equal_scores_give_the_mean_over_exactly_the_attended_window(kernel, n_ctx, n_past, m):
    """test_gpu_attention.py's window test at head size 96: one key too many or too few moves some channel by >= 1 / n_ctx"""
    case = ga._positions_case(HD, n_ctx, n_past, m)
    out, _, kc, vc, tickets = ga.run(kernel, case)
    assert np.isfinite(out).all() and (tickets == 0).all()
    v = vc.cpu().numpy().astype(np.float64)
    for t in (0, m // 2, m - 1):
        L = n_past + t + 1
        want = np.repeat(v[:, :L].mean(axis=1), case.H // case.HK, axis=0)
        if kernel == SPLIT and L <= lm.SPLIT_KEYS:
            want = want * (float(np.float16(np.float32(1.0 / L))) * L)  # the reference order: every p = fp16(1 / L)
        rel = float(np.abs(out[t] - want).max())
        print(f"{ga.NAME[kernel]} hd{HD} window {L}: {rel:.2e}")
        assert rel <= 3e-7, (ga.NAME[kernel], t, rel)


@pytest.mark.parametrize("n_head,n_head_kv,n_past", [(8, 2, 8191), (4, 4, 1000), (32, 8, 300)])
def test_decode_needles(n_head, n_head_kv, n_past):
    """one cached key per kv head set to 4 rope(q) of the group's first head: that key takes all the weight"""
    base = ga.Case(n_head, n_head_kv, HD, n_past + 1, n_past, 1, seed=HD + n_past, q_std=1.0)
    q_rot = lm.rope_mode0_rows(base.q, base.pos, HD)[0]
    group = n_head // n_head_kv
    for j in (0, 63, 64, 255, 256, 257, n_past - 1):
        case = ga.Case(n_head, n_head_kv, HD, n_past + 1, n_past, 1, seed=HD + n_past, q_std=1.0)
        case.kc[:, j] = torch.from_numpy((4 * q_rot[::group]).astype(np.float16)).cuda()
        out = ga.run_and_check(SPLIT, case)
        want = case.vc[:, j].cpu().numpy().astype(np.float32)
        assert np.abs(out[0, ::group] - want).max() <= 1e-6 * np.abs(want).max(), j


@pytest.mark.parametrize("m,n_past", [(200, 37), (65, 0), (5, 10)])
def test_prompt_diagonal_needle(m, n_past):
    """k_new = 4 q: each row's own key dominates, so its output is its own V row"""
    case = ga.Case(8, 2, HD, n_past + m, n_past, m, seed=m, q_std=1.0)
    case.k[:] = 4 * case.q[:, ::4]
    out = ga.run_and_check(MMA, case)
    want = case.v.astype(np.float16).astype(np.float32)
    assert np.abs(out[:, ::4] - want).max() <= 1e-3 * np.abs(want).max()


def test_workspace_reuse_and_determinism():
    """identical calls give identical bits; a 32-range call then a 1-range call on the same workspace are both right (the tickets
    were reset and read zero after every call)"""
    a = ga.Case(32, 8, HD, 8192, 8191, 1, seed=3)
    b = ga.Case(32, 8, HD, 8192, 100, 1, seed=4)
    ws = ga._ws(a)
    o1, o2 = ga.run(SPLIT, a, ws=ws), ga.run(SPLIT, a, ws=ws)
    assert o1[0].tobytes() == o2[0].tobytes() and (o1[4] == 0).all() and (o2[4] == 0).all()
    for c in (a, b, a, b):
        out, q_after, kc, vc, tickets = ga.run(SPLIT, c, ws=ws)
        assert (tickets == 0).all()
        _, q_rot = ga.check_cache_and_q(c, SPLIT, q_after, kc, vc)
        ga.check_output(c, SPLIT, out, kc, vc, ga.run(ns.ATTN_GENERIC, c)[1])
    p = ga.Case(8, 2, HD, 300, 37, 200, seed=5)
    assert ga.run(MMA, p)[0].tobytes() == ga.run(MMA, p)[0].tobytes()


# ------------------------------------------------------------------------------------------------------------- batched
def _rows(r, n, H, HK):
    return (torch.from_numpy(r.normal(0, 2, (n, H * HD)).astype(np.float32)).cuda(),
            torch.from_numpy(r.normal(0, 1, (n, HK * HD)).astype(np.float32)).cuda(),
            torch.from_numpy(r.normal(0, 1, (n, HK * HD)).astype(np.float32)).cuda())


def _caches(n_seq, HK, n_ctx, fill, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    kc = torch.randn((n_seq, HK, n_ctx, HD), generator=g, device="cuda").half()
    vc = torch.randn((n_seq, HK, n_ctx, HD), generator=g, device="cuda").half()
    for s, p in fill.items():  # NaN from each sequence's n_past on: never read before written
        kc[s, :, p:] = float("nan")
        vc[s, :, p:] = float("nan")
    return kc, vc


def _single(kernel, q, k, v, kc, vc, H, HK, n_ctx, n_past, m):
    """one ns_llama_attention call on block views; returns out"""
    case_ws = torch.zeros(ns.lib().ns_llama_attention_workspace_bytes(H, HD, n_ctx), dtype=torch.uint8, device="cuda")
    out = torch.full((m, H * HD), float("nan"), device="cuda")
    q = q.clone()
    torch.cuda.synchronize()
    rc = ns.lib().ns_llama_attention(kernel, q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), H, HK, HD, n_ctx,
                                     n_past, m, 10000.0, 1.0, out.data_ptr(), case_ws.data_ptr(), None)
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("H,HK", [(8, 2), (32, 32)])
def test_batched_rows_are_their_single_sequence_calls(H, HK):
    """ns_llama_attention_batch: each row (1 .. 32 ranges) bit-identical to ns_llama_attention(NS_ATTN_SPLIT_DECODE) on its block,
    and each block's cache too"""
    n_seq, n_ctx = 5, 8192
    seqs, past = [3, 0, 4, 1], [8191, 0, 300, 2047]
    r = np.random.default_rng(H + HK)
    q, k, v = _rows(r, 4, H, HK)
    kc, vc = _caches(n_seq, HK, n_ctx, dict(zip(seqs, past)), seed=H)
    kc1, vc1 = kc.clone(), vc.clone()
    out = torch.full((4, H * HD), float("nan"), device="cuda")
    ws = torch.zeros(ns.lib().ns_llama_attention_batch_workspace_bytes(4, H, HD, n_ctx), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert ns.attention_batch(q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), n_seq, seqs, past, H, HK, HD,
                              n_ctx, out.data_ptr(), ws.data_ptr()) == 0, ns.last_error()
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for i, (s, p) in enumerate(zip(seqs, past)):
        want = _single(SPLIT, q[i:i + 1], k[i:i + 1], v[i:i + 1], kc1[s], vc1[s], H, HK, n_ctx, p, 1)
        assert got[i].tobytes() == want[0].tobytes(), (i, s, p)
    assert torch.equal(kc.view(torch.int16), kc1.view(torch.int16)) and torch.equal(vc.view(torch.int16), vc1.view(torch.int16))


def test_ragged_segments_are_their_single_sequence_calls():
    """ns_llama_attention_ragged: each segment (1, 2 .. 7, 64 and 130 rows) bit-identical to ns_llama_attention(NS_ATTN_MMA) on its
    block, and each block's cache too"""
    H, HK, n_seq, n_ctx = 8, 2, 6, 1200
    seqs, toks, past = [2, 0, 5, 1, 3, 4], [1, 2, 7, 64, 130, 5], [10, 0, 1000, 37, 64, 1]
    r = np.random.default_rng(9)
    T = sum(toks)
    q, k, v = _rows(r, T, H, HK)
    kc, vc = _caches(n_seq, HK, n_ctx, dict(zip(seqs, past)), seed=9)
    kc1, vc1 = kc.clone(), vc.clone()
    q0 = q.clone()
    out = torch.full((T, H * HD), float("nan"), device="cuda")
    ws = torch.zeros(ns.lib().ns_llama_attention_ragged_workspace_bytes(len(seqs), T), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert ns.attention_ragged(q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), n_seq, seqs, toks, past, H, HK,
                               HD, n_ctx, out.data_ptr(), ws.data_ptr()) == 0, ns.last_error()
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    r0 = 0
    for s, n, p in zip(seqs, toks, past):
        want = _single(MMA, q0[r0:r0 + n], k[r0:r0 + n], v[r0:r0 + n], kc1[s], vc1[s], H, HK, n_ctx, p, n)
        assert got[r0:r0 + n].tobytes() == want.tobytes(), (s, n, p)
        r0 += n
    assert torch.equal(kc.view(torch.int16), kc1.view(torch.int16)) and torch.equal(vc.view(torch.int16), vc1.view(torch.int16))


def test_what_head_size_96_still_refuses():
    """NS_ATTN_ROWS, a Q8_0 cache and the streaming ring stay at 64 / 128: an error code and no launch"""
    L = ns.lib()
    before = L.ns_launch_count()
    for kernel, m in ((ns.ATTN_ROWS, 1), (ns.ATTN_ROWS, 3), (SPLIT, 2)):
        assert L.ns_llama_attention(kernel, 1, 1, 1, 1, 1, 4, 2, HD, 64, 10, m, 10000.0, 1.0, 1, 1, None) == -4, (kernel, m)
    ws = torch.zeros(ns.lib().ns_llama_attention_workspace_bytes(4, HD, 64), dtype=torch.uint8, device="cuda")
    t = torch.zeros(4 * HD * 4, device="cuda")
    kc = torch.zeros((2, 64, HD), dtype=torch.float16, device="cuda")
    rc = L.ns_llama_attention_ring(t.data_ptr(), t.data_ptr(), t.data_ptr(), kc.data_ptr(), kc.data_ptr(), 4, 2, HD, 64, 4, 70, 10000.0,
                                   t.data_ptr(), ws.data_ptr(), None)
    assert rc == -4 and "64 or 128" in ns.last_error()
    assert L.ns_launch_count() == before

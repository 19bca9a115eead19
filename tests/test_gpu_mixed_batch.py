"""Mixed prompt and decode batches in the eval step (ns_llama_eval_batch, include/ns_b200.h): one forward pass over token segments
of many sequences -- decode tokens, new prompts and prompt chunks at n_past > 0 together.

* the ragged prompt attention on its own against one NS_ATTN_MMA call per segment, bit for bit;
* mixed calls against the CPU restatement of the reference graph (oracle/llama_model.py), each sequence against itself alone;
* identities: all-one-token calls are decode_batch, one segment is eval_seq, segment order and block placement change nothing;
* a serving loop that admits requests into the running pass and prefills a long prompt in chunks next to the decodes;
* the launch structure, Llama-2-7B shapes against the reference engine, and the argument checks."""
import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
from llama_models import RunningBar, SeqOracle, bits, check_logits, close, llama2_7b_shaped, scale, toy, unambiguous
from oracle.llama_model import greedy

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4
WGMMA_BAR = 4e-2  # passes of more than 32 rows take the bf16 wgmma GEMM: tests/test_gpu_llama.py's bar for that path


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def _h(t):
    return t.view(torch.int16)


# ------------------------------------------------------------------------------------------------------------- 1. kernel
N_CTX_K = 512
LENS = (1, 2, 7, 63, 64, 65, 200)


def _segments(case, rng):
    """case 0: every length once at n_past 0 / 37 / n_ctx - len in turn (7 segments); case 1: 8 segments drawn from the lengths"""
    lens = list(LENS) if case == 0 else [int(x) for x in rng.choice(LENS, 8)]
    past = []
    for i, ln in enumerate(lens):
        p = (0, 37, N_CTX_K - ln)[(i + case) % 3]
        past.append(min(p, N_CTX_K - ln))
    return np.array(lens, np.int32), np.array(past, np.int32)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("n_head,n_head_kv", [(8, 8), (8, 2)])
@pytest.mark.parametrize("case", [0, 1])
def test_ragged_attention_is_the_mma_kernel_segment_by_segment(case, n_head, n_head_kv, hd):
    """segments of 1 .. 200 rows on shuffled blocks of a 10-block cache; every cache row from a segment's n_past on, and every
    row of an unused block, is NaN.  Against one ns_llama_attention(NS_ATTN_MMA) call per segment on a copy of its block: out,
    the rotated q and the whole block bit-identical; rows past each segment and the unused blocks unchanged."""
    H, HK = n_head, n_head_kv
    n_seq = 10
    rng = np.random.default_rng(100 * case + hd + HK)
    lens, past = _segments(case, rng)
    n = len(lens)
    seqs = rng.permutation(n_seq)[:n].astype(np.int32)
    T = int(lens.sum())
    g = torch.Generator(device="cuda").manual_seed(int(case * 7 + hd + HK))
    kc = torch.full((n_seq, HK, N_CTX_K, hd), float("nan"), dtype=torch.float16, device="cuda")
    vc = torch.full_like(kc, float("nan"))
    for s, p in zip(seqs.tolist(), past.tolist()):
        if p:
            kc[s, :, :p] = torch.randn((HK, p, hd), generator=g, device="cuda").half()
            vc[s, :, :p] = torch.randn((HK, p, hd), generator=g, device="cuda").half()
    q = torch.from_numpy(rng.normal(0, 2.0, (T, H * hd)).astype(np.float32)).cuda()
    k = torch.from_numpy(rng.normal(0, 1.0, (T, HK * hd)).astype(np.float32)).cuda()
    v = torch.from_numpy(rng.normal(0, 1.0, (T, HK * hd)).astype(np.float32)).cuda()
    q0, kc0, vc0 = q.clone(), kc.clone(), vc.clone()
    ws = torch.full((ns.lib().ns_llama_attention_ragged_workspace_bytes(n, T),), 0xFF, dtype=torch.uint8, device="cuda")
    out = torch.full((T, H * hd), float("nan"), device="cuda")
    torch.cuda.synchronize()
    rc = ns.attention_ragged(q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), n_seq, seqs, lens, past, H, HK, hd,
                             N_CTX_K, out.data_ptr(), ws.data_ptr())
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    assert torch.isfinite(out).all()
    used = set(seqs.tolist())
    for s in range(n_seq):
        if s not in used:
            assert torch.equal(_h(kc[s]), _h(kc0[s])) and torch.equal(_h(vc[s]), _h(vc0[s])), s
    wsb = ns.lib().ns_llama_attention_workspace_bytes(H, hd, N_CTX_K)
    r0 = 0
    for i, (s, ln, p) in enumerate(zip(seqs.tolist(), lens.tolist(), past.tolist())):
        rows = slice(r0, r0 + ln)
        kci, vci, qi = kc0[s].clone(), vc0[s].clone(), q0[rows].clone()
        one = torch.full((ln, H * hd), float("nan"), device="cuda")
        w1 = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()
        rc = ns.lib().ns_llama_attention(ns.ATTN_MMA, qi.data_ptr(), k[rows].data_ptr(), v[rows].data_ptr(),  # row slices: contiguous
                                         kci.data_ptr(), vci.data_ptr(), H, HK, hd, N_CTX_K, p, ln, 10000.0, 1.0, one.data_ptr(),
                                         w1.data_ptr(), None)
        assert rc == 0, ns.last_error()
        torch.cuda.synchronize()
        where = (i, s, ln, p)
        assert np.array_equal(bits(out[rows].cpu().numpy()), bits(one.cpu().numpy())), ("out",) + where
        assert np.array_equal(bits(q[rows].cpu().numpy()), bits(qi.cpu().numpy())), ("rotated q",) + where
        assert torch.equal(_h(kc[s]), _h(kci)) and torch.equal(_h(vc[s]), _h(vci)), ("block",) + where
        assert torch.equal(_h(kc[s, :, p + ln:]), _h(kc0[s, :, p + ln:])) and torch.equal(_h(vc[s, :, p + ln:]), _h(vc0[s, :, p + ln:])), \
            ("rows past the segment",) + where
        assert not torch.isnan(kc[s, :, p:p + ln].float()).any(), ("rows written",) + where
        r0 += ln


# ------------------------------------------------------------------------------------------------------------- 2. CPU graph
# (seq, tokens or a prompt length, n_past) per segment; prompt tokens are drawn per call.  Calls 1-2 keep T <= 32, 3-4 exceed it.
SCRIPT = [
    [(0, 5, 0), (1, 3, 0)],
    [(0, 1, 5), (1, 1, 3), (2, 6, 0), (3, 2, 0)],
    [(0, 1, 6), (2, 1, 6), (3, 4, 2), (4, 30, 0)],
    [(1, 1, 4), (4, 9, 30), (5, 40, 0), (0, 1, 7), (3, 1, 6)],
    [(5, 1, 40), (4, 1, 39), (2, 3, 7)],
]


@pytest.mark.parametrize("out_fmt", ["q4_0", "q6_K"])
def test_mixed_calls_match_the_cpu_graph_per_sequence(out_fmt):
    """GQA (4 heads on 2), six blocks: decode tokens with new prompts, prompt chunks continuing at n_past > 0, passes of 8 .. 51
    rows.  Each segment's last-token logits against the CPU graph evaluating that sequence alone; passes of T <= 32 rows under
    the running bar, longer ones (bf16 wgmma GEMM) under that bar or the wgmma bar of tests/test_gpu_llama.py, the larger."""
    m = toy(4, 2, out_fmt, seed=21, n_ctx=96)
    eng = m.engine(6)
    rng = np.random.default_rng(22)
    running = RunningBar()
    orcs = {s: SeqOracle(m, running) for s in range(6)}
    for call, segs in enumerate(SCRIPT):
        seqs = [s for s, _, _ in segs]
        toks = [[int(t) for t in rng.integers(3, 320, ln)] for _, ln, _ in segs]
        past = [p for _, _, p in segs]
        T = sum(len(t) for t in toks)
        logits, picks = eng.eval_batch(seqs, toks, past)
        for i, s in enumerate(seqs):
            want, tol = orcs[s].eval(toks[i], past[i])
            if T > 32:
                tol = max(tol, WGMMA_BAR)
            try:
                check_logits(logits[i], want, tol)
            except AssertionError as e:
                raise AssertionError(f"call {call} (T {T}) segment {i} (sequence {s}, n_past {past[i]}, {len(toks[i])} tokens): {e}") from None
            assert picks[i] == int(np.flatnonzero(logits[i] == logits[i].max())[0])
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 3. identities
def test_one_token_segments_are_decode_batch():
    m = toy(4, 2, seed=31, n_ctx=96)
    a, b = m.engine(4), m.engine(4)
    rng = np.random.default_rng(32)
    prompts = [[int(t) for t in rng.integers(3, 320, ln)] for ln in (3, 9, 5)]
    seqs = np.array([2, 0, 3], np.int32)
    for eng in (a, b):
        for s, p in zip(seqs, prompts):
            eng.eval_seq(int(s), p, 0, want_logits=False)
    past = np.array([len(p) for p in prompts], np.int32)
    for step in range(3):
        toks = rng.integers(3, 320, 3).astype(np.int32)
        la, pa = a.eval_batch(seqs, [[int(t)] for t in toks], past)
        lb, pb = b.decode_batch(seqs, toks, past)
        assert np.array_equal(bits(la), bits(lb)) and np.array_equal(pa, pb), step
        past += 1
    a.close()
    b.close()


@pytest.mark.parametrize("ln", [8, 20, 32])
def test_one_segment_is_eval_seq(ln):
    """a single segment of 8 .. 32 tokens at n_past 0 and a chunk after it: logits and pick bit-identical to eval_seq (both run
    attn_mma_kernel arithmetic and the integer tensor-core matmuls), then one-token steps that read the cache it left"""
    m = toy(4, 2, seed=33 + ln, n_ctx=96)
    a, b = m.engine(3), m.engine(3)
    rng = np.random.default_rng(ln)
    prompt = [int(t) for t in rng.integers(3, 320, ln)]
    chunk = [int(t) for t in rng.integers(3, 320, 8)]
    la, pa = a.eval_batch([1], [prompt], [0])
    lb, pb = b.eval_seq(1, prompt, 0)
    assert np.array_equal(bits(la[0]), bits(lb)) and pa[0] == pb
    la, pa = a.eval_batch([1], [chunk], [ln])
    lb, pb = b.eval_seq(1, chunk, ln)
    assert np.array_equal(bits(la[0]), bits(lb)) and pa[0] == pb
    n_past = ln + 8
    for t in (17, 250, 3):
        x, y = a.eval_seq(1, [t], n_past)[0], b.eval_seq(1, [t], n_past)[0]
        assert np.array_equal(bits(x), bits(y)), n_past
        n_past += 1
    a.close()
    b.close()


def test_segment_order_does_not_change_a_sequence():
    """T <= 32: the same five segments (two decodes, two prompts, a chunk) in two orders, then one more mixed call in two orders:
    per-sequence logits and picks bit-identical"""
    m = toy(4, 2, seed=35, n_ctx=96)
    a, b = m.engine(5), m.engine(5)
    rng = np.random.default_rng(36)
    pre = {s: [int(t) for t in rng.integers(3, 320, ln)] for s, ln in ((0, 4), (1, 6), (4, 3))}  # caches before the calls
    for eng in (a, b):
        for s, toks in pre.items():
            eng.eval_seq(s, toks, 0, want_logits=False)
    seqs, perm = [0, 1, 2, 3, 4], [3, 0, 4, 2, 1]
    # call 0: two decodes, two prompts and a chunk (23 rows); call 1: four decodes and a chunk (6 rows)
    for lens, past in (([1, 1, 9, 5, 7], [4, 6, 0, 0, 3]), ([1, 1, 1, 1, 2], [5, 7, 9, 5, 10])):
        toks = [[int(t) for t in rng.integers(3, 320, ln)] for ln in lens]
        la, pa = a.eval_batch(seqs, toks, past)
        lb, pb = b.eval_batch([seqs[j] for j in perm], [toks[j] for j in perm], [past[j] for j in perm])
        for jj, j in enumerate(perm):
            assert np.array_equal(bits(la[j]), bits(lb[jj])), (lens, seqs[j])
            assert pa[j] == pb[jj]
    a.close()
    b.close()


def test_the_block_holding_a_sequence_does_not_matter():
    """the same mixed calls with the sequences placed on other blocks: per-sequence logits bit-identical"""
    m = toy(4, 2, seed=37, n_ctx=96)
    a, b = m.engine(6), m.engine(6)
    rng = np.random.default_rng(38)
    place_b = {0: 5, 1: 2, 2: 0}
    prompts = {s: [int(t) for t in rng.integers(3, 320, ln)] for s, ln in ((0, 6), (1, 3))}
    for s, p in prompts.items():
        a.eval_seq(s, p, 0, want_logits=False)
        b.eval_seq(place_b[s], p, 0, want_logits=False)
    calls = [([0, 1, 2], [1, 1, 12], [6, 3, 0]), ([2, 0, 1], [5, 1, 4], [12, 7, 4])]
    for seqs, lens, past in calls:
        toks = [[int(t) for t in rng.integers(3, 320, ln)] for ln in lens]
        la, pa = a.eval_batch(seqs, toks, past)
        lb, pb = b.eval_batch([place_b[s] for s in seqs], toks, past)
        assert np.array_equal(bits(la), bits(lb)) and np.array_equal(pa, pb), seqs
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------------------- 4. serving
def test_a_serving_loop_admits_requests_into_the_running_pass():
    """five requests on four blocks.  Every step is one eval_batch: running requests decode their last pick, a new request's
    prompt joins the same pass, and a 40-token prompt is prefilled in chunks of 8 next to the decodes; the longest-running
    request retires after 8 decode steps and the next one takes its block at n_past 0.  The CPU graph of each request is fed the
    same segments: every segment's logits under the running bar (all passes stay at <= 32 rows), and every pick whose top-2
    margin there is unambiguous must be the CPU graph's greedy pick."""
    m = toy(4, 2, seed=41, n_ctx=64)
    eng = m.engine(4)
    running = RunningBar()
    rng = np.random.default_rng(42)
    arrivals = {0: [5, 3], 1: [40], 3: [6], 9: [4]}  # step -> prompt lengths of the requests arriving then
    chunk = 8

    class Req:
        def __init__(self, rid, block, prompt):
            self.rid, self.block, self.prompt, self.orc = rid, block, prompt, SeqOracle(m, running)
            self.done, self.n_past, self.last, self.decodes = 0, 0, None, 0

        def segment(self):
            if self.done < len(self.prompt):
                return self.prompt[self.done:self.done + chunk]
            return [self.last]

    active, next_id, free, checked = {}, 0, [0, 1, 2, 3], 0
    for step in range(14):
        for ln in arrivals.get(step, []):
            r = Req(next_id, free.pop(0), [int(t) for t in rng.integers(3, 320, ln)])
            active[r.block] = r
            next_id += 1
        reqs = [active[b] for b in sorted(active)]
        segs = [r.segment() for r in reqs]
        past = [r.n_past for r in reqs]
        assert sum(len(s) for s in segs) <= 32
        logits, picks = eng.eval_batch([r.block for r in reqs], segs, past)
        for r, seg, lg, pk in zip(reqs, segs, logits, picks):
            want, tol = r.orc.eval(seg, r.n_past)
            try:
                check_logits(lg, want, tol)
            except AssertionError as e:
                raise AssertionError(f"step {step} request {r.rid} (n_past {r.n_past}, {len(seg)} tokens): {e}") from None
            prefilling = r.done < len(r.prompt)
            r.done += len(seg) if prefilling else 0
            r.n_past += len(seg)
            if not prefilling:
                r.decodes += 1
            if r.done == len(r.prompt):
                if unambiguous(want):
                    assert int(pk) == greedy(want), (step, r.rid)
                    checked += 1
                r.last = int(pk)
        old = max(active.values(), key=lambda r: (r.decodes, -r.rid))
        if old.decodes >= 8:
            del active[old.block]
            free.append(old.block)
    assert next_id == 5 and checked >= 20, (next_id, checked)
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 5. launches
@pytest.mark.parametrize("lens", [(1, 1, 6), (1, 12, 20), (5, 9), (1, 3)])
def test_launch_structure_of_a_mixed_pass(lens):
    """per layer (two-layer count minus one-layer count), an eval_batch launches what a prompt of T = sum(lens) tokens does, plus
    one -- the batched decode attention of the one-token rows -- when the call has one-token and longer segments"""
    L = ns.lib()
    T = sum(lens)

    def counts(n_layer):
        eng = toy(4, 4, seed=43, n_layer=n_layer, n_ctx=96).engine(8)
        eng.eval_seq(7, [5] * T, 0, want_logits=False)  # buffers for T rows exist before counting
        eng.eval_batch([6, 7], [[3] * 2, [4] * 3], [0, T], want_logits=False)  # the plan tables too
        before = L.ns_launch_count()
        eng.eval_seq(5, [7] * T, 0, want_logits=False)
        prompt = L.ns_launch_count() - before
        before = L.ns_launch_count()
        eng.eval_batch(list(range(len(lens))), [[9] * ln for ln in lens], [10] * len(lens), want_logits=False)
        mixed = L.ns_launch_count() - before
        eng.close()
        return prompt, mixed

    p1, m1 = counts(1)
    p2, m2 = counts(2)
    extra = 1 if (1 in lens and max(lens) > 1) else 0
    assert m2 - m1 == (p2 - p1) + extra, (m2 - m1, p2 - p1, extra)


# ------------------------------------------------------------------------------------------------------------- 6. 7B shapes
def test_llama2_7b_shaped_mixed_pass_matches_the_reference_engine():
    """synthetic Llama-2-7B weights as tests/test_gpu_batch.py's 7B-shape test (Q4_0, two layers, the full output head).  Sequence
    A decodes, B's 30-token prompt arrives, C continues its prompt in chunks: one pass of 39 rows (bf16 wgmma GEMM), then one of
    6 rows.  Each segment against the reference engine (oracle.RefNeLlama where oracle/_ref is built, else OracleLlama) running
    that sequence alone, decode ids fed from it.  Bound: max(1e-2, 1.5 x the largest self-distance of the reference to its
    +-64 ulp jig seen so far), <= 2.5e-2; for the 39-row pass that bound or the wgmma bar, the larger."""
    rng = np.random.default_rng(78)
    m = llama2_7b_shaped(rng, n_ctx=64)
    m.draw_jig(rng)
    V = m.hp["n_vocab"]
    pa = [1] + [int(t) for t in rng.integers(3, V, 5)]
    pb = [1] + [int(t) for t in rng.integers(3, V, 29)]
    pc = [1] + [int(t) for t in rng.integers(3, V, 16)]  # C: 5 before the calls, then chunks of 8 and 4
    # per sequence: the segments it is evaluated in, in order ((tokens or None = the reference's previous pick), n_past)
    script = {"A": [(pa, 0), (None, 6), (None, 7)], "B": [(pb, 0), (None, 30)], "C": [(pc[:5], 0), (pc[5:13], 5), (pc[13:17], 13)]}
    wants, selfs, used = {}, {}, {}
    for which in ("ref", "jig"):
        r = m.reference(jig=which == "jig")
        for name, segs in script.items():
            out, toks_used = [], []
            for j, (toks, p) in enumerate(segs):
                if which == "jig":  # the reference's ids
                    toks = used[name][j]
                elif toks is None:
                    toks = [greedy(out[-1])]
                out.append(r.eval(toks, p))
                toks_used.append(toks)
            (wants if which == "ref" else selfs)[name] = out
            if which == "ref":
                used[name] = toks_used
        close(r)
    eng = m.engine(3)
    block = {"A": 2, "B": 0, "C": 1}
    eng.eval_seq(block["A"], pa, 0, want_logits=False)
    eng.eval_seq(block["C"], pc[:5], 0, want_logits=False)
    # call 1: A's first decode, B's prompt, C's first chunk (39 rows); call 2: A and B decode, C's second chunk (6 rows)
    calls = [[("A", 1), ("B", 0), ("C", 1)], [("A", 2), ("B", 1), ("C", 2)]]
    running, worst = RunningBar(), 0.0
    for ci, call in enumerate(calls):
        segs = [used[name][j] for name, j in call]
        past = [script[name][j][1] for name, j in call]
        T = sum(len(s) for s in segs)
        assert (T > 32) == (ci == 0), T
        logits, _ = eng.eval_batch([block[name] for name, _ in call], segs, past)
        for i, (name, j) in enumerate(call):
            want = wants[name][j]
            tol = running(want, selfs[name][j])
            if T > 32:
                tol = max(tol, WGMMA_BAR)
            s, err = scale(want), float(np.abs(logits[i] - want).max())
            assert err <= tol * s, (ci, name, err / s, running.floor)
            worst = max(worst, err / s)
    print(f"7B-shape mixed passes: worst |dlogit|/max|logit| {worst:.2e}; reference vs its jig {running.floor:.2e}")
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 7. arguments
def test_argument_checks_launch_nothing():
    L = ns.lib()
    eng = toy(4, 2, seed=44, n_ctx=16).engine(4)
    eng.eval_seq(1, [3, 4], 0, want_logits=False)
    h = eng.h
    i32 = lambda *v: np.array(v, np.int32)  # noqa: E731
    before = L.ns_launch_count()

    def rc_of(n, seq, n_tok, toks, past, handle=None):
        a = [x.ctypes.data if isinstance(x, np.ndarray) else x for x in (seq, n_tok, toks, past)]
        return L.ns_llama_eval_batch(h if handle is None else handle, n, *a, None, None)

    cases = [  # (n, seq, n_tokens, tokens, n_past), code, error text
        ((2, i32(0, 4), i32(1, 1), i32(1, 1), i32(0, 0)), E_INVALID, "outside [0, 4)"),
        ((1, i32(-1), i32(1), i32(1), i32(0)), E_INVALID, "outside [0, 4)"),
        ((2, i32(2, 2), i32(1, 3), i32(1, 1, 1, 1), i32(0, 0)), E_INVALID, "twice"),
        ((5, i32(0, 1, 2, 3, 0), i32(1, 1, 1, 1, 1), i32(1, 1, 1, 1, 1), i32(0, 0, 0, 0, 0)), E_INVALID, "outside [1, n_seq 4]"),
        ((0, i32(0), i32(1), i32(1), i32(0)), E_INVALID, "outside [1, n_seq 4]"),
        ((2, i32(0, 1), i32(2, 0), i32(1, 1), i32(0, 0)), E_INVALID, "n_tokens 0 < 1"),
        ((1, i32(0), i32(1), i32(1), i32(-1)), E_INVALID, "n_ctx 16"),
        ((1, i32(0), i32(5), i32(1, 1, 1, 1, 1), i32(12)), E_INVALID, "n_past 12 + 5 tokens outside n_ctx 16"),
        ((1, i32(0), i32(1), i32(1), i32(16)), E_INVALID, "n_ctx 16"),
        ((1, None, i32(1), i32(1), i32(0)), E_INVALID, "null"),
        ((1, i32(0), None, i32(1), i32(0)), E_INVALID, "null"),
        ((1, i32(0), i32(1), None, i32(0)), E_INVALID, "null"),
        ((1, i32(0), i32(1), i32(1), None), E_INVALID, "null"),
    ]
    for j, (args, code, text) in enumerate(cases):
        rc = rc_of(*args)
        assert rc == code and text in ns.last_error(), (j, rc, ns.last_error())
    assert L.ns_llama_eval_batch(None, 1, i32(0).ctypes.data, i32(1).ctypes.data, i32(1).ctypes.data, i32(0).ctypes.data, None,
                                 None) == E_INVALID and "null" in ns.last_error()
    # the one-layer ragged attention entry: the same segment rules, then the head size
    q = torch.zeros(64, device="cuda")
    p_ = q.data_ptr()
    for (n_seq, n, s, t, p, hd, n_ctx), code, text in (((2, 2, i32(0, 0), i32(1, 1), i32(0, 0), 64, 64), E_INVALID, "twice"),
                                                         ((2, 1, i32(2), i32(1), i32(0), 64, 64), E_INVALID, "outside [0, 2)"),
                                                         ((2, 1, i32(0), i32(0), i32(0), 64, 64), E_INVALID, "n_tokens 0"),
                                                         ((2, 1, i32(0), i32(9), i32(60), 64, 64), E_INVALID, "n_ctx 64"),
                                                         ((33, 1, i32(0), i32(1), i32(0), 64, 64), E_INVALID, "invalid arguments"),
                                                         ((2, 1, i32(0), i32(1), i32(0), 80, 64), E_UNSUPPORTED, "head size 80")):
        rc = L.ns_llama_attention_ragged(p_, p_, p_, p_, p_, n_seq, n, s.ctypes.data, t.ctypes.data, p.ctypes.data, 8, 2, hd, n_ctx,
                                         10000.0, 1.0, p_, p_, None)
        assert rc == code and text in ns.last_error(), (n_seq, n, rc, ns.last_error())
    assert L.ns_launch_count() == before
    eng.close()
    big = toy(4, 2, seed=45, n_ctx=4200, n_layer=1).engine(2)  # the per-call row cap
    exact = toy(4, 2, seed=46, n_ctx=64, n_layer=1).engine(4)
    exact.set_exact_prefill(True)
    ring = toy(4, 2, seed=47, n_ctx=16, n_layer=1).engine(1)
    ring.set_streaming(4)
    odd = toy(8, 4, seed=48, n_ctx=16, n_layer=1).engine(1)  # head size 32
    before = L.ns_launch_count()
    assert rc_of(2, i32(0, 1), i32(4000, 97), np.ones(4097, np.int32), i32(0, 0), big.h) == E_INVALID
    assert "4097 rows in one pass, at most 4096" in ns.last_error()
    assert rc_of(3, i32(0, 1, 2), i32(11, 11, 11), np.ones(33, np.int32), i32(0, 0, 0), exact.h) == E_UNSUPPORTED
    assert "exact-prefill" in ns.last_error()
    assert rc_of(1, i32(0), i32(1), i32(1), i32(0), ring.h) == E_UNSUPPORTED and "streaming" in ns.last_error()
    assert rc_of(1, i32(0), i32(3), i32(1, 2, 3), i32(0), odd.h) == E_UNSUPPORTED and "head size 32" in ns.last_error()
    assert L.ns_launch_count() == before
    for e in (big, exact, ring, odd):
        e.close()

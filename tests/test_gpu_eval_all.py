"""Every token's logits and target log-probabilities from one eval-step pass (ns_llama_eval_all, include/ns_b200.h): the
reference's model_eval with logits_all, over the segments of ns_llama_eval_batch, scored on the device.

1. the log-prob kernel on its own equals its host restatement bit for bit (ties, -inf and NaN rows, poisoned workspace);
2. every row's logits against the CPU restatement of the reference graph (oracle/llama_model.py), each sequence alone;
3. the log-probs and picks are the host restatement applied to the returned logits, bit for bit;
4. identities with ns_llama_decode_batch and ns_llama_eval_batch, the KV cache left behind, segment order and block placement;
5. Llama-2-7B shapes against the reference engine, every row of a prompt;
6. the launch structure per lm_head route, and 7. refusals that launch nothing."""
import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
from llama_models import RunningBar, bar, bits, close, distance, llama2_7b_shaped, rows, scale, toy, unambiguous
from oracle.llama_model import greedy

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4
WGMMA_BAR = 4e-2  # passes of more than 32 rows take the bf16 wgmma GEMM in the body: tests/test_gpu_llama.py's bar for that path


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def _targets(rng, token_lists):
    return [[int(t) for t in rng.integers(0, 320, len(toks))] for toks in token_lists]


# ------------------------------------------------------------------------------------------------------------- 1. kernel
def _special_rows(rng, n, V):
    """random rows with ties, -inf entries, an all -inf row and a NaN row among them"""
    x = (rng.standard_normal((n, V)) * rng.choice([1e-2, 1.0, 30.0], (n, 1))).astype(np.float32)
    for r in range(n):
        kind = r % 6
        if kind == 1:
            peak = x[r].max() + 1
            x[r, rng.integers(0, V, 3)] = peak  # a three-way tie for the max
        elif kind == 2:
            x[r, ::5] = -np.inf
        elif kind == 3 and r > 6:
            x[r] = -np.inf
        elif kind == 4 and r > 6:
            x[r] = np.nan
        elif kind == 5:
            x[r, rng.integers(0, V)] = np.nan
    return x


@pytest.mark.parametrize("V", [320, 32000, 128256])
def test_kernel_equals_the_host_restatement(V):
    """1 .. 32 rows; targets include -inf entries and the argmax; workspace poisoned with 0xFF apart from the zeroed tickets, which
    are zero again after every call; argmax alone, and log-probs alone, too"""
    rng = np.random.default_rng(V)
    ns_list = (1, 2, 3, 7, 13, 31, 32) if V == 320 else (1, 6, 32)
    wsb = ns.lib().ns_llama_logprob_workspace_bytes(32, V)
    ws = torch.full((wsb,), 0xFF, dtype=torch.uint8, device="cuda")
    ws[:128] = 0
    for n in ns_list:
        x = _special_rows(rng, n, V)
        t = rng.integers(0, V, n).astype(np.int32)
        t[0] = int(np.nanargmax(np.where(np.isnan(x[0]), -np.inf, x[0])))
        if n > 2:
            t[2] = 0  # a -inf entry of row 2
        xd, td = torch.from_numpy(x).cuda(), torch.from_numpy(t).cuda()
        lp = torch.full((n,), 7.0, device="cuda")
        am = torch.full((n,), -5, dtype=torch.int32, device="cuda")
        for mode in ("both", "argmax", "logprob"):
            lp.fill_(7.0)
            am.fill_(-5)
            torch.cuda.synchronize()
            rc = ns.logprob(xd.data_ptr(), n, V, td.data_ptr() if mode != "argmax" else None, lp.data_ptr() if mode != "argmax" else None,
                            am.data_ptr() if mode != "logprob" else None, ws.data_ptr())
            assert rc == 0, ns.last_error()
            torch.cuda.synchronize()
            assert torch.count_nonzero(ws[:128]).item() == 0, (n, mode)
            glp, gam = lp.cpu().numpy(), am.cpu().numpy()
            for r in range(n):
                wlp, wam = ns.logprob_row_host(x[r], int(t[r]))
                if mode != "argmax":
                    assert bits(np.float32(wlp)) == bits(glp[r:r + 1])[0] or (np.isnan(wlp) and np.isnan(glp[r])), (n, r, wlp, glp[r])
                else:
                    assert glp[r] == 7.0
                if mode != "logprob":
                    assert gam[r] == wam, (n, r, gam[r], wam)
                else:
                    assert gam[r] == -5
    # row kinds seen: ties, -inf targets, an all -inf row and a NaN row
    assert np.isneginf(ns.logprob_row_host(_special_rows(np.random.default_rng(V), 3, V)[2], 0)[0])


def test_kernel_argument_checks():
    L = ns.lib()
    x = torch.zeros(4, 320, device="cuda")
    p = x.data_ptr()
    before = L.ns_launch_count()
    for args in ((p, 0, 320, p, p, p, p), (p, 33, 320, p, p, p, p), (p, 1, 0, p, p, p, p), (p, 1, 320, p, None, p, p),
                 (p, 1, 320, None, p, p, p), (p, 1, 320, None, None, None, p), (None, 1, 320, p, p, p, p), (p, 1, 320, p, p, p, None)):
        assert L.ns_llama_logprob(*args, None) == E_INVALID, args
    assert L.ns_launch_count() == before


# ------------------------------------------------------------------------------------------------------------- 2. CPU graph
# (seq, length, n_past) per segment: lengths 1, 2 .. 7, 8 .. 32 and > 64, at n_past 0 and > 0; call 2 exceeds 32 rows
SCRIPT = [
    [(0, 5, 0), (1, 3, 0)],
    [(0, 1, 5), (1, 1, 3), (2, 7, 0), (3, 12, 0)],
    [(2, 1, 7), (3, 70, 12), (4, 2, 0)],
    [(0, 1, 6), (4, 24, 2), (1, 1, 4)],
]


@pytest.mark.parametrize("out_fmt", ["q4_0", "q6_K"])
def test_every_row_matches_the_cpu_graph_per_sequence(out_fmt):
    """every row's logits against the CPU graph evaluating that sequence alone, row by row (rows: the reference's logits_all).  The
    bar is the running bar over the whole script: the CPU graph and its jig run every call first (the segments do not depend on the
    engine), so the bar holds the model's conditioning over every row the test checks, not only over the rows before the one
    being checked; passes of T > 32 rows take that bar or the wgmma bar, the larger.  Where a row's top-2 margin is unambiguous
    its pick is the CPU graph's greedy pick."""
    m = toy(4, 2, out_fmt, seed=51, n_ctx=96)
    eng = m.engine(6)
    rng = np.random.default_rng(52)
    orcs = {s: (m.graph(), m.graph(jig=True)) for s in range(6)}
    running = RunningBar()
    calls = []
    for segs in SCRIPT:
        seqs = [s for s, _, _ in segs]
        toks = [[int(t) for t in rng.integers(3, 320, ln)] for _, ln, _ in segs]
        past = [p for _, _, p in segs]
        wants = []
        for i, s in enumerate(seqs):
            want = rows(orcs[s][0], toks[i], past[i])
            jig = rows(orcs[s][1], toks[i], past[i])
            for r in range(len(toks[i])):
                tol = running(want[r], jig[r])
            wants.append(want)
        calls.append((seqs, toks, past, wants))
    picked = 0
    for call, (seqs, toks, past, wants) in enumerate(calls):
        T = sum(len(t) for t in toks)
        _, picks, logits = eng.eval_all(seqs, toks, past, want_logits=True)
        tol_T = max(tol, WGMMA_BAR) if T > 32 else tol
        for i, s in enumerate(seqs):
            for r in range(len(toks[i])):
                w = wants[i][r]
                sc, err = scale(w), float(np.abs(logits[i][r] - w).max())
                assert err <= tol_T * sc, (call, T, i, s, r, err / sc, tol_T)
                if unambiguous(w, 2 * tol_T):
                    assert int(picks[i][r]) == greedy(w), (call, i, r)
                    picked += 1
    print(f"{out_fmt} lm_head: bar {tol:.2e} of max|logit|, {picked} unambiguous picks")
    assert picked >= 20, picked
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 3. own logits
@pytest.mark.parametrize("out_fmt", ["q4_0", "q6_K"])
def test_logprobs_are_the_host_arithmetic_on_the_returned_logits(out_fmt):
    """targets drawn per token; passes of 8, 21, 73 (three lm_head chunks) and 27 rows: every log-prob and pick equals
    ns_logprob_row_host on that row of logits_host, bit for bit, and a call without logits_host returns the same"""
    m = toy(4, 2, out_fmt, seed=53, n_ctx=96)
    a, b = m.engine(6), m.engine(6)
    rng = np.random.default_rng(54)
    for call, segs in enumerate(SCRIPT):
        seqs = [s for s, _, _ in segs]
        toks = [[int(t) for t in rng.integers(3, 320, ln)] for _, ln, _ in segs]
        past = [p for _, _, p in segs]
        tg = _targets(rng, toks)
        lp, am, lg = a.eval_all(seqs, toks, past, targets=tg, want_logits=True)
        lp2, am2, lg2 = b.eval_all(seqs, toks, past, targets=tg)
        assert lg2 is None
        T = sum(len(t) for t in toks)
        for i in range(len(seqs)):
            for r in range(len(toks[i])):
                wlp, wam = ns.logprob_row_host(lg[i][r], tg[i][r])
                assert bits(np.float32(wlp)) == bits(lp[i][r:r + 1])[0], (call, i, r, wlp, lp[i][r])
                assert am[i][r] == wam, (call, i, r)
            if T <= 32:  # larger passes take the bf16 GEMM's split-K in the body: not bit-reproducible across engines
                assert np.array_equal(bits(lp[i]), bits(lp2[i])) and np.array_equal(am[i], am2[i]), (call, i)
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------------------- 4. identities
def _history(engs, rng, prompts):
    for eng in engs:
        for s, p in prompts.items():
            eng.eval_seq(s, p, 0, want_logits=False)


def test_one_token_segments_are_decode_batch():
    """three one-token segments: the logits and picks of every row bit-identical to ns_llama_decode_batch (same kernels, same
    lm_head route and RMSNorm fold at that row count), and the next steps of both agree"""
    m = toy(4, 2, seed=61, n_ctx=96)
    a, b = m.engine(4), m.engine(4)
    rng = np.random.default_rng(62)
    prompts = {2: [int(t) for t in rng.integers(3, 320, 3)], 0: [int(t) for t in rng.integers(3, 320, 9)],
               3: [int(t) for t in rng.integers(3, 320, 5)]}
    _history((a, b), rng, prompts)
    seqs = np.array([2, 0, 3], np.int32)
    past = np.array([3, 9, 5], np.int32)
    for step in range(3):
        toks = rng.integers(3, 320, 3).astype(np.int32)
        _, pa, la = a.eval_all(seqs, [[int(t)] for t in toks], past, want_logits=True)
        lb, pb = b.decode_batch(seqs, toks, past)
        assert np.array_equal(bits(np.concatenate(la)), bits(lb)) and np.array_equal(np.concatenate(pa), pb), step
        past += 1
    a.close()
    b.close()


@pytest.mark.parametrize("out_fmt", ["q6_K", "q4_0"])
def test_last_rows_are_eval_batch(out_fmt):
    """mixed passes of T <= 32 rows: each segment's last-row logits against ns_llama_eval_batch on another engine -- bit for bit
    with the Q6_K lm_head (its 4-row tiles are row-exact), within 1e-4 of max|logit| with Q4_0 (the lm_head runs at the chunk's
    row count, where only the fp32 order of the integer block sums differs).  Then the KV caches the two passes left: one
    decode_batch step on each, bit-identical."""
    m = toy(4, 2, out_fmt, seed=63, n_ctx=96)
    a, b = m.engine(5), m.engine(5)
    rng = np.random.default_rng(64)
    _history((a, b), rng, {0: [int(t) for t in rng.integers(3, 320, 4)], 1: [int(t) for t in rng.integers(3, 320, 6)]})
    calls = [([0, 1, 2, 3], [1, 1, 9, 5], [4, 6, 0, 0]), ([2, 4, 0], [3, 20, 1], [9, 0, 5]), ([1, 3, 4], [2, 8, 1], [7, 5, 20])]
    for seqs, lens, past in calls:
        toks = [[int(t) for t in rng.integers(3, 320, ln)] for ln in lens]
        _, _, la = a.eval_all(seqs, toks, past, want_logits=True)
        lb, _ = b.eval_batch(seqs, toks, past)
        for i in range(len(seqs)):
            if out_fmt == "q6_K":
                assert np.array_equal(bits(la[i][-1]), bits(lb[i])), (seqs, i)
            else:
                assert float(np.abs(la[i][-1] - lb[i]).max()) <= 1e-4 * float(np.abs(lb[i]).max()), (seqs, i)
    seqs = [0, 1, 2, 3, 4]
    past = [6, 9, 12, 13, 21]
    toks = rng.integers(3, 320, 5).astype(np.int32)
    x, px = a.decode_batch(seqs, toks, past)
    y, py = b.decode_batch(seqs, toks, past)
    assert np.array_equal(bits(x), bits(y)) and np.array_equal(px, py)
    a.close()
    b.close()


def test_segment_order_and_block_placement_change_nothing():
    """T <= 32: the same segments in two orders on two block placements, targets along: per-sequence log-probs, picks and logits
    bit-identical"""
    m = toy(4, 2, seed=65, n_ctx=96)
    a, b = m.engine(6), m.engine(6)
    rng = np.random.default_rng(66)
    place = {0: 5, 1: 2, 2: 0, 3: 4, 4: 1}
    pre = {s: [int(t) for t in rng.integers(3, 320, ln)] for s, ln in ((0, 4), (1, 6), (4, 3))}
    for s, toks in pre.items():
        a.eval_seq(s, toks, 0, want_logits=False)
        b.eval_seq(place[s], toks, 0, want_logits=False)
    seqs, perm = [0, 1, 2, 3, 4], [3, 0, 4, 2, 1]
    for lens, past in (([1, 1, 9, 5, 7], [4, 6, 0, 0, 3]), ([1, 1, 1, 1, 2], [5, 7, 9, 5, 10])):
        toks = [[int(t) for t in rng.integers(3, 320, ln)] for ln in lens]
        tg = _targets(rng, toks)
        la = a.eval_all(seqs, toks, past, targets=tg, want_logits=True)
        lb = b.eval_all([place[seqs[j]] for j in perm], [toks[j] for j in perm], [past[j] for j in perm], targets=[tg[j] for j in perm],
                        want_logits=True)
        for jj, j in enumerate(perm):
            for k in range(3):
                assert np.array_equal(bits(la[k][j]), bits(lb[k][jj])), (lens, j, k)
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------------------- 5. 7B shapes
def test_llama2_7b_shaped_prompt_rows_match_the_reference_engine():
    """synthetic Llama-2-7B weights as tests/test_gpu_llama.py's 7B-shape test (Q4_0, two layers, the full output head).  Every row
    of a 12-token prompt against the reference engine's logits_all rows (rows: the prompt evaluated token by token, as that test
    does, on oracle.RefNeLlama where oracle/_ref is built, else OracleLlama), under that test's bar: max(1e-2, 1.5 x the largest
    self-distance of the reference to its +-64 ulp jig over the rows), <= 2.5e-2.  Log-probs of the next prompt token along, against float64 log_softmax of the reference's rows."""
    rng = np.random.default_rng(2024)
    m = llama2_7b_shaped(rng, n_ctx=64)
    prompt = [1] + [int(t) for t in rng.integers(3, m.hp["n_vocab"], 11)]
    m.draw_jig(rng)
    refs = m.reference(), m.reference(jig=True)
    want, self_w = (rows(r, prompt, 0) for r in refs)
    close(*refs)
    eng = m.engine()
    targets = prompt[1:] + [prompt[0]]
    lp, am, got = eng.eval_all([0], [prompt], [0], targets=[targets], want_logits=True)
    lp, am, got = lp[0], am[0], got[0]
    worst_self = max(distance(self_w[r], want[r]) for r in range(len(prompt)))
    bound = bar(worst_self)
    worst, worst_lp = 0.0, 0.0
    for r in range(len(prompt)):
        sc, err = scale(want[r]), float(np.abs(got[r] - want[r]).max())
        assert err <= bound * sc, (r, err / sc, worst_self)
        worst = max(worst, err / sc)
        w64 = want[r].astype(np.float64)
        wlp = w64[targets[r]] - w64.max() - np.log(np.exp(w64 - w64.max()).sum())
        worst_lp = max(worst_lp, abs(float(lp[r]) - wlp))
        assert abs(float(lp[r]) - wlp) <= 2 * bound * sc, (r, float(lp[r]), wlp)
        if unambiguous(want[r], 2 * bound):
            assert int(am[r]) == greedy(want[r]), r
    print(f"7B-shape logits_all rows: worst |dlogit|/max|logit| {worst:.2e}; reference vs its jig {worst_self:.2e}; "
          f"worst |dlogprob| {worst_lp:.2e}")
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 6. launches
def _mm_launches(w, rows, E, V):
    """launches of the lm_head's ns_mul_mat at `rows` rows on its own"""
    L = ns.lib()
    act = torch.zeros(rows, E, device="cuda")
    out = torch.zeros(rows, V, device="cuda")
    before = L.ns_launch_count()
    ns.mul_mat(w, act.data_ptr(), E, out.data_ptr(), V, rows)
    n = L.ns_launch_count() - before
    torch.cuda.synchronize()
    return n


@pytest.mark.parametrize("out_fmt", ["q4_0", "q6_K"])
@pytest.mark.parametrize("lens", [(1, 1, 6), (1, 12, 20), (5, 9), (40, 30)])
def test_launch_structure(out_fmt, lens):
    """eval_all launches the body of eval_batch on the same segments, then the final RMSNorm unless folded, then per chunk of <= 32
    rows the lm_head's own launches at that row count and one log-prob launch; asking only for picks adds nothing"""
    L = ns.lib()
    m = toy(4, 4, out_fmt, seed=71, n_ctx=96)
    eng = m.engine(8)
    T, n = sum(lens), len(lens)
    E, V = 256, 320
    seqs, toks, past = list(range(n)), [[9] * ln for ln in lens], [10] * n
    eng.eval_batch([6, 7], [[3] * 2, [4] * T], [0, 0], want_logits=False)  # buffers and plan tables exist before counting
    eng.eval_all([6, 7], [[3] * 2, [4] * T], [0, 0], targets=[[1] * 2, [1] * T], want_logits=True)
    before = L.ns_launch_count()
    eng.eval_batch(seqs, toks, past, want_logits=False)
    batch = L.ns_launch_count() - before
    counts = {}
    for mode in ("targets", "picks", "logits"):
        before = L.ns_launch_count()
        eng.eval_all(seqs, toks, past, targets=[[2] * ln for ln in lens] if mode == "targets" else None, want_logits=mode == "logits")
        counts[mode] = L.ns_launch_count() - before
    w = (ns.Weight.from_q6_K_host if out_fmt == "q6_K" else ns.Weight.from_q4_0_host)(m.out_rows, V, E)
    fold_n = ns.rmsnorm_fusable([w], n)
    body = batch - (1 + (0 if fold_n else 1) + _mm_launches(w, n, E, V) + 1)  # gather, norm, lm_head, argmax
    fold_T = T <= 32 and ns.rmsnorm_fusable([w], T)
    head = (0 if fold_T else 1) + sum(_mm_launches(w, min(32, T - r0), E, V) + 1 for r0 in range(0, T, 32))
    assert counts["targets"] == counts["picks"] == counts["logits"] == body + head, (counts, body, head, batch)
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 7. refusals
def test_refusals_launch_nothing():
    L = ns.lib()
    eng = toy(4, 2, seed=72, n_ctx=16).engine(4)
    eng.eval_seq(1, [3, 4], 0, want_logits=False)
    h = eng.h
    i32 = lambda *v: np.array(v, np.int32)  # noqa: E731
    lp = np.zeros(4200, np.float32)
    am = np.zeros(4200, np.int32)
    tg = np.zeros(4200, np.int32)

    def rc_of(n, seq, n_tok, toks, past, handle=None, targets=tg, logprobs=lp, argmax=am, logits=None):
        a = [x.ctypes.data if isinstance(x, np.ndarray) else x for x in (seq, n_tok, toks, past, targets, logprobs, argmax, logits)]
        return L.ns_llama_eval_all(h if handle is None else handle, n, *a)

    ok = (1, i32(0), i32(2), i32(1, 1), i32(0))
    cases = [  # eval_batch's rules, then the new ones
        (dict(args=(2, i32(0, 4), i32(1, 1), i32(1, 1), i32(0, 0))), E_INVALID, "outside [0, 4)"),
        (dict(args=(2, i32(2, 2), i32(1, 3), i32(1, 1, 1, 1), i32(0, 0))), E_INVALID, "twice"),
        (dict(args=(0, i32(0), i32(1), i32(1), i32(0))), E_INVALID, "outside [1, n_seq 4]"),
        (dict(args=(2, i32(0, 1), i32(2, 0), i32(1, 1), i32(0, 0))), E_INVALID, "n_tokens 0 < 1"),
        (dict(args=(1, i32(0), i32(5), i32(1, 1, 1, 1, 1), i32(12))), E_INVALID, "n_past 12 + 5 tokens outside n_ctx 16"),
        (dict(args=(1, None, i32(1), i32(1), i32(0))), E_INVALID, "null"),
        (dict(args=(1, i32(0), None, i32(1), i32(0))), E_INVALID, "null"),
        (dict(args=(1, i32(0), i32(1), None, i32(0))), E_INVALID, "null"),
        (dict(args=(1, i32(0), i32(1), i32(1), None)), E_INVALID, "null"),
        (dict(args=ok, targets=i32(3, 320)), E_INVALID, "target 320 of row 1 outside [0, n_vocab 320)"),
        (dict(args=ok, targets=i32(-1, 0)), E_INVALID, "target -1 of row 0"),
        (dict(args=ok, targets=None), E_INVALID, "both null or both non-null"),
        (dict(args=ok, logprobs=None), E_INVALID, "both null or both non-null"),
        (dict(args=ok, targets=None, logprobs=None, argmax=None, logits=None), E_INVALID, "one output"),
    ]
    before = L.ns_launch_count()
    for j, (kw, code, text) in enumerate(cases):
        args = kw.pop("args")
        rc = rc_of(*args, **kw)
        assert rc == code and text in ns.last_error(), (j, rc, ns.last_error())
    one, zero = i32(1), i32(0)
    assert L.ns_llama_eval_all(None, 1, zero.ctypes.data, one.ctypes.data, one.ctypes.data, zero.ctypes.data, None, None, am.ctypes.data,
                               None) == E_INVALID and "null" in ns.last_error()
    eng.set_sampling(top_k=40, seed=3)
    assert rc_of(*ok) == E_UNSUPPORTED and "sampling" in ns.last_error()
    assert L.ns_launch_count() == before
    eng.set_sampling(None)
    eng.close()
    big = toy(4, 2, seed=73, n_ctx=4200, n_layer=1).engine(2)  # the per-call row cap
    exact = toy(4, 2, seed=74, n_ctx=64, n_layer=1).engine(4)
    exact.set_exact_prefill(True)
    ring = toy(4, 2, seed=75, n_ctx=16, n_layer=1).engine(1)
    ring.set_streaming(4)
    odd = toy(8, 4, seed=76, n_ctx=16, n_layer=1).engine(1)  # head size 32
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

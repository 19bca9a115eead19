"""Continuous batching in the eval step (ns_llama_set_sequences / eval_seq / decode_batch / generate_batch, include/ns_b200.h):
one KV block per sequence, one forward pass for the decode tokens of many sequences.

* the batched decode attention on its own against the single-sequence split decode kernel, row by row, bit for bit;
* batched steps against the CPU restatement of the reference graph (oracle/llama_model.py), each row against its sequence alone;
* results independent of the batch: row order, which block holds a sequence, and how many blocks the context has;
* device-fed generation against a loop of batched steps, a serving loop that retires and admits requests between chunks;
* the launch structure of a batched step, Llama-2-7B shapes against the reference engine, and the argument checks."""
import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
from llama_models import RunningBar, SeqOracle, bits, check_logits, close, llama2_7b_shaped, scale, toy, unambiguous
from oracle import llama_model as lm
from oracle.llama_model import greedy

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


# ------------------------------------------------------------------------------------------------------------- 1. kernel
N_CTX_K = 1100  # 5 ranges of 256 positions
PASTS = (0, 255, 256, 257, N_CTX_K - 1)


def _single(q, k, v, kc, vc, H, HK, hd, n_past, kernel=ns.ATTN_SPLIT_DECODE):
    """one ns_llama_attention call on the library's stream: torch's work on the inputs is finished first, the call's after"""
    ws = torch.zeros(ns.lib().ns_llama_attention_workspace_bytes(H, hd, N_CTX_K), dtype=torch.uint8, device="cuda")
    out = torch.full((1, H * hd), float("nan"), device="cuda")
    torch.cuda.synchronize()
    rc = ns.lib().ns_llama_attention(kernel, q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), H, HK, hd, N_CTX_K,
                                     n_past, 1, 10000.0, 1.0, out.data_ptr(), ws.data_ptr(), None)
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    return out


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("n_head,n_head_kv", [(8, 8), (8, 2)])
@pytest.mark.parametrize("n", [1, 3, 8, 32])
def test_batched_attention_is_the_split_decode_kernel_row_by_row(n, n_head, n_head_kv, hd):
    """n rows on n of n_seq blocks (n_seq = min(n + 2, 32): unused blocks for n < 32), per-row n_past 0, 255, 256, 257 and
    n_ctx - 1 mixed with random ones.  Every cache row from a row's n_past on, and every row of an unused block, is NaN: reading
    one would poison that row's output.  Against n ns_llama_attention(NS_ATTN_SPLIT_DECODE) calls on copies of the same blocks:
    out and every block bit-identical; unused blocks unchanged; tickets zero; the output against the CPU attention model within
    test_gpu_attention.py's split decode bars: 5e-5 of max|V| for any element, 1e-3 of the reference order, and for the mean
    2e-6 -- on these inputs the split decode kernel itself (bit-identical) reaches 1.7e-6 on one row (hd 128, GQA, n = 32),
    above the 1e-6 that file's cases allow."""
    H, HK = n_head, n_head_kv
    n_seq = min(n + 2, 32)
    rng = np.random.default_rng(n * 1000 + hd + HK)
    seqs = rng.permutation(n_seq)[:n].astype(np.int32)
    past = np.array([PASTS[i] if i < len(PASTS) else int(rng.integers(0, N_CTX_K)) for i in range(n)], np.int32)
    rng.shuffle(past)
    g = torch.Generator(device="cuda").manual_seed(int(n * 7 + hd))
    kc = torch.full((n_seq, HK, N_CTX_K, hd), float("nan"), dtype=torch.float16, device="cuda")
    vc = torch.full_like(kc, float("nan"))
    for s, p in zip(seqs.tolist(), past.tolist()):
        if p:
            kc[s, :, :p] = torch.randn((HK, int(p), hd), generator=g, device="cuda").half()
            vc[s, :, :p] = torch.randn((HK, int(p), hd), generator=g, device="cuda").half()
    q = torch.from_numpy(rng.normal(0, 2.0, (n, H * hd)).astype(np.float32)).cuda()
    k = torch.from_numpy(rng.normal(0, 1.0, (n, HK * hd)).astype(np.float32)).cuda()
    v = torch.from_numpy(rng.normal(0, 1.0, (n, HK * hd)).astype(np.float32)).cuda()
    kc0, vc0 = kc.clone(), vc.clone()

    wsb = ns.lib().ns_llama_attention_batch_workspace_bytes(n, H, hd, N_CTX_K)
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    t_off = (16 * n + (4 * n + 15) // 16 * 16)
    p_off = t_off + (4 * n * H + 15) // 16 * 16
    ws[p_off:] = 0xFF  # partials NaN: no value may be carried into a call
    out = torch.full((n, H * hd), float("nan"), device="cuda")
    torch.cuda.synchronize()
    rc = ns.attention_batch(q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), n_seq, seqs, past, H, HK, hd, N_CTX_K,
                            out.data_ptr(), ws.data_ptr())
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    assert (ws[t_off:t_off + 4 * n * H].view(torch.int32) == 0).all(), "tickets not zero after the call"
    got = out.cpu().numpy()
    assert np.isfinite(got).all()
    used = set(int(s) for s in seqs)
    for s in range(n_seq):
        if s not in used:
            assert torch.equal(kc[s].view(torch.int16), kc0[s].view(torch.int16)) and torch.equal(vc[s].view(torch.int16), vc0[s].view(torch.int16)), s
    bar_max, bar_mean = 5e-5, 2e-6  # BARS[SPLIT] of tests/test_gpu_attention.py, the mean as measured here (docstring)
    for i, (s, p) in enumerate(zip(seqs.tolist(), past.tolist())):
        kci, vci = kc0[s].clone(), vc0[s].clone()
        qi = q[i:i + 1].clone()
        one = _single(qi, k[i:i + 1], v[i:i + 1], kci, vci, H, HK, hd, int(p))
        assert np.array_equal(bits(one.cpu().numpy()[0]), bits(got[i])), ("out", i, int(s), int(p))
        assert torch.equal(kc[s].view(torch.int16), kci.view(torch.int16)) and torch.equal(vc[s].view(torch.int16), vci.view(torch.int16)), \
            ("cache block", i, int(s), int(p))
        # against the CPU model, with q rotated by rope_kv_kernel (the fused kernel's sincosf arithmetic), as test_gpu_attention.py
        qr = q[i:i + 1].clone()
        _single(qr, k[i:i + 1], v[i:i + 1], kc0[s].clone(), vc0[s].clone(), H, HK, hd, int(p), kernel=ns.ATTN_GENERIC)
        q_rot = qr.cpu().numpy().reshape(1, H, hd)
        L = int(p) + 1
        kch, vch = kc[s, :, :L].cpu().numpy(), vc[s, :, :L].cpu().numpy()
        vmax = float(np.abs(vch.astype(np.float32)).max())
        ref = lm.attention_reference(q_rot, kch, vch, int(p))
        mine = got[i].reshape(1, H, hd)
        if (L + lm.SPLIT_KEYS - 1) // lm.SPLIT_KEYS > 1:
            stated = lm.attention_stated(q_rot, kch, vch, int(p), "split")
            assert float(np.abs(mine - ref).max()) / float(np.abs(ref).max()) <= 1e-3
        else:
            stated = ref
        d = np.abs(mine.astype(np.float64) - stated)
        assert float(d.max()) / vmax <= bar_max and float(d.mean()) / vmax <= bar_mean, (i, p, float(d.max()) / vmax, float(d.mean()) / vmax)


# ------------------------------------------------------------------------------------------------------------- 2. CPU graph
@pytest.mark.parametrize("n,out_fmt", [(2, "q4_0"), (3, "q4_0"), (8, "q4_0"), (32, "q4_0"), (3, "q6_K"), (8, "q6_K")])
def test_decode_batch_matches_the_cpu_graph_per_sequence(n, out_fmt):
    """GQA (4 heads on 2), prompts of 1 .. 7 tokens per sequence through eval_seq (below the tensor-core prompt attention, whose
    numerics tests/test_gpu_llama.py covers), then three batched steps; every row against the CPU graph evaluating that sequence
    alone.  n = 2 runs the matmuls as GEMV tiles, 3 and more on the integer tensor cores."""
    m = toy(4, 2, out_fmt, seed=40 + n)
    eng = m.engine(n)
    rng = np.random.default_rng(n)
    seqs = rng.permutation(n).astype(np.int32)
    running = RunningBar()
    orcs = [SeqOracle(m, running) for _ in range(n)]
    past = np.zeros(n, np.int32)
    for i in range(n):
        prompt = [int(t) for t in rng.integers(3, 320, 1 + (5 * i) % 7)]
        orcs[i].eval(prompt, 0)
        eng.eval_seq(int(seqs[i]), prompt, 0, want_logits=False)
        past[i] = len(prompt)
    for step in range(3):
        toks = rng.integers(3, 320, n).astype(np.int32)
        logits, picks = eng.decode_batch(seqs, toks, past)
        for i in range(n):
            want, tol = orcs[i].eval([int(toks[i])], int(past[i]))
            try:
                check_logits(logits[i], want, tol)
            except AssertionError as e:
                raise AssertionError(f"step {step} row {i} (block {seqs[i]}, n_past {past[i]}): {e}") from None
            assert picks[i] == int(np.flatnonzero(logits[i] == logits[i].max())[0])  # lowest index among the maxima
        past += 1
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 3. independence
def test_row_order_does_not_change_a_sequence():
    """the same four sequences in two orders, three steps: per-sequence logits bit-identical; the KV blocks the steps appended to
    are compared through the steps after them, which read them"""
    m = toy(4, 2, seed=3)
    a, b = m.engine(4), m.engine(4)
    rng = np.random.default_rng(5)
    prompts = [[int(t) for t in rng.integers(3, 320, ln)] for ln in (2, 7, 4, 9)]
    for eng in (a, b):
        for s, p in enumerate(prompts):
            eng.eval_seq(s, p, 0, want_logits=False)
    past = np.array([len(p) for p in prompts], np.int32)
    order = np.array([2, 0, 3, 1], np.int32)
    for step in range(3):
        toks = rng.integers(3, 320, 4).astype(np.int32)
        la, pa = a.decode_batch(np.arange(4, dtype=np.int32), toks, past)
        lb, pb = b.decode_batch(order, toks[order], past[order])
        for j, s in enumerate(order):
            assert np.array_equal(bits(la[s]), bits(lb[j])), (step, int(s))
            assert pa[s] == pb[j]
        past += 1
    a.close()
    b.close()


def test_the_block_holding_a_sequence_does_not_matter():
    """eval_seq on block 3 of a four-block context against eval_seq on block 0 of a fresh one-block context: a prompt, single
    steps, a batched step with other sequences around it on the first, alone on the second -- bit-identical logits"""
    m = toy(4, 2, seed=4)
    multi, single = m.engine(4), m.engine(1)
    rng = np.random.default_rng(6)
    prompt = [int(t) for t in rng.integers(3, 320, 6)]
    other = [int(t) for t in rng.integers(3, 320, 5)]
    multi.eval_seq(0, other, 0, want_logits=False)  # a neighbour in block 0
    x, y = multi.eval_seq(3, prompt, 0)[0], single.eval_seq(0, prompt, 0)[0]
    assert np.array_equal(bits(x), bits(y))
    n_past = len(prompt)
    for t in (17, 250, 3):
        x, y = multi.eval_seq(3, [t], n_past)[0], single.eval_seq(0, [t], n_past)[0]
        assert np.array_equal(bits(x), bits(y)), n_past
        n_past += 1
    # one-row batched steps: the same arithmetic wherever the block lies
    x = multi.decode_batch([3], [42], [n_past])[0][0]
    y = single.decode_batch([0], [42], [n_past])[0][0]
    assert np.array_equal(bits(x), bits(y))
    multi.close()
    single.close()


def test_sequence_zero_of_a_four_block_context_is_the_plain_eval_step():
    """ns_llama_eval / ns_llama_generate on an n_seq = 4 context: logits and picks bit-identical to an n_seq = 1 context, and the
    same ns_launch_count() per step (the first one-token step builds the decode graph: one eager pass and the captured one)"""
    m = toy(4, 4, seed=8)
    L = ns.lib()
    runs = []
    for n_seq in (1, 4):
        eng = m.engine(n_seq)
        prompt = [1, 200, 31, 77]
        outs, counts = [eng.eval(prompt, 0)[0]], []
        for pos, t in enumerate((8, 250, 19), start=len(prompt)):
            before = L.ns_launch_count()
            outs.append(eng.eval([t], pos)[0])
            counts.append(L.ns_launch_count() - before)
        gen = eng.generate(5, 7, 6)
        runs.append((outs, counts, gen))
        eng.close()
    (o1, c1, g1), (o4, c4, g4) = runs
    for x, y in zip(o1, o4):
        assert np.array_equal(bits(x), bits(y))
    assert c1 == c4 and c1[0] > 0, (c1, c4)
    assert list(g1) == list(g4)


# ------------------------------------------------------------------------------------------------------------- 4. generation
def test_generate_batch_is_the_decode_batch_loop():
    m = toy(4, 2, seed=9)
    a, b = m.engine(4), m.engine(4)
    rng = np.random.default_rng(10)
    prompts = [[int(t) for t in rng.integers(3, 320, ln)] for ln in (3, 8, 5)]
    seqs = np.array([3, 0, 2], np.int32)
    firsts = []
    for eng in (a, b):
        firsts = []
        for s, p in zip(seqs, prompts):
            firsts.append(eng.eval_seq(int(s), p, 0, want_logits=False)[1])
    past = np.array([len(p) for p in prompts], np.int32)
    n_new = 9
    gen = a.generate_batch(seqs, firsts, past, n_new)
    assert gen.shape == (3, n_new)
    toks, ref = np.array(firsts, np.int32), []
    for i in range(n_new):
        _, toks = b.decode_batch(seqs, toks, past + i, want_logits=False)
        ref.append(toks.copy())
    assert np.array_equal(gen, np.stack(ref, axis=1))
    a.close()
    b.close()


# ------------------------------------------------------------------------------------------------------------- 5. serving
def test_a_serving_loop_retires_and_admits_requests():
    """six requests on four blocks: three start, the fourth block is taken after the first chunk; after every chunk of
    generate_batch the longest-running request retires and the next one is admitted into its block at n_past 0 (the block's stale
    rows beyond the new prompt must be ignored).  The CPU graph of each request is fed the engine's picks, and every pick whose
    top-2 margin there is unambiguous must be the CPU graph's greedy pick."""
    m = toy(4, 2, seed=11, n_ctx=48)
    eng = m.engine(4)
    rng = np.random.default_rng(12)
    pending = [[int(t) for t in rng.integers(3, 320, ln)] for ln in (9, 3, 6, 4, 8, 2)]
    chunk = 4

    class Req:
        def __init__(self, rid, block, prompt):
            self.rid, self.block, self.orc, self.steps = rid, block, m.graph(), 0
            self.n_past = len(prompt)
            want = self.orc.eval(prompt, 0)
            _, self.last = eng.eval_seq(block, prompt, 0, want_logits=False)
            self.check(want, self.last)

        def check(self, want, pick):
            if not unambiguous(want):
                return 0
            assert pick == greedy(want), (self.rid, self.n_past)
            return 1

    active, next_id, checked = {}, 0, 0
    for blk in range(3):
        active[blk] = Req(next_id, blk, pending.pop(0))
        next_id += 1
    for round_ in range(6):
        blocks = sorted(active)
        reqs = [active[b] for b in blocks]
        out = eng.generate_batch(blocks, [r.last for r in reqs], [r.n_past for r in reqs], chunk)
        for r, picks in zip(reqs, out):
            t = r.last
            for j in range(chunk):
                checked += r.check(r.orc.eval([t], r.n_past + j), int(picks[j]))
                t = int(picks[j])
            r.n_past += chunk
            r.last = int(picks[-1])
            r.steps += chunk
        if round_ == 0:
            active[3] = Req(next_id, 3, pending.pop(0))
            next_id += 1
        elif pending:
            old = max(active.values(), key=lambda r: (r.steps, -r.rid))
            active[old.block] = Req(next_id, old.block, pending.pop(0))
            next_id += 1
    assert next_id == 6 and checked >= 40, (next_id, checked)
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 6. launches
def test_launch_structure_of_a_batched_step():
    """Q4_0 lm_head (Q6_K runs in tiles of up to 4 rows).  A batched step at n = 8 and at n = 3 launches the same number of
    kernels, and per layer exactly one fewer than a prompt of n tokens, whose attention is two launches (RoPE + KV append, then
    attention) where the batched step has one.  The first decode_batch of a size builds its graph: one eager pass and the
    captured one, each counted."""
    L = ns.lib()

    def counts(n_layer, n):
        eng = toy(4, 4, seed=13, n_layer=n_layer).engine(8)
        eng.eval_seq(1, [5] * 3, 0, want_logits=False)  # buffers for 8 rows exist before counting
        eng.eval_seq(0, [1] * 8, 0, want_logits=False)
        before = L.ns_launch_count()
        eng.eval_seq(2, [7] * n, 0, want_logits=False)
        prompt = L.ns_launch_count() - before
        before = L.ns_launch_count()
        eng.decode_batch(np.arange(n, dtype=np.int32), np.full(n, 9, np.int32), np.full(n, 10, np.int32), want_logits=False)
        batch = L.ns_launch_count() - before
        eng.close()
        assert batch % 2 == 0, batch
        return prompt, batch // 2

    p1_3, b1_3 = counts(1, 3)
    p2_3, b2_3 = counts(2, 3)
    p1_8, b1_8 = counts(1, 8)
    p2_8, b2_8 = counts(2, 8)
    assert b2_3 == b2_8 and b1_3 == b1_8, (b2_3, b2_8)
    assert b2_3 - b1_3 == (p2_3 - p1_3) - 1, (b2_3 - b1_3, p2_3 - p1_3)
    assert b2_8 - b1_8 == (p2_8 - p1_8) - 1, (b2_8 - b1_8, p2_8 - p1_8)


# ------------------------------------------------------------------------------------------------------------- 7. 7B shapes
def test_llama2_7b_shaped_batched_decode_matches_the_reference_engine():
    """synthetic Llama-2-7B weights as test_llama2_7b_shaped_greedy_decode_matches_the_reference_engine (Q4_0, two layers, the full
    output head): three sequences with 6-token prompts, then six batched greedy steps, each row against the reference engine
    (oracle.RefNeLlama where oracle/_ref is built, else OracleLlama) evaluating that sequence alone.  Ids are fed from the
    reference.  Bound: max(1e-2, 1.5 x the largest self-distance of the reference to its +-64 ulp jig seen so far), <= 2.5e-2."""
    rng = np.random.default_rng(77)
    m = llama2_7b_shaped(rng, n_ctx=64)
    m.draw_jig(rng)
    V = m.hp["n_vocab"]
    n, n_steps, plen = 3, 6, 6
    prompts = [[1] + [int(t) for t in rng.integers(3, V, plen - 1)] for _ in range(n)]
    # the reference, one sequence after the other (a restart at n_past 0 overwrites its cache): the fed ids and the wanted logits
    wants, selfs, feeds = [], [], []
    for which in ("ref", "jig"):
        r = m.reference(jig=which == "jig")
        for s in range(n):
            w = [r.eval(prompts[s], 0)]
            if which == "ref":
                feeds.append([greedy(w[0])])
            for j in range(n_steps):
                w.append(r.eval([feeds[s][j]], plen + j))
                if which == "ref":
                    feeds[s].append(greedy(w[-1]))
            (wants if which == "ref" else selfs).append(w)
        close(r)
    eng = m.engine(n)
    seqs = np.array([2, 0, 1], np.int32)
    for i in range(n):
        eng.eval_seq(int(seqs[i]), prompts[i], 0, want_logits=False)
    running, worst, agree, checked = RunningBar(), 0.0, 0, 0
    for j in range(n_steps):
        toks = np.array([feeds[i][j] for i in range(n)], np.int32)
        logits, picks = eng.decode_batch(seqs, toks, np.full(n, plen + j, np.int32))
        for i in range(n):
            want = wants[i][j + 1]
            tol = running(want, selfs[i][j + 1])
            s, err = scale(want), float(np.abs(logits[i] - want).max())
            assert err <= tol * s, (j, i, err / s, running.floor)
            worst = max(worst, err / s)
            if unambiguous(want, 2 * tol):
                checked += 1
                agree += int(picks[i] == greedy(want))
    print(f"7B-shape batched decode: worst |dlogit|/max|logit| {worst:.2e}; reference vs its jig {running.floor:.2e}; ids {agree}/{checked}")
    assert checked >= 6 and agree == checked, (agree, checked)
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 8. arguments
def test_argument_checks_launch_nothing():
    L = ns.lib()
    m = toy(4, 2, seed=14, n_ctx=16)
    eng = m.engine(4)
    eng.eval_seq(1, [3, 4], 0, want_logits=False)
    h = eng.h
    i32 = lambda *v: np.array(v, np.int32)
    out = np.zeros((4, 8), np.int32)
    before = L.ns_launch_count()

    def rc_of(fn, *args):
        return fn(h, *[a.ctypes.data if isinstance(a, np.ndarray) else a for a in args])

    cases = [  # (call, code, error text)
        (lambda: rc_of(L.ns_llama_decode_batch, 2, i32(0, 4), i32(1, 1), i32(0, 0), None, None), E_INVALID, "outside [0, 4)"),
        (lambda: rc_of(L.ns_llama_decode_batch, 1, i32(-1), i32(1), i32(0), None, None), E_INVALID, "outside [0, 4)"),
        (lambda: rc_of(L.ns_llama_decode_batch, 2, i32(2, 2), i32(1, 1), i32(0, 0), None, None), E_INVALID, "twice"),
        (lambda: rc_of(L.ns_llama_decode_batch, 5, i32(0, 1, 2, 3, 0), i32(1, 1, 1, 1, 1), i32(0, 0, 0, 0, 0), None, None), E_INVALID,
         "outside [1, n_seq 4]"),
        (lambda: rc_of(L.ns_llama_decode_batch, 0, i32(0), i32(1), i32(0), None, None), E_INVALID, "outside [1, n_seq 4]"),
        (lambda: rc_of(L.ns_llama_decode_batch, 1, i32(0), i32(1), i32(16), None, None), E_INVALID, "n_ctx 16"),
        (lambda: rc_of(L.ns_llama_decode_batch, 1, i32(0), i32(1), i32(-1), None, None), E_INVALID, "n_ctx 16"),
        (lambda: rc_of(L.ns_llama_decode_batch, 1, None, i32(1), i32(0), None, None), E_INVALID, "null"),
        (lambda: rc_of(L.ns_llama_decode_batch, 1, i32(0), None, i32(0), None, None), E_INVALID, "null"),
        (lambda: rc_of(L.ns_llama_decode_batch, 1, i32(0), i32(1), None, None, None), E_INVALID, "null"),
        (lambda: rc_of(L.ns_llama_generate_batch, 2, i32(0, 1), i32(1, 1), i32(10, 2), 7, out), E_INVALID, "n_ctx 16"),
        (lambda: rc_of(L.ns_llama_generate_batch, 2, i32(0, 0), i32(1, 1), i32(0, 2), 2, out), E_INVALID, "twice"),
        (lambda: rc_of(L.ns_llama_generate_batch, 1, i32(0), i32(1), i32(0), 2, None), E_INVALID, "null"),
        (lambda: rc_of(L.ns_llama_generate_batch, 1, i32(0), i32(1), i32(0), 0, out), E_INVALID, "steps"),
        (lambda: rc_of(L.ns_llama_eval_seq, 4, i32(1), 1, 0, None, None), E_INVALID, "outside [0, 4)"),
        (lambda: rc_of(L.ns_llama_eval_seq, 1, i32(1), 1, 16, None, None), E_INVALID, "n_ctx"),
        (lambda: rc_of(L.ns_llama_set_sequences, 0), E_INVALID, "outside [1, 32]"),
        (lambda: rc_of(L.ns_llama_set_sequences, 33), E_INVALID, "outside [1, 32]"),
        (lambda: rc_of(L.ns_llama_set_streaming, 4), E_UNSUPPORTED, "sequences"),
        (lambda: L.ns_llama_decode_batch(None, 1, i32(0).ctypes.data, i32(1).ctypes.data, i32(0).ctypes.data, None, None), E_INVALID, "null"),
    ]
    for j, (call, code, text) in enumerate(cases):
        rc = call()
        assert rc == code and text in ns.last_error(), (j, rc, ns.last_error())
    # the one-layer attention entry: the same row rules, then the head size
    q = torch.zeros(64, device="cuda")
    for args, code, text in (((2, 2, i32(0, 0), i32(0, 0), 8, 64), E_INVALID, "twice"),
                             ((2, 1, i32(2), i32(0), 8, 64), E_INVALID, "outside [0, 2)"),
                             ((2, 1, i32(0), i32(64), 8, 64), E_INVALID, "n_ctx 64"),
                             ((2, 3, i32(0, 1, 0), i32(0, 0, 0), 8, 64), E_INVALID, "outside [1, n_seq 2]"),
                             ((33, 1, i32(0), i32(0), 8, 64), E_INVALID, "invalid arguments"),
                             ((2, 1, i32(0), i32(0), 5, 64), E_UNSUPPORTED, "head size 80")):
        n_seq, n, s, p, H, n_ctx = args
        hd = 80 if H == 5 else 64
        p_ = q.data_ptr()
        rc = L.ns_llama_attention_batch(p_, p_, p_, p_, p_, n_seq, n, s.ctypes.data, p.ctypes.data, 8 if H == 5 else H, 2, hd, n_ctx,
                                        10000.0, 1.0, p_, p_, None)
        assert rc == code and text in ns.last_error(), (args, rc, ns.last_error())
    assert L.ns_launch_count() == before
    eng.close()
    # n_seq > 1 with streaming on, and head sizes the batched attention does not take
    ring = m.engine(1)
    ring.set_streaming(4)
    before = L.ns_launch_count()  # (loading weights launches kernels)
    assert L.ns_llama_set_sequences(ring.h, 2) == E_UNSUPPORTED and "streaming" in ns.last_error()
    assert L.ns_llama_decode_batch(ring.h, 1, i32(0).ctypes.data, i32(1).ctypes.data, i32(0).ctypes.data, None, None) == E_UNSUPPORTED
    ring.close()
    assert L.ns_launch_count() == before
    odd = toy(8, 4, seed=15, n_ctx=16).engine(1)  # head size 32
    before = L.ns_launch_count()
    assert L.ns_llama_set_sequences(odd.h, 2) == E_UNSUPPORTED and "head size 32" in ns.last_error()
    assert L.ns_llama_decode_batch(odd.h, 1, i32(0).ctypes.data, i32(1).ctypes.data, i32(0).ctypes.data, None, None) == E_UNSUPPORTED
    assert L.ns_llama_set_sequences(odd.h, 1) == 0  # one block is always fine
    assert L.ns_launch_count() == before
    odd.close()

"""Sampling in the eval step (ns_llama_set_sampling / ns_llama_sample, include/ns_b200.h): the reference's repetition-penalty /
top-k / top-p / temperature sampler on the device, in place of the argmax.

* ns_llama_sample against ns_sample_row_host bit for bit (picks, kept counts, ids, probabilities, generator state), on one
  generator carried across calls and twists, with -inf logits, ties and one-candidate rows in the middle of a batch;
* ns_llama_generate (also on the streaming ring past n_ctx), ns_llama_generate_batch and ns_llama_eval_batch against an eval loop
  sampled on the host with the host's own windows and generator kept in lockstep;
* modes: top_k = 1 is greedy, the same seed gives the same tokens, set_sampling(None) is greedy bit for bit, and the draws follow
  the probabilities (chi-square);
* a sampled step launches as many kernels as a greedy one, and every refused call launches nothing and keeps the mode."""
import ctypes as C

import numpy as np
import pytest
import torch

import llama_models
import neural_speed_b200 as ns

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


# ------------------------------------------------------------------------------------------------------ the entry on its own
class Dev:
    """device generator, windows and workspace for ns_llama_sample"""

    def __init__(self, seed, n_max=32, k_max=1024):
        self.mt = torch.from_numpy(ns.sample_seed_host(seed).view(np.int32)).cuda()
        self.ws = torch.zeros(ns.lib().ns_llama_sample_workspace_bytes(n_max, k_max), dtype=torch.uint8, device="cuda")

    def state(self):
        return self.mt.cpu().numpy().view(np.uint32)

    def run(self, logits, windows, s):
        n, nv = logits.shape
        k = s.top_k
        lg = torch.from_numpy(np.ascontiguousarray(logits)).cuda()
        w = torch.from_numpy(np.ascontiguousarray(windows, np.int32)).cuda() if windows.size else None
        picks = torch.zeros(n, dtype=torch.int32, device="cuda")
        kept = torch.zeros(n, dtype=torch.int32, device="cuda")
        ids = torch.full((n, k), -7, dtype=torch.int32, device="cuda")
        probs = torch.full((n, k), -7.0, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        rc = ns.sample(lg.data_ptr(), n, nv, w.data_ptr() if w is not None else None, windows.shape[1] if windows.size else 0, s,
                       self.mt.data_ptr(), picks.data_ptr(), kept.data_ptr(), ids.data_ptr(), probs.data_ptr(), self.ws.data_ptr())
        ns.lib().bestla_device_sync(None)
        torch.cuda.synchronize()
        return rc, picks.cpu().numpy(), kept.cpu().numpy(), ids.cpu().numpy(), probs.cpu().numpy()


def _rows(rng, n, nv, W, kind):
    lg = (rng.standard_normal((n, nv)) * rng.uniform(0.5, 4)).astype(np.float32)
    if kind % 3 == 1:  # -inf logits
        lg[rng.random((n, nv)) < 0.3] = -np.inf
    if kind % 3 == 2:  # ties, and a dominant logit in every other row (one candidate left at small top_p)
        lg = np.round(lg * 2) / 2
        lg[1::2, rng.integers(0, nv)] = 40.0
    w = rng.integers(0, nv, (n, W)).astype(np.int32)
    if W:
        w[:, : W // 4] = 0
        w[:, W // 4: W // 2] = np.argsort(-lg, axis=1)[:, : W // 2 - W // 4]  # the top logits are penalised
    return lg, w


@pytest.mark.parametrize("n_vocab", [256, 32000, 128256])
@pytest.mark.parametrize("top_k", [1, 2, 40, 1024])
def test_entry_matches_host_bit_for_bit(n_vocab, top_k):
    rng = np.random.default_rng(n_vocab + top_k)
    seed = 77 + top_k
    dev, host = Dev(seed), ns.sample_seed_host(seed)
    it = 0
    for top_p in (0.3, 0.95, 1.0):
        for temp in (0.3, 0.8, 1.5):
            for pen in (1.0, 1.1, 0.8):
                n = 1 + (it * 11) % 32
                W = (0, 17, 64, 256)[it % 4]
                lg, w = _rows(rng, n, n_vocab, W, it)
                s = ns.sampling(top_k, top_p, temp, pen, W, seed)
                rc, picks, kept, ids, probs = dev.run(lg, w, s)
                assert rc == 0, ns.last_error()
                K = min(top_k, n_vocab)
                for r in range(n):
                    hp, hk, hi, hq = ns.sample_row_host(lg[r], w[r], s, host)
                    case = (top_p, temp, pen, n, r)
                    assert (picks[r], kept[r]) == (hp, hk), case
                    assert np.array_equal(ids[r, :K], hi), case
                    assert np.array_equal(probs[r, :K].view(np.uint32), hq.view(np.uint32)), case
                assert np.array_equal(dev.state(), host), (top_p, temp, pen)
                it += 1


def test_entry_single_candidate_rows_shift_later_draws():
    rng = np.random.default_rng(3)
    dev, host = Dev(9), ns.sample_seed_host(9)
    lg = rng.standard_normal((6, 1000)).astype(np.float32)
    lg[2, 5] = lg[4, 9] = 60.0  # rows 2 and 4 keep one candidate at top_p 0.5
    s = ns.sampling(40, 0.5, 1.0, 1.0, 0, 9)
    for _ in range(400):  # 2400 draws: twists inside the calls
        rc, picks, kept, _, _ = dev.run(lg, np.zeros((6, 0), np.int32), s)
        assert rc == 0
        assert kept[2] == 1 and kept[4] == 1 and picks[2] == 5 and picks[4] == 9
        for r in range(6):
            assert picks[r] == ns.sample_row_host(lg[r], np.zeros(0, np.int32), s, host)[0]
    assert np.array_equal(dev.state(), host)


def test_entry_draws_follow_the_probabilities():
    from scipy.stats import chisquare
    rng = np.random.default_rng(11)
    lg = np.tile(rng.standard_normal(500).astype(np.float32) * 2, (32, 1))
    s = ns.sampling(40, 0.95, 0.8, 1.0, 0, 5)
    dev = Dev(5)
    _, kept, ids, probs = ns.sample_row_host(lg[0], np.zeros(0, np.int32), s, ns.sample_seed_host(0))
    counts = np.zeros(kept)
    pos = {int(t): i for i, t in enumerate(ids[:kept])}
    for _ in range(625):  # 20000 draws
        rc, picks, _, _, _ = dev.run(lg, np.zeros((32, 0), np.int32), s)
        assert rc == 0
        for p in picks:
            counts[pos[int(p)]] += 1
    want = probs[:kept].astype(np.float64) / probs[:kept].astype(np.float64).sum() * counts.sum()
    assert chisquare(counts, want).pvalue > 1e-4


def test_entry_refusals_launch_nothing():
    L = ns.lib()
    dev = Dev(1)
    lg = torch.zeros(2, 100, device="cuda")
    out = torch.zeros(2, dtype=torch.int32, device="cuda")
    good = ns.sampling(40, 0.9, 0.8, 1.1, 0, 1)
    bad = [(dict(top_k=0), E_INVALID), (dict(top_p=0.0), E_INVALID), (dict(top_p=1.01), E_INVALID), (dict(temperature=0.0), E_INVALID),
           (dict(temperature=float("nan")), E_INVALID), (dict(repeat_penalty=0.0), E_INVALID),
           (dict(repeat_penalty=float("inf")), E_INVALID), (dict(repeat_last_n=-1), E_INVALID), (dict(repeat_last_n=300), E_INVALID),
           (dict(top_k=1025), E_UNSUPPORTED)]
    for kw, code in bad:
        s = ns.sampling(**{**dict(top_k=40, top_p=0.9, temperature=0.8, repeat_penalty=1.1, repeat_last_n=0, seed=1), **kw})
        before = L.ns_launch_count()
        assert ns.sample(lg.data_ptr(), 2, 100, None, 0, s, dev.mt.data_ptr(), out.data_ptr(), None, None, None, dev.ws.data_ptr()) == code
        assert L.ns_launch_count() == before
    for n, nv, nw in [(0, 100, 0), (33, 100, 0), (2, 0, 0), (2, 100, 257), (2, 100, 4)]:  # the last: windows missing
        before = L.ns_launch_count()
        assert ns.sample(lg.data_ptr(), n, nv, None, nw, good, dev.mt.data_ptr(), out.data_ptr(), None, None, None,
                         dev.ws.data_ptr()) == E_INVALID
        assert L.ns_launch_count() == before


# --------------------------------------------------------------------------------------------------------------- engine
@pytest.fixture(scope="module")
def toy():
    """the toy Llama with GQA (4 heads on 2, head size 64)"""
    return llama_models.toy(4, 2, n_ctx=160)


SAMPLE = dict(top_k=40, top_p=0.95, temperature=0.8, repeat_penalty=1.1, repeat_last_n=64)


class HostSeq:
    """a sequence's history as the reference keeps it: n_ctx zeros, then every evaluated token"""

    def __init__(self, n_ctx, W):
        self.h, self.W = [0] * n_ctx, W

    def push(self, toks):
        self.h += [int(t) for t in toks]

    def window(self):
        return np.array(self.h[len(self.h) - self.W:] if self.W else [], np.int32)


def _generate_vs_eval_loop(eng, n_ctx, prompt, steps, seed):
    s = ns.sampling(seed=seed, **SAMPLE)
    W = min(SAMPLE["repeat_last_n"], n_ctx)
    eng.set_sampling(seed=seed, **SAMPLE)
    _, first = eng.eval(prompt, 0, want_logits=False)
    gen = eng.generate(first, len(prompt), steps)
    # the same run as an eval loop, every pick drawn again on the host from the returned logits
    eng.set_sampling(seed=seed, **SAMPLE)
    st, hs = ns.sample_seed_host(seed), HostSeq(n_ctx, W)
    hs.push(prompt)
    lg, pick = eng.eval(prompt, 0)
    assert pick == ns.sample_row_host(lg, hs.window(), s, st)[0] == first
    got, tok, n_past = [], pick, len(prompt)
    for i in range(steps):
        hs.push([tok])
        lg, pick = eng.eval([tok], n_past)
        assert pick == ns.sample_row_host(lg, hs.window(), s, st)[0], i
        got.append(pick)
        tok, n_past = pick, n_past + 1
    assert np.array_equal(gen, got)
    return gen


def test_generate_matches_host_sampled_eval_loop(toy):
    eng = toy.engine()
    prompt = [1, 17, 0, 250, 17, 3, 99, 42]
    gen = _generate_vs_eval_loop(eng, toy.hp["n_ctx"], prompt, 120, seed=1234)
    assert len(set(gen.tolist())) > 10  # it samples: not one token over and over


def test_generate_on_the_streaming_ring_matches_host_sampled_eval_loop():
    eng = llama_models.toy(4, 2, seed=1, n_ctx=48).engine()
    eng.set_streaming(4)
    _generate_vs_eval_loop(eng, 48, [5, 6, 7, 8, 9, 10], 110, seed=99)


@pytest.mark.parametrize("n", [1, 3, 8])
def test_generate_batch_matches_host_sampled_decode_loop(toy, n):
    seqs = [5, 0, 3, 7, 1, 6, 2, 4][:n]
    prompts = [[(13 * i + j) % 320 for j in range(3 + i)] for i in range(n)]
    steps, seed = 70, 2024 + n
    s = ns.sampling(seed=seed, **SAMPLE)
    eng = toy.engine(8)

    def start():
        eng.set_sampling(seed=seed, **SAMPLE)
        return [eng.eval_seq(sq, p, 0) for sq, p in zip(seqs, prompts)]

    firsts = [p for _, p in start()]
    past = [len(p) for p in prompts]
    gen = eng.generate_batch(seqs, firsts, past, steps)
    outs = start()
    st = ns.sample_seed_host(seed)
    hs = [HostSeq(toy.hp["n_ctx"], 64) for _ in range(n)]
    toks = []
    for i, (lg, pick) in enumerate(outs):
        hs[i].push(prompts[i])
        assert pick == ns.sample_row_host(lg, hs[i].window(), s, st)[0] == firsts[i]
        toks.append(pick)
    past = [len(p) for p in prompts]
    for step in range(steps):
        for i in range(n):
            hs[i].push([toks[i]])
        lg, picks = eng.decode_batch(seqs, toks, past)
        for i in range(n):  # caller row order: the reference's bs order
            assert picks[i] == ns.sample_row_host(lg[i], hs[i].window(), s, st)[0], (step, i)
        assert np.array_equal(picks, gen[:, step])
        toks, past = list(picks), [p + 1 for p in past]


def test_eval_batch_draws_in_caller_order(toy):
    eng = toy.engine(4)
    s = ns.sampling(seed=8, **{**SAMPLE, "top_p": 1.0})
    segs = [(2, [9, 8, 7, 6, 5]), (0, [4]), (3, [1, 2, 3]), (1, [11])]  # internal order: seq 0, seq 1, seq 2, seq 3
    eng.set_sampling(seed=8, **{**SAMPLE, "top_p": 1.0})
    lg, picks = eng.eval_batch([q for q, _ in segs], [t for _, t in segs], [0] * 4)
    st = ns.sample_seed_host(8)
    for i, (_, t) in enumerate(segs):
        hs = HostSeq(toy.hp["n_ctx"], 64)
        hs.push(t)
        assert picks[i] == ns.sample_row_host(lg[i], hs.window(), s, st)[0], i


def test_top_k_one_is_greedy_and_null_returns_to_greedy(toy):
    prompt = [3, 1, 4, 1, 5]
    ref = toy.engine()
    _, first = ref.eval(prompt, 0, want_logits=False)
    greedy = ref.generate(first, len(prompt), 40)
    eng = toy.engine()
    eng.set_sampling(top_k=1, top_p=0.95, temperature=0.8, repeat_penalty=1.0, repeat_last_n=64, seed=3)
    _, f1 = eng.eval(prompt, 0, want_logits=False)
    assert f1 == first
    assert np.array_equal(eng.generate(f1, len(prompt), 40), greedy)
    eng.set_sampling(seed=3, **SAMPLE)
    _, f2 = eng.eval(prompt, 0, want_logits=False)
    a = eng.generate(f2, len(prompt), 40)
    eng.set_sampling(seed=3, **SAMPLE)
    _, f3 = eng.eval(prompt, 0, want_logits=False)
    assert f3 == f2 and np.array_equal(eng.generate(f3, len(prompt), 40), a)  # same seed, same tokens
    assert not np.array_equal(a, greedy)
    eng.set_sampling(None)
    lg0, g1 = eng.eval(prompt, 0)
    lr, _ = ref.eval(prompt, 0)
    assert g1 == first and np.array_equal(lg0, lr)
    assert np.array_equal(eng.generate(g1, len(prompt), 40), greedy)


def _launches(fn):
    L = ns.lib()
    before = L.ns_launch_count()
    fn()
    return L.ns_launch_count() - before


def test_sampled_steps_launch_as_many_kernels_as_greedy(toy):
    counts = {}
    for mode in ("greedy", "sampled"):
        eng = toy.engine(4)
        if mode == "sampled":
            eng.set_sampling(seed=1, **SAMPLE)
        c = [_launches(lambda: eng.eval_seq(0, [1, 2, 3, 4], 0)),
             _launches(lambda: eng.eval([5], 4)),                       # decode graph: eager pass + capture
             _launches(lambda: eng.decode_batch([0, 2], [6, 7], [5, 0])),
             _launches(lambda: eng.eval_batch([1, 3], [[8], [9, 10, 11]], [0, 0]))]
        counts[mode] = c
    assert counts["greedy"] == counts["sampled"], counts


def test_set_sampling_refusals_keep_the_mode(toy):
    L = ns.lib()
    eng = toy.engine()
    prompt = [7, 7, 8]
    _, first = eng.eval(prompt, 0, want_logits=False)
    greedy = eng.generate(first, len(prompt), 20)
    for kw, code in [(dict(top_k=0), E_INVALID), (dict(top_p=0.0), E_INVALID), (dict(top_p=2.0), E_INVALID),
                     (dict(temperature=-1.0), E_INVALID), (dict(temperature=float("inf")), E_INVALID),
                     (dict(repeat_penalty=0.0), E_INVALID), (dict(repeat_penalty=float("nan")), E_INVALID),
                     (dict(repeat_last_n=-1), E_INVALID), (dict(repeat_last_n=257), E_INVALID), (dict(top_k=1025), E_UNSUPPORTED)]:
        s = ns.sampling(**{**SAMPLE, "seed": 4, **kw})
        before = L.ns_launch_count()
        assert L.ns_llama_set_sampling(eng.h, C.byref(s)) == code, kw
        assert L.ns_launch_count() == before
    _, f = eng.eval(prompt, 0, want_logits=False)
    assert f == first and np.array_equal(eng.generate(f, len(prompt), 20), greedy)  # still greedy
    eng.set_sampling(seed=4, **SAMPLE)
    _, f = eng.eval(prompt, 0, want_logits=False)
    a = eng.generate(f, len(prompt), 20)
    s = ns.sampling(**{**SAMPLE, "seed": 4, "top_k": 2000})
    assert L.ns_llama_set_sampling(eng.h, C.byref(s)) == E_UNSUPPORTED
    # still sampling with the old parameters: a restart at n_past 0 continues the old generator, so compare against a fresh run
    e2 = toy.engine()
    e2.set_sampling(seed=4, **SAMPLE)
    _, g = e2.eval(prompt, 0, want_logits=False)
    assert np.array_equal(e2.generate(g, len(prompt), 20), a)
    _, f2 = eng.eval(prompt, 0, want_logits=False)
    _, g2 = e2.eval(prompt, 0, want_logits=False)
    assert f2 == g2

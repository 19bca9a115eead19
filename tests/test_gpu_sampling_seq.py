"""Per-sequence sampling in the eval step (ns_llama_set_sequence_sampling / ns_llama_sample_rows, include/ns_b200.h): each KV
block its own parameters, generator and window, changed between steps without a recapture.

* ns_llama_sample_rows against ns_sample_row_host row by row, bit for bit (picks, kept counts, ids, probabilities, every
  generator), over consecutive calls; rows are independent of each other and of their order; refusals write nothing;
* generate_batch, eval_batch and eval / generate (also on the streaming ring) against a loop sampled on the host with each block's
  own window and generator; a greedy block picks the argmax of its logits;
* determinism per request, greedy equivalence, no recapture on a config change, and the way out of the mode."""
import ctypes as C

import numpy as np
import pytest
import torch

import llama_models
import neural_speed_b200 as ns

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4
N_WINDOW = 256


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def _launches(fn):
    L = ns.lib()
    before = L.ns_launch_count()
    fn()
    return L.ns_launch_count() - before


# ------------------------------------------------------------------------------------------------------ the entry on its own
class Rows:
    """device generators [n_max][625] and a workspace for ns_llama_sample_rows"""

    def __init__(self, seeds, k_max=1024):
        self.mt = torch.from_numpy(np.stack([ns.sample_seed_host(s) for s in seeds]).view(np.int32)).cuda()
        self.ws = torch.zeros(ns.lib().ns_llama_sample_workspace_bytes(len(seeds), k_max), dtype=torch.uint8, device="cuda")

    def states(self):
        return self.mt.cpu().numpy().view(np.uint32).copy()

    def run(self, logits, windows, cfgs):
        n, nv = logits.shape
        k = max(s.top_k for s in cfgs)
        lg = torch.from_numpy(np.ascontiguousarray(logits)).cuda()
        w = torch.from_numpy(np.ascontiguousarray(windows, np.int32)).cuda()
        picks = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        kept = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        ids = torch.full((n, k), -7, dtype=torch.int32, device="cuda")
        probs = torch.full((n, k), -7.0, dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        rc = ns.sample_rows(lg.data_ptr(), n, nv, w.data_ptr(), windows.shape[1], cfgs, self.mt.data_ptr(), picks.data_ptr(),
                            kept.data_ptr(), ids.data_ptr(), probs.data_ptr(), self.ws.data_ptr())
        ns.lib().bestla_device_sync(None)
        torch.cuda.synchronize()
        return rc, picks.cpu().numpy(), kept.cpu().numpy(), ids.cpu().numpy(), probs.cpu().numpy()


def _logits(rng, n, nv, kind):
    lg = (rng.standard_normal((n, nv)) * rng.uniform(0.5, 4)).astype(np.float32)
    if kind == 1:  # -inf logits
        lg[rng.random((n, nv)) < 0.3] = -np.inf
    if kind == 2:  # ties, and a dominant logit in every other row (one candidate left at top_p 0.8)
        lg = np.round(lg * 2) / 2
        lg[1::2, rng.integers(0, nv)] = 40.0
    return lg


def _windows(rng, lg):
    n, nv = lg.shape
    w = rng.integers(0, nv, (n, N_WINDOW)).astype(np.int32)
    w[:, -32:] = np.argsort(-lg, axis=1)[:, :32]  # the latest tokens are top logits: the penalty moves the selection
    return w


def _configs(rng, n):
    """a mix of every top_k, top_p, temperature, penalty and window length"""
    return [ns.sampling(int(rng.choice([1, 2, 40, 1024])), float(rng.choice([0.8, 1.0])), float(rng.choice([0.3, 0.8, 1.5])),
                        float(rng.choice([1.0, 1.1, 0.8])), int(rng.choice([0, 64, 256])), 0) for _ in range(n)]


def _host_rows(lg, w, cfgs, states):
    """ns_sample_row_host on each row with its own config, window and generator (states advanced in place)"""
    out = []
    for r, s in enumerate(cfgs):
        W = min(s.repeat_last_n, w.shape[1])
        out.append(ns.sample_row_host(lg[r], w[r, w.shape[1] - W:], s, states[r]))
    return out


@pytest.mark.parametrize("n_vocab", [320, 32000, 128256])
@pytest.mark.parametrize("n", [1, 7, 32])
def test_entry_matches_host_row_by_row(n, n_vocab):
    rng = np.random.default_rng(n * 1000 + n_vocab)
    seeds = [int(x) for x in rng.integers(0, 2**32, n)]
    dev, host = Rows(seeds), np.stack([ns.sample_seed_host(s) for s in seeds])
    for call in range(3):  # consecutive calls on the same generators, the configs drawn again each time
        lg = _logits(rng, n, n_vocab, call)
        w = _windows(rng, lg)
        cfgs = _configs(rng, n)
        rc, picks, kept, ids, probs = dev.run(lg, w, cfgs)
        assert rc == 0, ns.last_error()
        for r, (hp, hk, hi, hq) in enumerate(_host_rows(lg, w, cfgs, host)):
            K = min(cfgs[r].top_k, n_vocab)
            case = (call, r, cfgs[r].top_k, cfgs[r].top_p, cfgs[r].temperature, cfgs[r].repeat_penalty, cfgs[r].repeat_last_n)
            assert (picks[r], kept[r]) == (hp, hk), case
            assert np.array_equal(ids[r, :K], hi), case
            assert np.array_equal(probs[r, :K].view(np.uint32), hq.view(np.uint32)), case
        assert np.array_equal(dev.states(), host), call


def test_entry_rows_are_independent():
    rng = np.random.default_rng(5)
    n, nv = 8, 32000
    seeds = list(range(100, 100 + n))
    lg = _logits(rng, n, nv, 0)
    w = _windows(rng, lg)
    cfgs = [ns.sampling(k, 0.95, 0.8, 1.1, 64, 0) for k in (40, 1024, 1, 2, 40, 40, 1024, 3)]
    base = Rows(seeds)
    ref = base.run(lg, w, cfgs)
    assert ref[0] == 0
    ref_mt = base.states()
    # permuting the rows together with their generators permutes every output
    perm = rng.permutation(n)
    pr = Rows([seeds[i] for i in perm])
    got = pr.run(lg[perm], w[perm], [cfgs[i] for i in perm])
    assert got[0] == 0
    for a, b in zip(got[1:], ref[1:]):  # picks, kept, ids, probs
        assert np.array_equal(a, b[perm])
    assert np.array_equal(pr.states(), ref_mt[perm])
    # another row's logits and config changed: rows 0-2 keep their outputs and generators
    lg2, cfg2 = lg.copy(), list(cfgs)
    lg2[3:] = _logits(rng, n - 3, nv, 2)
    cfg2[3:] = [ns.sampling(1024, 1.0, 1.5, 0.8, 256, 0)] * (n - 3)
    other = Rows(seeds)
    got = other.run(lg2, w, cfg2)
    assert got[0] == 0
    for r in range(3):
        assert got[1][r] == ref[1][r] and got[2][r] == ref[2][r]
        K = cfgs[r].top_k
        assert np.array_equal(got[3][r, :K], ref[3][r, :K]) and np.array_equal(got[4][r, :K], ref[4][r, :K])
    assert np.array_equal(other.states()[:3], ref_mt[:3])


def test_entry_refusals_launch_nothing_and_write_nothing():
    L = ns.lib()
    n = 4
    dev = Rows(range(n))
    lg = torch.zeros(n, 100, device="cuda")
    w = torch.zeros(n, 16, dtype=torch.int32, device="cuda")
    outs = [torch.full((n,), -7, dtype=torch.int32, device="cuda"), torch.full((n,), -7, dtype=torch.int32, device="cuda"),
            torch.full((n, 1024), -7, dtype=torch.int32, device="cuda"), torch.full((n, 1024), -7.0, device="cuda")]
    before_mt = dev.states()
    good = dict(top_k=40, top_p=0.9, temperature=0.8, repeat_penalty=1.1, repeat_last_n=0, seed=1)

    def call(cfgs, n=n, nv=100, nw=16, win=True):
        torch.cuda.synchronize()
        c0 = L.ns_launch_count()
        rc = ns.sample_rows(lg.data_ptr(), n, nv, w.data_ptr() if win else None, nw, cfgs, dev.mt.data_ptr(),
                            *(o.data_ptr() for o in outs), dev.ws.data_ptr())
        torch.cuda.synchronize()
        assert L.ns_launch_count() == c0
        return rc

    bad = [(dict(top_k=0), E_INVALID), (dict(top_p=0.0), E_INVALID), (dict(temperature=float("nan")), E_INVALID),
           (dict(repeat_penalty=0.0), E_INVALID), (dict(repeat_last_n=257), E_INVALID), (dict(top_k=1025), E_UNSUPPORTED)]
    for kw, code in bad:
        cfgs = [ns.sampling(**good)] * n
        cfgs[2] = ns.sampling(**{**good, **kw})  # one refused row refuses the call
        assert call(cfgs) == code, kw
    cfgs = [ns.sampling(**good)] * n
    assert call(cfgs, n=0) == E_INVALID
    assert call([ns.sampling(**good)] * 33, n=33) == E_INVALID
    assert call(cfgs, nv=0) == E_INVALID
    assert call(cfgs, nw=257) == E_INVALID
    assert call(cfgs, win=False) == E_INVALID  # windows missing
    assert np.array_equal(dev.states(), before_mt)
    for o in outs:
        assert bool((o == -7).all())


# --------------------------------------------------------------------------------------------------------------- engine
@pytest.fixture(scope="module")
def toy():
    """the toy Llama with GQA (4 heads on 2, head size 64)"""
    return llama_models.toy(4, 2, n_ctx=160)


GREEDY = None
A = dict(top_k=40, top_p=0.95, temperature=0.8, repeat_penalty=1.1, repeat_last_n=64)
WIDE = dict(top_k=1024, top_p=1.0, temperature=1.3, repeat_penalty=1.0, repeat_last_n=64)
PEN = dict(top_k=40, top_p=0.9, temperature=0.9, repeat_penalty=1.5, repeat_last_n=16)
# block configs (kwargs with a seed, or GREEDY): one greedy, two equal parameters with different seeds, top_k 1024 / top_p 1,
# a strong penalty on a window of 16
MIX = [dict(PEN, seed=7), GREEDY, dict(A, seed=11), dict(A, seed=12), dict(WIDE, seed=13), dict(A, seed=14), GREEDY,
       dict(PEN, seed=15)]


class HostBlock:
    """a block as the sampler keeps it: its config, generator and history (n_ctx zeros, then every token evaluated since the
    config was set or the block restarted at n_past 0)"""

    def __init__(self, n_ctx, cfg):
        self.n_ctx, self.cfg = n_ctx, cfg
        self.s = ns.sampling(**cfg) if cfg is not None else None
        self.st = ns.sample_seed_host(cfg["seed"]) if cfg is not None else None
        self.restart()

    def restart(self):
        self.h = [0] * self.n_ctx

    def push(self, toks):
        self.h += [int(t) for t in toks]

    def pick(self, logits):
        if self.s is None:
            return int(np.argmax(logits))  # the argmax, lowest id on ties
        W = min(self.s.repeat_last_n, self.n_ctx)
        return ns.sample_row_host(logits, np.array(self.h[len(self.h) - W:] if W else [], np.int32), self.s, self.st)[0]


def _configure(eng, seqs, cfgs):
    for sq, cfg in zip(seqs, cfgs):
        eng.set_sequence_sampling(sq, **(cfg if cfg is not None else dict(top_k=None)))


def _prompts(n):
    return [[(13 * i + j) % 320 for j in range(3 + i)] for i in range(n)]


@pytest.mark.parametrize("n", [1, 3, 8])
def test_generate_batch_matches_host_decode_loop(toy, n):
    seqs = [5, 0, 3, 7, 1, 6, 2, 4][:n]
    cfgs = MIX[:n]
    prompts = _prompts(n)
    steps = 60
    n_ctx = toy.hp["n_ctx"]
    eng = toy.engine(8)

    def start():
        _configure(eng, seqs, cfgs)
        return [eng.eval_seq(sq, p, 0) for sq, p in zip(seqs, prompts)]

    firsts = [p for _, p in start()]
    past = [len(p) for p in prompts]
    gen = eng.generate_batch(seqs, firsts, past, steps)
    outs = start()
    hb = [HostBlock(n_ctx, c) for c in cfgs]
    toks = []
    for i, (lg, pick) in enumerate(outs):
        hb[i].push(prompts[i])
        assert pick == hb[i].pick(lg) == firsts[i], i
        toks.append(pick)
    for step in range(steps):
        for i in range(n):
            hb[i].push([toks[i]])
        lg, picks = eng.decode_batch(seqs, toks, past)
        for i in range(n):
            assert picks[i] == hb[i].pick(lg[i]), (step, i, cfgs[i])
        assert np.array_equal(picks, gen[:, step]), step
        toks, past = list(picks), [p + 1 for p in past]
    if n == 8:
        assert not np.array_equal(gen[2], gen[3])  # equal parameters, different seeds


def test_eval_batch_prompts_and_decode_tokens_match_host(toy):
    n_ctx = toy.hp["n_ctx"]
    eng = toy.engine(4)
    seqs = [2, 0, 3, 1]
    cfgs = [dict(A, seed=21), dict(PEN, seed=22), GREEDY, dict(WIDE, seed=23)]
    _configure(eng, seqs, cfgs)
    hb = dict(zip(seqs, (HostBlock(n_ctx, c) for c in cfgs)))
    # prompts of every block in one pass
    segs = [[9, 8, 7, 6, 5], [4], [1, 2, 3], [11, 12]]
    past = {sq: 0 for sq in seqs}
    last = {}
    for _ in range(2):
        lg, picks = eng.eval_batch(seqs, segs, [past[sq] for sq in seqs])
        for i, sq in enumerate(seqs):
            if past[sq] == 0:
                hb[sq].restart()
            hb[sq].push(segs[i])
            assert picks[i] == hb[sq].pick(lg[i]), (sq, segs[i])
            past[sq] += len(segs[i])
            last[sq] = int(picks[i])
        # next pass: block 0 restarts with a new prompt, block 1 takes a prompt chunk, blocks 2 and 3 a decode token
        segs = [[last[2]], [30, 31, 32, 33], [last[3]], [40, 41, 42]]
        past[0] = 0


def _generate_vs_eval_loop(eng, n_ctx, prompt, steps, cfg):
    eng.set_sequence_sampling(0, **cfg)
    _, first = eng.eval(prompt, 0, want_logits=False)
    gen = eng.generate(first, len(prompt), steps)
    eng.set_sequence_sampling(0, **cfg)
    hb = HostBlock(n_ctx, cfg)
    hb.push(prompt)
    lg, pick = eng.eval(prompt, 0)
    assert pick == hb.pick(lg) == first
    got, tok, n_past = [], pick, len(prompt)
    for i in range(steps):
        hb.push([tok])
        lg, pick = eng.eval([tok], n_past)
        assert pick == hb.pick(lg), i
        got.append(pick)
        tok, n_past = pick, n_past + 1
    assert np.array_equal(gen, got)
    return gen


def test_eval_and_generate_on_block_0_match_host(toy):
    gen = _generate_vs_eval_loop(toy.engine(), toy.hp["n_ctx"], [1, 17, 0, 250, 17, 3, 99, 42], 100, dict(A, seed=1234))
    assert len(set(gen.tolist())) > 10


def test_generate_on_the_streaming_ring_matches_host():
    eng = llama_models.toy(4, 2, seed=1, n_ctx=48).engine()
    eng.set_streaming(4)
    _generate_vs_eval_loop(eng, 48, [5, 6, 7, 8, 9, 10], 110, dict(A, seed=99))


def test_requests_are_deterministic_per_block(toy):
    eng = toy.engine(8)
    prompt = [3, 1, 4, 1, 5, 9, 2, 6]
    seqs = [0, 1, 2, 3, 4, 5]

    def run(order, cfgs):
        _configure(eng, order, [cfgs[sq] for sq in order])
        firsts = [eng.eval_seq(sq, prompt, 0, want_logits=False)[1] for sq in order]
        out = eng.generate_batch(order, firsts, [len(prompt)] * len(order), 40)
        return {sq: np.concatenate([[firsts[i]], out[i]]) for i, sq in enumerate(order)}

    base = {0: dict(A, seed=5), 1: dict(A, seed=5), 2: dict(A, seed=6), 3: GREEDY, 4: dict(WIDE, seed=8), 5: dict(PEN, seed=9)}
    a = run(seqs, base)
    assert np.array_equal(a[0], a[1])        # same prompt, parameters and seed
    assert not np.array_equal(a[0], a[2])    # another seed
    # the companions change their configs and the rows come in another order (n equal): blocks 0 and 2 generate the same
    other = {**base, 1: dict(WIDE, seed=77), 3: dict(PEN, seed=3), 4: GREEDY, 5: dict(A, seed=1)}
    b = run([5, 2, 4, 0, 3, 1], other)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[2], b[2])


def test_all_greedy_blocks_equal_a_greedy_context(toy):
    seqs, prompts = [1, 0, 2], _prompts(3)
    ref = toy.engine(4)
    eng = toy.engine(4)
    eng.set_sequence_sampling(3, top_k=None)  # enters the mode: every block greedy
    outs = []
    for e in (ref, eng):
        firsts = [e.eval_seq(sq, p, 0)[1] for sq, p in zip(seqs, prompts)]
        gen = e.generate_batch(seqs, firsts, [len(p) for p in prompts], 30)
        lg, picks = e.decode_batch(seqs, gen[:, -1], [len(p) + 30 for p in prompts])
        outs.append((firsts, gen, lg, picks))
    assert outs[0][0] == outs[1][0]
    assert np.array_equal(outs[0][1], outs[1][1])
    assert np.array_equal(outs[0][2], outs[1][2]) and np.array_equal(outs[0][3], outs[1][3])


def test_config_change_applies_at_the_next_step_without_recapture(toy):
    n_ctx = toy.hp["n_ctx"]
    eng = toy.engine(4)
    seqs = [0, 1, 2]
    cfgs = [dict(A, seed=31), GREEDY, dict(PEN, seed=32)]
    prompts = _prompts(3)
    _configure(eng, seqs, cfgs)
    for sq, p in zip(seqs, prompts):  # sizes the buffers for the prompts: a later growth would drop the graphs
        eng.eval_seq(sq, p, 0, want_logits=False)
    eng.decode_batch(seqs, [1, 2, 3], [0, 0, 0])  # captures the step of 3 rows
    replay = _launches(lambda: eng.decode_batch(seqs, [1, 2, 3], [0, 0, 0]))
    _configure(eng, seqs, cfgs)  # generators reseeded, windows restarted
    hb = [HostBlock(n_ctx, c) for c in cfgs]
    toks = []
    for i, (sq, p) in enumerate(zip(seqs, prompts)):
        lg, pick = eng.eval_seq(sq, p, 0)
        hb[i].push(p)
        assert pick == hb[i].pick(lg)
        toks.append(pick)
    past = [len(p) for p in prompts]
    for step in range(24):
        if step == 8:  # block 1 starts sampling, block 0 turns greedy, block 2 changes parameters
            new = [GREEDY, dict(WIDE, seed=33), dict(A, seed=34)]
            assert _launches(lambda: _configure(eng, seqs, new)) == 0
            hb = [HostBlock(n_ctx, c) for c in new]  # every window restarts, generators reseeded
        for i in range(3):
            hb[i].push([toks[i]])
        box = {}
        count = _launches(lambda: box.update(out=eng.decode_batch(seqs, toks, past)))
        assert count == replay, step  # a plain replay: nothing recaptured
        lg, picks = box["out"]
        for i in range(3):
            assert picks[i] == hb[i].pick(lg[i]), (step, i)
        toks, past = list(picks), [p + 1 for p in past]


def test_sampled_steps_launch_as_many_kernels_as_greedy(toy):
    counts = {}
    for mode in ("greedy", "per_seq"):
        eng = toy.engine(4)
        if mode == "per_seq":
            _configure(eng, [0, 1, 2, 3], [dict(A, seed=1), dict(WIDE, seed=2), GREEDY, dict(PEN, seed=3)])
        counts[mode] = [_launches(lambda: eng.eval_seq(0, [1, 2, 3, 4], 0)),
                        _launches(lambda: eng.eval([5], 4)),                       # decode graph: eager pass + capture
                        _launches(lambda: eng.eval([6], 5)),                       # replay
                        _launches(lambda: eng.decode_batch([0, 2], [6, 7], [6, 0])),
                        _launches(lambda: eng.generate_batch([0, 2], [6, 7], [7, 1], 5)),
                        _launches(lambda: eng.eval_batch([1, 3], [[8], [9, 10, 11]], [0, 0]))]
    assert counts["greedy"] == counts["per_seq"], counts


def _run(eng, seqs, prompts, steps=20):
    """each block's prompt at n_past 0, then steps tokens of generate_batch"""
    firsts = [eng.eval_seq(sq, p, 0)[1] for sq, p in zip(seqs, prompts)]
    return eng.generate_batch(seqs, firsts, [len(p) for p in prompts], steps)


def test_leaving_and_resetting_the_mode(toy):
    seqs, prompts = [0, 1, 2], _prompts(3)
    greedy = _run(toy.engine(4), seqs, prompts)
    prompt = [7, 8, 9, 10]
    fresh = toy.engine(4)
    fresh.set_sampling(seed=3, **A)
    _, f = fresh.eval(prompt, 0, want_logits=False)
    want = fresh.generate(f, len(prompt), 40)

    eng = toy.engine(4)
    _configure(eng, seqs, [dict(A, seed=1), dict(PEN, seed=2), dict(WIDE, seed=3)])
    _run(eng, seqs, prompts)
    # set_sampling(s) leaves the mode: the context picks as one that never entered it
    eng.set_sampling(seed=3, **A)
    _, g = eng.eval(prompt, 0, want_logits=False)
    assert g == f and np.array_equal(eng.generate(g, len(prompt), 40), want)
    # set_sampling(None) after per-sequence use: greedy
    _configure(eng, seqs, [dict(A, seed=1), dict(PEN, seed=2), dict(WIDE, seed=3)])
    _run(eng, seqs, prompts)
    eng.set_sampling(None)
    assert np.array_equal(_run(eng, seqs, prompts), greedy)
    # set_sequences: every block greedy again, still in per-sequence mode (a later change recaptures nothing)
    _configure(eng, seqs, [dict(A, seed=1), dict(PEN, seed=2), dict(WIDE, seed=3)])
    _run(eng, seqs, prompts)
    eng.set_sequences(4)
    assert np.array_equal(_run(eng, seqs, prompts), greedy)
    eng.set_sequence_sampling(1, **A, seed=5)
    firsts = [eng.eval_seq(sq, p, 0)[1] for sq, p in zip(seqs, prompts)]
    assert _launches(lambda: eng.generate_batch(seqs, firsts, [len(p) for p in prompts], 20)) == 0


def test_scoring_and_beams_refused_while_a_block_samples(toy):
    L = ns.lib()
    eng = toy.engine(4)
    eng.set_sequence_sampling(2, **A, seed=1)
    for fn, what in [(lambda: eng.eval_all([0], [[1, 2, 3]], [0]), "eval_all"), (lambda: eng.beam_search([[1, 2]], 2, 3), "beam")]:
        before = L.ns_launch_count()
        with pytest.raises(RuntimeError, match="sampling"):
            fn()
        assert L.ns_launch_count() == before, what
    eng.set_sequence_sampling(2, top_k=None)  # every block greedy: both run
    _, am, _ = eng.eval_all([0], [[1, 2, 3]], [0])
    assert len(am[0]) == 3
    assert len(eng.beam_search([[1, 2]], 2, 3)) == 1


def test_set_sequence_sampling_refusals_change_nothing(toy):
    L = ns.lib()
    seqs, prompts = [0, 1], _prompts(2)
    eng = toy.engine(2)
    greedy = _run(eng, seqs, prompts)
    good = dict(A, seed=4)
    bad = [(dict(top_k=0), E_INVALID), (dict(top_p=0.0), E_INVALID), (dict(top_p=2.0), E_INVALID),
           (dict(temperature=-1.0), E_INVALID), (dict(repeat_penalty=float("nan")), E_INVALID),
           (dict(repeat_last_n=-1), E_INVALID), (dict(repeat_last_n=257), E_INVALID), (dict(top_k=1025), E_UNSUPPORTED)]

    def refuse():
        for seq in (-1, 2):
            assert L.ns_llama_set_sequence_sampling(eng.h, seq, C.byref(ns.sampling(**good))) == E_INVALID
        assert L.ns_llama_set_sequence_sampling(eng.h, 2, None) == E_INVALID
        for kw, code in bad:
            assert L.ns_llama_set_sequence_sampling(eng.h, 1, C.byref(ns.sampling(**{**good, **kw}))) == code, kw

    # outside the mode: still greedy, and the captured graphs were kept (not entering the mode)
    assert _launches(refuse) == 0
    firsts = [eng.eval_seq(sq, p, 0)[1] for sq, p in zip(seqs, prompts)]
    assert _launches(lambda: eng.generate_batch(seqs, firsts, [len(p) for p in prompts], 20)) == 0
    assert np.array_equal(_run(eng, seqs, prompts), greedy)
    # inside the mode: block 1 keeps its config and generator
    ref = toy.engine(2)
    for e in (eng, ref):
        e.set_sequence_sampling(1, **good)
    refuse()
    assert np.array_equal(_run(eng, seqs, prompts, 30), _run(ref, seqs, prompts, 30))

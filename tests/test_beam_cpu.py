"""Beam search without a device: the library's flow (ns_beam_search_host, include/ns_b200.h) against the C++ restatement of the
reference's beam_search_flow (oracle/beam_search.cpp), which keeps the reference's structures and calls std::make_heap / pop_heap /
push_heap / sort / max_element where the reference does.

1. With the library's per-row arithmetic (ns_beam_candidates_row_host) the two agree bit for bit -- tokens, lengths and scores --
   over num_beams 2 / 3 / 4 / 8, 1-4 requests with different prompt lengths, min_new_tokens 0 / 3, length_penalty -1 / 0 / 0.5 / 1
   / 2, early stopping both ways and max_new_tokens from 1 up.  The model is synthetic: each row's logits are a hash of its token
   history, with an EOS bias that fills the hypotheses and makes early stopping fire, and every other run rounds the logits to a
   coarse grid so that equal scores exercise the tie rules.
2. With the reference's arithmetic (glibc expf / logf, a sequential sum) the oracle's outputs differ from the library's only
   where a score moves by an ulp across a near tie: the rate over a few hundred runs is reported and bounded.
3. The row arithmetic against float64 log_softmax within a bound derived from it, and the library's log within 1 ulp of glibc's
   logf on every float in (0, 1], where the scores' probabilities lie."""
import ctypes as C
import math
import os
import subprocess
import tempfile
import zlib

import numpy as np
import pytest

import neural_speed_b200 as ns

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BEAM_CPP = os.path.join(ROOT, "oracle", "beam_search.cpp")
CSRC = os.path.join(ROOT, "neural_speed_b200", "csrc")
U = 2.0 ** -24
E_INVALID = -1


@pytest.fixture(scope="module")
def orc():
    """oracle/beam_search.cpp built with the host C++ compiler into a temporary directory (the tree is left as it is)"""
    tmp = tempfile.mkdtemp(prefix="ns_beam_oracle_")
    so = os.path.join(tmp, "libbeam_oracle.so")
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-ffp-contract=off", "-Wall", "-o", so, BEAM_CPP]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, " ".join(cmd) + "\n" + r.stdout + r.stderr
    L = C.CDLL(so)
    vp, i = C.c_void_p, C.c_int
    L.orc_beam_search.argtypes = [i, i, vp, vp, i, i, i, C.c_float, i, C.c_int32, ns.BEAM_LOGITS_FN, vp, vp, vp, vp, vp]
    return L


def oracle_search(L, n_vocab, prompts, logits_fn, num_beams, max_new_tokens, min_new_tokens, length_penalty, early_stopping, eos,
                  library_rows=True):
    """oracle/beam_search.cpp over the same callback as ns.beam_search_host -> [(tokens, score)]"""
    lens = np.array([len(p) for p in prompts], np.int32)
    t = np.ascontiguousarray(np.concatenate([np.asarray(p, np.int32) for p in prompts]))
    n = lens.size
    err = []

    def cb(_user, rows, req, hist, hist_len, out):
        try:
            hs = [np.ctypeslib.as_array(hist[i], (hist_len[i],)).copy() for i in range(rows)]
            lg = np.ascontiguousarray(logits_fn([req[i] for i in range(rows)], hs), np.float32)
            C.memmove(out, lg.ctypes.data, lg.nbytes)
            return 0
        except Exception as e:  # noqa: BLE001 -- reported after the call
            err.append(e)
            return -1

    fn = ns.BEAM_LOGITS_FN(cb)
    row = C.cast(ns.lib().ns_beam_candidates_row_host, C.c_void_p).value if library_rows else None
    out = np.zeros((n, max_new_tokens), np.int32)
    out_len = np.zeros(n, np.int32)
    score = np.zeros(n, np.float32)
    rc = L.orc_beam_search(n_vocab, n, lens.ctypes.data, t.ctypes.data, num_beams, max_new_tokens, min_new_tokens, length_penalty,
                           1 if early_stopping else 0, eos, fn, None, row, out.ctypes.data, out_len.ctypes.data, score.ctypes.data)
    if err:
        raise err[0]
    assert rc == 0
    return [(out[r, :out_len[r]].copy(), float(score[r])) for r in range(n)]


class Synthetic:
    """logits of a row = a hash of its whole token history; eos_bias added to the EOS logit; grid > 0 rounds every logit to
    multiples of it (equal logits and equal scores)"""

    def __init__(self, n_vocab, eos, eos_bias=0.0, grid=0.0, salt=0):
        self.V, self.eos, self.bias, self.grid, self.salt = n_vocab, eos, eos_bias, grid, salt
        self.calls = []

    def __call__(self, req, hists):
        self.calls.append(len(hists))
        out = np.empty((len(hists), self.V), np.float32)
        for i, h in enumerate(hists):
            seed = zlib.crc32(np.asarray(h, np.int32).tobytes(), self.salt)
            x = np.random.default_rng(seed).standard_normal(self.V) * 2.0
            if self.grid:
                x = np.round(x / self.grid) * self.grid
            x[self.eos] += self.bias
            out[i] = x.astype(np.float32)
        return out


def _same(a, b):
    return len(a) == len(b) and all(np.array_equal(x[0], y[0]) and np.float32(x[1]).view(np.uint32) == np.float32(y[1]).view(np.uint32)
                                    for x, y in zip(a, b))


# ------------------------------------------------------------------------------------------------------- 1. bit for bit
@pytest.mark.parametrize("num_beams", [2, 3, 4, 8])
@pytest.mark.parametrize("min_new", [0, 3])
@pytest.mark.parametrize("early", [False, True])
def test_flow_equals_the_oracle_with_the_library_arithmetic(orc, num_beams, min_new, early):
    rng = np.random.default_rng(num_beams * 100 + min_new * 10 + early)
    V, eos = 40, 5
    runs = finished_early = hyp_eos = 0
    for lp in (-1.0, 0.0, 0.5, 1.0, 2.0):
        for n in range(1, min(4, 32 // num_beams) + 1):
            for max_new in (1, 2, int(rng.integers(3, 9)), 12):
                prompts = [rng.integers(0, V, int(rng.integers(1, 7))).tolist() for _ in range(n)]
                model = Synthetic(V, eos, eos_bias=float(rng.choice([0.0, 2.0, 4.0])), grid=float(rng.choice([0.0, 0.5])),
                                  salt=int(rng.integers(0, 2 ** 31)))
                got = ns.beam_search_host(V, 64, prompts, model, num_beams, max_new, min_new, lp, early, eos)
                calls = list(model.calls)
                want = oracle_search(orc, V, prompts, model, num_beams, max_new, min_new, lp, early, eos)
                assert _same(got, want), (lp, n, max_new, prompts, got, want)
                assert model.calls[len(calls):] == calls  # the same passes, the same rows
                runs += 1
                finished_early += len(calls) < max_new
                hyp_eos += any(len(t) < max_new for t, _ in got)
                for t, _ in got:
                    assert 1 <= len(t) <= max_new
                    if min_new:
                        assert eos not in t[1:min_new]  # masked from the second step on; the first step takes EOS as the reference
    assert hyp_eos > 0  # hypotheses closed by EOS were returned
    if early:
        assert finished_early > 0  # early stopping ended some searches before max_new_tokens
    print(f"B {num_beams} min_new {min_new} early {early}: {runs} runs equal, {finished_early} ended early, {hyp_eos} with EOS")


def test_first_step_takes_eos_whatever_min_new_tokens_is(orc):
    """the reference's first step reads min_new_tokens from the inputs Model::beam_generate builds without a gen_conf, so 0: EOS is
    never masked there.  After every prompt EOS is by far the best token; with length_penalty 0 the one-step search returns the
    beam [EOS] (score / 0 ^ 0 = score), and longer searches carry that beam on, equal to the oracle"""
    V, eos = 40, 5

    class FirstEos(Synthetic):
        def __init__(self, prompts):
            super().__init__(V, eos, salt=3)
            self.prompts = {tuple(p) for p in prompts}

        def __call__(self, req, hists):
            out = super().__call__(req, hists)
            for i, h in enumerate(hists):
                if tuple(int(t) for t in h) in self.prompts:
                    out[i, eos] = 40.0
            return out

    prompts = [[1, 2, 3], [4, 5]]
    for min_new in (0, 1, 3):
        got = ns.beam_search_host(V, 64, prompts, FirstEos(prompts), 2, 1, min_new, 0.0, False, eos)
        assert [t.tolist() for t, _ in got] == [[eos], [eos]], (min_new, got)
        assert all(s > -1e-3 for _, s in got)
        for max_new in (2, 5):
            for lp in (0.0, 1.0):
                got = ns.beam_search_host(V, 64, prompts, FirstEos(prompts), 3, max_new, min_new, lp, False, eos)
                want = oracle_search(orc, V, prompts, FirstEos(prompts), 3, max_new, min_new, lp, False, eos)
                assert _same(got, want), (min_new, max_new, lp, got, want)
                if lp == 0.0:
                    assert all(t[0] == eos for t, _ in got)  # the EOS beam wins: its first pick cost nothing


def test_refusals():
    model = Synthetic(40, 5)
    for kw, prompts in [(dict(num_beams=1), [[1]]), (dict(num_beams=33), [[1]]), (dict(num_beams=21), [[1]]),  # 2 B > n_vocab
                        (dict(max_new_tokens=0), [[1]]), (dict(min_new_tokens=-1), [[1]]), (dict(length_penalty=math.inf), [[1]]),
                        (dict(eos_token_id=40), [[1]]), (dict(num_beams=4, max_new_tokens=60), [[1] * 5]),  # 5 + 60 - 1 > 63
                        (dict(num_beams=8), [[1]] * 5), (dict(), [[]])]:
        args = dict(num_beams=2, max_new_tokens=4, min_new_tokens=0, length_penalty=1.0, early_stopping=False, eos_token_id=5)
        args.update(kw)
        with pytest.raises(RuntimeError):
            ns.beam_search_host(40, 63, prompts, model, **args)
    assert model.calls == []
    # the context holds the prompt and every evaluated pick: the last pick is never evaluated
    assert len(ns.beam_search_host(40, 63, [[1] * 4], model, 2, 60, 0, 1.0, False, 5)) == 1


# ------------------------------------------------------------------------------------------------------- 2. the reference
def test_reference_arithmetic_differs_only_at_near_ties(orc):
    rng = np.random.default_rng(7)
    V, eos = 64, 3
    runs = differ = 0
    worst = 0.0
    for _ in range(300):
        B = int(rng.choice([2, 3, 4, 8]))
        n = int(rng.integers(1, min(4, 32 // B) + 1))
        prompts = [rng.integers(0, V, int(rng.integers(1, 7))).tolist() for _ in range(n)]
        model = Synthetic(V, eos, eos_bias=float(rng.choice([0.0, 2.0])), salt=int(rng.integers(0, 2 ** 31)))
        args = (B, int(rng.integers(1, 10)), int(rng.choice([0, 3])), float(rng.choice([-1.0, 0.0, 0.5, 1.0, 2.0])), bool(rng.integers(0, 2)),
                eos)
        ours = oracle_search(orc, V, prompts, model, *args)
        ref = oracle_search(orc, V, prompts, model, *args, library_rows=False)
        runs += 1
        if any(not np.array_equal(a[0], b[0]) for a, b in zip(ours, ref)):
            differ += 1
        else:
            worst = max(worst, max(abs(a[1] - b[1]) / max(1.0, abs(b[1])) for a, b in zip(ours, ref)))
    print(f"library vs reference arithmetic: {differ} of {runs} runs differ in tokens; worst relative score distance {worst:.2e}")
    assert differ <= runs // 50
    assert worst <= 64 * U


# ------------------------------------------------------------------------------------------------------- 3. the row
def _bound(n_vocab, lp, S):
    """as tests/test_logprob_cpu.py's: S along its chain of fp32 additions, the log, then norm = 1 / S and the product with the
    exp (one rounding each, and the exp within 2 u) before the log of a value in (0, 1]"""
    per = -(-n_vocab // 32)
    depth = -(-per // 256) + 5 + 7 + 32
    rel_S = (depth + 4) * U * 1.01
    return rel_S + 5 * U + 2 * U * abs(lp) + 1e-30


@pytest.mark.parametrize("n_vocab", [320, 32000, 128256])
@pytest.mark.parametrize("spread", [1e-2, 1.0, 30.0])
def test_row_matches_float64_log_softmax(n_vocab, spread):
    rng = np.random.default_rng(n_vocab + int(spread * 100))
    for k in (4, 17, 64):
        x = (rng.standard_normal(n_vocab) * spread).astype(np.float32)
        x[rng.integers(0, n_vocab, 3)] = -np.inf
        ids, sc = ns.beam_candidates_row_host(x, k, 0.0, False, 2)
        key = np.lexsort((np.arange(n_vocab), -x.astype(np.float64)))[:k]  # logit descending, id ascending
        assert np.array_equal(ids, key)
        x64 = x.astype(np.float64)
        m = x64.max()
        S = float(np.exp(x64 - m).sum())
        want = x64[ids] - m - math.log(S)
        for j in range(k):
            assert abs(sc[j] - want[j]) <= _bound(n_vocab, want[j], S), (j, sc[j], want[j])
        ids2, sc2 = ns.beam_candidates_row_host(x, k, -3.25, False, 2)  # the prior score is added in fp32
        assert np.array_equal(ids2, ids) and np.array_equal(sc2, (sc + np.float32(-3.25)).astype(np.float32))


def test_mask_moves_the_selection_only():
    """min_new_tokens: EOS becomes -FLT_MAX for the selection; the max and the sum stay those of the raw row (the reference takes
    them before the mask)"""
    x = np.array([0.0, 5.0, 1.0, 4.0, -1.0, 2.0], np.float32)
    ids, sc = ns.beam_candidates_row_host(x, 3, 0.0, False, 1)
    ids_m, sc_m = ns.beam_candidates_row_host(x, 3, 0.0, True, 1)
    assert ids.tolist() == [1, 3, 5] and ids_m.tolist() == [3, 5, 2]
    assert sc_m[0] == sc[1] and sc_m[1] == sc[2]
    ids_a, sc_a = ns.beam_candidates_row_host(x, 6, 0.0, True, 1)  # the whole row: EOS last, at -inf
    assert ids_a[-1] == 1 and sc_a[-1] == -np.inf
    eq = np.array([1.0, 3.0, 3.0, 0.5, 3.0], np.float32)  # equal logits: ascending id
    assert ns.beam_candidates_row_host(eq, 3, 0.0, False, 0)[0].tolist() == [1, 2, 4]


LOG_SWEEP = r"""
#include "logprob.h"
#include <stdio.h>
// every float in (0, 1]: the largest distance in ulps of ns_logf to glibc's logf, and how many inputs differ at all
int main() {
  long long worst = 0, differ = 0, n = 0;
  float at = 1.f;
  for (uint32_t u = 1; u <= ns_float_bits(1.f); ++u, ++n) {
    const float x = ns_bits_float(u);
    const long long d = (long long)ns_float_bits(-ns_logf(x)) - (long long)ns_float_bits(-logf(x));  // both >= 0 negated
    const long long a = d < 0 ? -d : d;
    differ += a != 0;
    if (a > worst) { worst = a; at = x; }
  }
  printf("%lld %lld %lld %a\n", n, worst, differ, at);
  return 0;
}
"""


def test_log_is_within_one_ulp_of_glibc_on_every_probability():
    """compiled with the host compiler into a temporary directory (no FMA contraction, as the library's host objects); the sweep
    covers every positive float up to 1, subnormals included"""
    tmp = tempfile.mkdtemp(prefix="ns_logf_unit_sweep_")
    src, exe = os.path.join(tmp, "sweep.cpp"), os.path.join(tmp, "sweep")
    with open(src, "w") as fh:
        fh.write(LOG_SWEEP)
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I", CSRC, "-o", exe, src, "-lm"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, " ".join(cmd) + "\n" + r.stdout + r.stderr
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    n, worst, differ = int(out[0]), int(out[1]), int(out[2])
    assert n == 0x3F800000
    assert worst <= 1, (worst, out[3])
    assert ns.logf_host(1.0) == 0.0 and ns.logf_host(0.0) == -np.inf
    print(f"ns_logf vs glibc logf over (0, 1]: worst {worst} ulp, {differ} of {n} inputs ({100 * differ / n:.2f} %) differ")

"""The scoring pass's stated arithmetic on the host (neural_speed_b200/csrc/logprob.h, ns_logprob_row_host in include/ns_b200.h).

- The header's log against glibc's logf on every float in [1, 2^17], the range the row's sum S takes (S >= 1: the max's own term
  is exp(0); S <= n_vocab <= 131072).  Within 1 ulp everywhere; about 3 % of those inputs differ by that ulp.
- Rows of vocab 320 / 32000 / 128256 with logit spreads 1e-3 .. 1e3 against float64 log_softmax of the same fp32 logits, within a
  bound derived from the stated arithmetic.
- Ties, -inf entries, an all -inf row, NaN and +inf rows behave as logprob.h documents."""
import math
import os
import subprocess
import tempfile

import numpy as np
import pytest

import neural_speed_b200 as ns

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "neural_speed_b200", "csrc")
U = 2.0 ** -24  # fp32 unit roundoff

LOG_SWEEP = r"""
#include "logprob.h"
#include <stdio.h>
// every float in [1, 2^17]: the largest distance in ulps of ns_logf to glibc's logf, and how many inputs differ at all
int main() {
  long long worst = 0, differ = 0, n = 0;
  float at = 1.f;
  for (uint32_t u = ns_float_bits(1.f); u <= ns_float_bits(131072.f); ++u, ++n) {
    const float x = ns_bits_float(u);
    const long long d = (long long)ns_float_bits(ns_logf(x)) - (long long)ns_float_bits(logf(x));  // both >= 0: bits order
    const long long a = d < 0 ? -d : d;
    differ += a != 0;
    if (a > worst) { worst = a; at = x; }
  }
  printf("%lld %lld %lld %a\n", n, worst, differ, at);
  return 0;
}
"""


def test_log_is_within_one_ulp_of_glibc_on_every_float_the_sum_can_take():
    """compiled with the host compiler into a temporary directory (no FMA contraction, as the library's host objects); the sweep
    covers 17 * 2^23 + 1 inputs"""
    tmp = tempfile.mkdtemp(prefix="ns_logf_sweep_")
    src, exe = os.path.join(tmp, "sweep.cpp"), os.path.join(tmp, "sweep")
    with open(src, "w") as fh:
        fh.write(LOG_SWEEP)
    cmd = ["g++", "-O2", "-std=c++17", "-ffp-contract=off", "-I", CSRC, "-o", exe, src, "-lm"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, " ".join(cmd) + "\n" + r.stdout + r.stderr
    out = subprocess.run([exe], capture_output=True, text=True, check=True).stdout.split()
    n, worst, differ = int(out[0]), int(out[1]), int(out[2])
    assert n == 17 * 2 ** 23 + 1
    assert worst <= 1, (worst, out[3])
    print(f"ns_logf vs glibc logf over [1, 2^17]: worst {worst} ulp, {differ} of {n} inputs ({100 * differ / n:.2f} %) differ")


def _log_softmax64(x, t):
    x64 = x.astype(np.float64)
    m = x64.max()
    return float(x64[t] - m - math.log(np.exp(x64 - m).sum()))


def _bound(n_vocab, lp, S):
    """|lp - exact| from the stated arithmetic: S is a sum of exps (each within 2 u of exact: our exp is within 1 ulp of glibc's)
    along a chain of at most `depth` fp32 additions (a thread's share of its slice, 5 butterfly levels, 8 warps, the 32-slice
    merge with one rescale each); log S adds 1 ulp of itself plus S's relative error; x_t - M and the final subtraction one
    rounding each."""
    per = -(-n_vocab // 32)
    depth = -(-per // 256) + 5 + 7 + 32
    rel_S = (depth + 4) * U * 1.01
    return rel_S + 2 * U * abs(math.log(S)) + 3 * U * abs(lp) + 1e-30


@pytest.mark.parametrize("n_vocab", [320, 32000, 128256])
@pytest.mark.parametrize("spread", [1e-3, 1e-1, 1.0, 10.0, 1e3])
def test_row_matches_float64_log_softmax(n_vocab, spread):
    rng = np.random.default_rng(n_vocab + int(spread * 1000))
    worst = 0.0
    for rep in range(3):
        x = (rng.standard_normal(n_vocab) * spread).astype(np.float32)
        if rep == 2:
            x[rng.integers(0, n_vocab, 5)] += np.float32(3 * spread)  # a few peaks
        x64 = x.astype(np.float64)
        S = float(np.exp(x64 - x64.max()).sum())
        for t in [int(np.argmax(x)), int(np.argmin(x)), *rng.integers(0, n_vocab, 6).tolist()]:
            lp, am = ns.logprob_row_host(x, t)
            want = _log_softmax64(x, t)
            err = abs(lp - want)
            assert err <= _bound(n_vocab, want, S), (t, lp, want, err, _bound(n_vocab, want, S))
            assert am == int(np.argmax(x))
            worst = max(worst, err / (1e-5 + 1e-6 * abs(want)))
    assert worst <= 1.0
    print(f"vocab {n_vocab} spread {spread:g}: worst |dlp| / (1e-5 + 1e-6 |lp|) = {worst:.3f}")


def test_ties_take_the_lowest_id():
    x = np.zeros(1000, np.float32)
    x[[700, 31, 500]] = 2.0
    lp, am = ns.logprob_row_host(x, 31)
    assert am == 31
    assert lp == ns.logprob_row_host(x, 700)[0] == ns.logprob_row_host(x, 500)[0]
    x = np.full(64, -0.0, np.float32)
    x[5] = 0.0  # +0 and -0 are equal logits
    assert ns.logprob_row_host(x, None)[1] == 0


def test_minus_inf_entries_and_rows():
    rng = np.random.default_rng(3)
    x = rng.standard_normal(32000).astype(np.float32)
    x[::7] = -np.inf
    lp, am = ns.logprob_row_host(x, 14)
    assert lp == -np.inf and am == int(np.argmax(x))
    lp2, _ = ns.logprob_row_host(x, 1)
    keep = np.isfinite(x)
    assert abs(lp2 - _log_softmax64(x[keep], int(np.flatnonzero(keep).tolist().index(1)))) < 1e-5
    # a row with nothing above -inf: no distribution, NaN log-prob; the argmax is the lowest id, 0
    lp, am = ns.logprob_row_host(np.full(320, -np.inf, np.float32), 7)
    assert math.isnan(lp) and am == 0


def test_nan_and_plus_inf():
    rng = np.random.default_rng(4)
    x = rng.standard_normal(320).astype(np.float32)
    y = x.copy()
    y[100] = np.nan  # one NaN: every log-prob of the row NaN, the argmax skips it
    for t in (0, 100, int(np.argmax(x))):
        assert math.isnan(ns.logprob_row_host(y, t)[0])
    assert ns.logprob_row_host(y, None)[1] == int(np.argmax(x))
    z = np.full(320, np.nan, np.float32)
    lp, am = ns.logprob_row_host(z, 3)
    assert math.isnan(lp) and am == 0  # an all-NaN row: argmax_kernel's id 0
    w = x.copy()
    w[9] = np.inf
    lp, am = ns.logprob_row_host(w, 9)
    assert math.isnan(lp) and am == 9


def test_argument_checks():
    x = np.zeros(10, np.float32)
    L = ns.lib()
    f = np.zeros(1, np.float32)
    i = np.zeros(1, np.int32)
    assert L.ns_logprob_row_host(x.ctypes.data, 10, 10, f.ctypes.data, i.ctypes.data) == -1
    assert L.ns_logprob_row_host(x.ctypes.data, 10, -1, f.ctypes.data, None) == -1
    assert L.ns_logprob_row_host(x.ctypes.data, 10, 0, None, None) == -1
    assert L.ns_logprob_row_host(x.ctypes.data, 0, 0, f.ctypes.data, None) == -1
    assert L.ns_logprob_row_host(x.ctypes.data, 10, 99, None, i.ctypes.data) == 0  # target unread without a log-prob

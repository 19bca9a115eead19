"""The sampler's stated arithmetic on the host (ns_sample_seed_host / ns_sample_row_host / ns_sample_expf_host, include/ns_b200.h)
against the C++ restatement of the reference's model_post_sample_top_k_top_p_repeat (oracle/sampling.cpp), which calls
std::partial_sort, std::mt19937 and std::discrete_distribution where the reference does.

- The generator and the draw equal std::mt19937 + std::discrete_distribution for many seeds and probability vectors, across the
  twist, and a one-candidate list consumes no output.
- A whole row equals the oracle run with the library's exp bit for bit: pick, kept count, ids, probabilities and the generator
  state after the row.
- The library's exp is within 1 ulp of glibc's expf on every finite x <= 0.
- The oracle with the library's exp against the oracle with glibc's expf (the reference): picks differ only where the draw or
  the top-p running sum lies next to a boundary the two exps move.
- Equal logits are taken in ascending id order."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import neural_speed_b200 as ns

SAMPLING_CPP = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "sampling.cpp")


@pytest.fixture(scope="module")
def orc():
    """oracle/sampling.cpp built with the host C++ compiler into a temporary directory (the tree is left as it is)"""
    tmp = tempfile.mkdtemp(prefix="ns_sampling_oracle_")
    so = os.path.join(tmp, "libsampling_oracle.so")
    cmd = ["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-fvisibility=hidden", "-ffp-contract=off", "-pthread", "-Wall", "-o", so,
           SAMPLING_CPP]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, " ".join(cmd) + "\n" + r.stdout + r.stderr
    L = C.CDLL(so)
    vp = C.c_void_p
    L.orc_mt_new.restype = vp
    L.orc_mt_new.argtypes = [C.c_uint32]
    L.orc_mt_free.restype = None
    L.orc_mt_free.argtypes = [vp]
    L.orc_mt_next.restype = C.c_uint32
    L.orc_mt_next.argtypes = [vp]
    L.orc_mt_state.restype = None
    L.orc_mt_state.argtypes = [vp, vp]
    L.orc_discrete_draw.argtypes = [vp, vp, C.c_int]
    L.orc_sample_row.argtypes = [vp, vp, C.c_int, vp, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, vp, vp, vp, vp]
    L.orc_expf_compare.restype = None
    L.orc_expf_compare.argtypes = [vp, vp, vp, vp]
    return L


def _stated_exp():
    return C.cast(ns.lib().ns_sample_expf_host, C.c_void_p).value


class Gen:
    """the oracle's std::mt19937"""

    def __init__(self, L, seed):
        self.L, self.g = L, C.c_void_p(L.orc_mt_new(seed & 0xFFFFFFFF))

    def state(self):
        out = np.zeros(625, np.uint32)
        self.L.orc_mt_state(self.g, out.ctypes.data)
        return out

    def row(self, logits, window, s, exp_fn):
        lg = np.ascontiguousarray(logits, np.float32)
        w = np.ascontiguousarray(window, np.int32)
        k = max(1, min(s.top_k, lg.size))
        ids, probs, kept = np.zeros(k, np.int32), np.zeros(k, np.float32), C.c_int(0)
        pick = self.L.orc_sample_row(self.g, lg.ctypes.data, lg.size, w.ctypes.data if w.size else None, w.size, s.top_k, s.top_p,
                                     s.temperature, s.repeat_penalty, exp_fn, C.byref(kept), ids.ctypes.data, probs.ctypes.data)
        return pick, kept.value, ids[:kept.value], probs[:kept.value]

    def __del__(self):
        self.L.orc_mt_free(self.g)


def _pen(v, pen):
    v = v.copy()
    neg = v <= 0
    v[neg] = (v[neg] * np.float32(pen)).astype(np.float32)
    v[~neg] = (v[~neg] / np.float32(pen)).astype(np.float32)
    return v


def tie_free_row(rng, n_vocab, W, pen, scale=3.0):
    """logits whose top 1025 values after the penalty are distinct, and a window with duplicates, zeros and ids of the top logits"""
    while True:
        lg = (rng.standard_normal(n_vocab) * scale).astype(np.float32)
        top = np.argsort(-lg)[:64]
        w = np.concatenate([rng.choice(top, W // 2), rng.integers(0, n_vocab, W - W // 2)]).astype(np.int32)
        w[: W // 8] = 0
        w[W // 8: W // 4] = w[W // 4: W // 4 + W // 8]  # duplicates
        rng.shuffle(w)
        v = lg.copy()
        hit = np.unique(w)
        v[hit] = _pen(lg[hit], pen)
        head = np.sort(v)[::-1][:1025]  # the selection and its order only see the top 1025 (top_k <= 1024)
        if np.unique(head).size == head.size:
            return lg, w


@pytest.mark.parametrize("size", [1, 2, 40, 1024])
@pytest.mark.parametrize("seed", [0, 5489, 0xFFFFFFFF, 123456789])
def test_draw_equals_discrete_distribution(orc, size, seed):
    rng = np.random.default_rng(seed ^ size)
    g = Gen(orc, seed)
    st = ns.sample_seed_host(seed)
    assert np.array_equal(st, g.state())
    s = ns.sampling(top_k=size, top_p=1.0, temperature=1.0, repeat_penalty=1.0, repeat_last_n=0)
    for it in range(2000):
        lg = (rng.standard_normal(size) * rng.uniform(0.1, 4)).astype(np.float32)
        if it % 7 == 3 and size > 1:
            lg[rng.integers(0, size)] = -np.inf
        before = st.copy()
        pick, kept, ids, probs = ns.sample_row_host(lg, np.zeros(0, np.int32), s, st)
        assert kept == size
        idx = orc.orc_discrete_draw(g.g, probs.ctypes.data, kept)
        assert ids[idx] == pick, (it, idx)
        if size == 1:
            assert np.array_equal(st, before)  # no table: the generator does not advance
        if it % 250 == 0 or it == 1999:
            assert np.array_equal(st, g.state()), it
    if size > 1:
        assert st[624] != 624 or size == 1  # the stream went through at least one twist


GRID = [(nv, k, p, t, r) for nv in (256, 32000, 128256) for k in (1, 2, 40, 1024) for p in (0.3, 0.95, 1.0) for t in (0.3, 0.8, 1.5)
        for r in (1.0, 1.1, 0.8)]


@pytest.mark.parametrize("n_vocab", [256, 32000, 128256])
def test_row_equals_oracle_stated_exp(orc, n_vocab):
    rng = np.random.default_rng(n_vocab)
    seed = 1000 + n_vocab
    g = Gen(orc, seed)
    st = ns.sample_seed_host(seed)
    ef = _stated_exp()
    for (nv, k, p, t, r) in GRID:
        if nv != n_vocab:
            continue
        W = int(rng.choice([0, 17, 64, 256]))
        lg, w = tie_free_row(rng, nv, W, r, scale=float(rng.choice([0.5, 3.0])))
        s = ns.sampling(top_k=k, top_p=p, temperature=t, repeat_penalty=r, repeat_last_n=W)
        pick, kept, ids, probs = ns.sample_row_host(lg, w, s, st)
        opick, okept, oids, oprobs = g.row(lg, w, s, ef)
        case = (nv, k, p, t, r, W)
        assert (pick, kept) == (opick, okept), case
        assert np.array_equal(ids[:kept], oids), case
        assert np.array_equal(probs[:kept].view(np.uint32), oprobs.view(np.uint32)), case
        assert np.all(probs[kept:] == 0), case
        assert np.array_equal(st, g.state()), case


def test_stated_expf_against_glibc(orc):
    mx, nd, nt = C.c_int(0), C.c_longlong(0), C.c_longlong(0)
    orc.orc_expf_compare(_stated_exp(), C.byref(mx), C.byref(nd), C.byref(nt))
    frac = nd.value / nt.value
    print(f"stated expf vs glibc expf over {nt.value} finite x <= 0: max {mx.value} ulp, {frac:.3%} differ")
    assert nt.value == 0x7f800000 + 1
    assert mx.value <= 1
    assert frac < 0.05


def test_stated_expf_special_values():
    assert ns.sample_expf_host(0.0) == 1.0
    assert ns.sample_expf_host(-0.0) == 1.0
    assert ns.sample_expf_host(float("-inf")) == 0.0
    assert ns.sample_expf_host(-200.0) == 0.0
    assert np.isnan(ns.sample_expf_host(float("nan")))


def test_stated_exp_against_reference_exp(orc):
    """The oracle with the library's exp against the oracle with glibc's expf, each on its own std::mt19937 of the same seed.
    Where the picks differ, the two kept lists differ in length (the top-p running sum passed top_p within 1e-5 of it) or the
    draw u fell between the two cumulative tables' values at one boundary, which lie within 1e-5 of each other."""
    rng = np.random.default_rng(7)
    ga, gb = Gen(orc, 42), Gen(orc, 42)
    ef = _stated_exp()
    rows, kept_diff, pick_diff = 600, 0, 0
    for it in range(rows):
        nv = 32000
        s = ns.sampling(top_k=int(rng.choice([40, 1024])), top_p=float(rng.choice([0.95, 0.8, 1.0])), temperature=0.8,
                        repeat_penalty=1.1, repeat_last_n=64)
        lg, w = tie_free_row(rng, nv, 64, 1.1, scale=float(rng.choice([1.0, 3.0])))
        pa, ka, ia, qa = ga.row(lg, w, s, ef)
        pb, kb, ib, qb = gb.row(lg, w, s, None)
        assert np.array_equal(ia[:min(ka, kb)], ib[:min(ka, kb)])  # the order is the exp's business only through top-p
        assert np.abs(qa[:min(ka, kb)] - qb[:min(ka, kb)]).max() < 1e-5
        if ka != kb:
            kept_diff += 1
            continue
        if pa != pb:
            pick_diff += 1
            ca, cb = np.cumsum(qa.astype(np.float64) / np.cumsum(qa.astype(np.float64))[-1]), np.cumsum(
                qb.astype(np.float64) / np.cumsum(qb.astype(np.float64))[-1])
            ja, jb = list(ia).index(pa), list(ib).index(pb)
            assert abs(ja - jb) == 1, (it, ja, jb)
            j = min(ja, jb)
            assert abs(ca[j] - cb[j]) < 1e-5, (it, ca[j], cb[j])
        assert np.array_equal(ga.state(), gb.state())
    print(f"stated exp vs glibc expf over {rows} rows: {kept_diff} top-p cut(s) and {pick_diff} pick(s) differ")
    assert kept_diff + pick_diff <= rows // 50


def test_ties_take_ascending_ids():
    lg = np.zeros(300, np.float32)
    lg[[250, 7, 120, 3]] = 5.0
    lg[[299, 0, 64]] = 4.0
    st = ns.sample_seed_host(1)
    s = ns.sampling(top_k=6, top_p=1.0, temperature=1.0, repeat_penalty=1.0, repeat_last_n=0)
    _, kept, ids, probs = ns.sample_row_host(lg, np.zeros(0, np.int32), s, st)
    assert kept == 6
    assert list(ids) == [3, 7, 120, 250, 0, 64]
    assert probs[0] == probs[3] and probs[4] == probs[5]
    # the penalty can make ties too: id 9 at 5.5 / 1.1 lands on 5.0 (in fp32) and joins the tie at its id
    lg[9] = np.float32(5.5)
    if np.float32(np.float32(5.5) / np.float32(1.1)) == np.float32(5.0):
        s = ns.sampling(top_k=5, top_p=1.0, temperature=1.0, repeat_penalty=1.1, repeat_last_n=1)
        _, _, ids, _ = ns.sample_row_host(lg, np.array([9], np.int32), s, st)
        assert list(ids) == [3, 7, 9, 120, 250]


def test_host_argument_checks():
    st = ns.sample_seed_host(0)
    lg = np.zeros(10, np.float32)
    for bad, code in [(dict(top_k=0), -1), (dict(top_p=0.0), -1), (dict(top_p=1.5), -1), (dict(temperature=0.0), -1),
                      (dict(temperature=float("inf")), -1), (dict(repeat_penalty=-1.0), -1), (dict(repeat_penalty=float("nan")), -1),
                      (dict(repeat_last_n=257), -1), (dict(repeat_last_n=-1), -1), (dict(top_k=1025), -4)]:
        s = ns.sampling(**bad)
        pick = C.c_int32(0)
        rc = ns.lib().ns_sample_row_host(lg.ctypes.data, lg.size, None, 0, C.byref(s), st.ctypes.data, C.byref(pick), None, None, None)
        assert rc == code, bad

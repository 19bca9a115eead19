"""Qwen2 in the eval step (ns_llama_set_arch(NS_LLAMA_ARCH_QWEN2)): q / k / v biases in the matmul epilogues and NeoX RoPE as the
mode-0 kernels on W_q / W_k rows in the interleaved head order P (include/ns_b200.h).

1. the context's P-order copy of a weight dequantises to exactly the row-permuted dequant of the caller's weight, for Q4_0, Q8_0,
   Q6_K, a BesTLA int4 blob and NF4, and the caller's weight is unchanged;
2. identity: a Qwen2 context with zero biases is bit-identical to a Llama context whose W_q / W_k rows were permuted on the host;
3. the engine against the Qwen2 CPU graph (tests/qwen2_models.py) under the running bar, on every pass kind and with a Q8_0 cache;
4. a Qwen2-7B-shaped model against the reference engine's qwen2 graph;
5. a Qwen2 decode step launches what the Llama step launches and replays one graph; refusals launch nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
import oracle
import qwen2_models
from llama_models import RunningBar, _moved, bar, bits, check_logits, close, distance, scale, unambiguous
from oracle.llama_model import greedy
from oracle.qwen2 import RefNeQwen2, ref_ne_qwen2

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4
ARCH_QWEN2 = 1


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


def _dequant(handle, n, k):
    out = torch.zeros((n, k), dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    assert ns.lib().ns_weight_dequant_f32(handle, C.c_void_p(out.data_ptr()), k, None) == 0, ns.last_error()
    torch.cuda.synchronize()
    ns.lib().bestla_device_sync(None)
    return out.cpu().numpy()


def _weight(fmt, rng, n, k):
    w = rng.normal(0, 0.05, (n, k)).astype(np.float32)
    if fmt == "q4_0":
        return ns.Weight.from_q4_0_host(oracle.quantize_q4_0(w), n, k)
    if fmt == "q8_0":
        return ns.Weight.from_q8_0_host(oracle.quantize_q8_0(w), n, k)
    if fmt == "q6_K":
        return ns.Weight.from_q6_K_host(oracle.quantize_q6_K(w), n, k)
    if fmt == "btla_int4":
        return ns.Weight.from_blob(ns.np_bestla_quantize(w, "int4", 128, "sym", "fp32", "int8"))
    assert fmt == "nf4"
    g = 64
    q = rng.integers(0, 16, (k, n), dtype=np.int8)
    sc = (rng.uniform(0.5, 1.5, (k // g, n)) / 16).astype(np.float16).astype(np.float32)
    return ns.Weight.from_unpacked(q, sc, None, g, ns.W_NF4, ns.S_F16, ns.COMP_F32)


@pytest.mark.parametrize("fmt", ["q4_0", "q8_0", "q6_K", "btla_int4", "nf4"])
@pytest.mark.parametrize("n_head,n_head_kv", [(4, 2), (2, 1)])
def test_interleaved_copy_is_the_row_permuted_weight(fmt, n_head, n_head_kv):
    E = 256
    hd = E // n_head
    kvd = hd * n_head_kv
    rng = np.random.default_rng(7)
    eng = ns.Llama(320, E, n_head, n_head_kv, 1, 512, 32, arch="qwen2")
    L = ns.lib()
    for tid, n in ((ns.Llama.WQ, E), (ns.Llama.WK, kvd), (ns.Llama.WQ, E)):  # WQ twice: the slot's copy is replaced
        w = _weight(fmt, rng, n, E)
        before = _dequant(w.h, n, E)
        eng.set_weight(tid, 0, w)
        cp = L.ns_llama_weight(eng.h, tid, 0)
        assert cp and cp != w.h.value
        got = _dequant(cp, n, E)
        assert np.array_equal(bits(got), bits(before[qwen2_models.row_perm(n, hd)])), fmt
        assert np.array_equal(bits(_dequant(w.h, n, E)), bits(before))  # the caller's weight is untouched
    # V is not permuted: the context runs the caller's handle
    wv = _weight(fmt, rng, kvd, E)
    eng.set_weight(ns.Llama.WV, 0, wv)
    got = L.ns_llama_weight(eng.h, ns.Llama.WV, 0)
    assert got == wv.h.value
    eng.close()


# ------------------------------------------------------------------------------------------------------------- identity
CONFIGS = [(4, 4), (4, 2), (2, 2), (2, 1)]  # MHA / GQA at head sizes 64 and 128


@pytest.mark.parametrize("n_head,n_head_kv", CONFIGS)
def test_zero_bias_qwen2_is_the_llama_step_on_interleaved_rows(n_head, n_head_kv):
    """eval (prompts of 1, 5, 12 and 40 tokens, then single tokens), generate, decode_batch and eval_batch: np.array_equal"""
    m = qwen2_models.toy(n_head, n_head_kv, seed=n_head + n_head_kv, n_ctx=96)
    q, l = m.engine(zero_bias=True), m.llama_twin()
    rng = np.random.default_rng(3)
    pos = 0
    for n in (1, 5, 12, 40):
        toks = [int(t) for t in rng.integers(0, 320, n)]
        (a, na), (b, nb) = q.eval(toks, pos), l.eval(toks, pos)
        assert np.array_equal(a, b) and na == nb, n
        pos += n
    for t in (4, 77, 300):
        (a, na), (b, nb) = q.eval([t], pos), l.eval([t], pos)
        assert np.array_equal(a, b) and na == nb
        pos += 1
    assert np.array_equal(q.generate(9, pos, 8), l.generate(9, pos, 8))
    q.close(), l.close()
    q, l = m.engine(n_seq=4, zero_bias=True), m.llama_twin(n_seq=4)
    segs = [[int(t) for t in rng.integers(0, 320, n)] for n in (7, 1, 20, 3)]
    (a, na), (b, nb) = q.eval_batch([0, 1, 2, 3], segs, [0, 0, 0, 0]), l.eval_batch([0, 1, 2, 3], segs, [0, 0, 0, 0])
    assert np.array_equal(a, b) and np.array_equal(na, nb)
    past = [7, 1, 20, 3]
    (a, na), (b, nb) = q.decode_batch([0, 1, 2, 3], [5, 6, 7, 8], past), l.decode_batch([0, 1, 2, 3], [5, 6, 7, 8], past)
    assert np.array_equal(a, b) and np.array_equal(na, nb)
    q.close(), l.close()


# ------------------------------------------------------------------------------------------------- against the CPU graph
TC_TOL = 4e-2  # passes of more than 32 rows run the bf16 wgmma GEMM, and the KV rows they leave are bf16-precise (test_gpu_llama.py)


class Checked:
    """device logits against the Qwen2 CPU graph, held to the bar on the largest distance of that graph to its jig over the whole
    test (RunningBar's floor, taken once every step has been evaluated, as tests/test_gpu_kv_q8.py does: the floor is a property
    of the model, not of one step); greedy ids where unambiguous.  tol: a fixed bar instead (TC_TOL), checked at once."""

    def __init__(self):
        self.running, self.rows = RunningBar(), []

    def __call__(self, got, want, jig_want, what="", tol=None):
        self.running(want, jig_want)
        if tol is not None:
            check_logits(got, want, tol)
        else:
            self.rows.append((distance(got, want), what, int(np.argmax(got)), want))

    def check(self):
        b = bar(self.running.floor)
        bad = [(d, w) for d, w, _, _ in self.rows if d > b]
        assert not bad, (bad[:5], b, self.running.floor)
        for _, w, pick, want in self.rows:
            if unambiguous(want, 2 * b):
                assert pick == greedy(want), w
        return max([d for d, _, _, _ in self.rows] + [0.0]), b


@pytest.mark.parametrize("n_head,n_head_kv", CONFIGS)
def test_engine_against_the_qwen2_graph(n_head, n_head_kv):
    """prompts of 1, 5, 12 and 40 tokens (GEMV, integer tensor-core and wgmma matmuls; decode, prompt and tensor-core attention),
    single steps and generate on one sequence; in exact-prefill mode every pass under the bar, else the 40-token prompt and the
    steps after it (bf16 KV rows) under TC_TOL"""
    m = qwen2_models.toy(n_head, n_head_kv, seed=10 + n_head_kv, n_ctx=128)
    chk = Checked()
    rng = np.random.default_rng(n_head_kv)
    for exact in (True, False):
        eng, orc, jig = m.engine(), m.graph(), m.graph(jig=True)
        eng.set_exact_prefill(exact)
        pos, tol = 0, None
        for n in (1, 5, 12, 40):
            toks = [int(t) for t in rng.integers(0, 320, n)]
            tol = TC_TOL if n > 32 and not exact else tol
            got, nxt = eng.eval(toks, pos)
            chk(got, orc.eval(toks, pos), jig.eval(toks, pos), f"prompt {n} exact={exact}", tol)
            pos += n
        t = 11
        for _ in range(4):
            got, nxt = eng.eval([t], pos)
            want = orc.eval([t], pos)
            chk(got, want, jig.eval([t], pos), f"step exact={exact}", tol)
            t, pos = greedy(want), pos + 1
        # generate, fed from its own picks: the graph follows them, and each pick must be the graph's where unambiguous
        gen = eng.generate(t, pos, 6)
        for g in gen:
            want = orc.eval([t], pos)
            chk.running(want, jig.eval([t], pos))
            if unambiguous(want, 2 * (tol or bar(chk.running.floor))):
                assert int(g) == greedy(want)
            t, pos = int(g), pos + 1
        eng.close()
    worst, b = chk.check()
    print(f"Qwen2 {n_head}/{n_head_kv}: worst {worst:.2e}, bar {b:.2e}, floor {chk.running.floor:.2e}")


@pytest.mark.parametrize("n_head,n_head_kv", [(4, 4), (2, 1)])
def test_batched_passes_against_the_qwen2_graph(n_head, n_head_kv):
    """decode_batch, generate_batch, a mixed eval_batch and eval_all targets on four KV blocks"""
    m = qwen2_models.toy(n_head, n_head_kv, seed=20 + n_head, n_ctx=96)
    chk = Checked()
    eng = m.engine(n_seq=4)
    orcs = [(m.graph(), m.graph(jig=True)) for _ in range(4)]
    rng = np.random.default_rng(5)
    segs = [[int(t) for t in rng.integers(0, 320, n)] for n in (6, 1, 17, 5)]  # 29 rows: integer tensor cores
    logits, nxt = eng.eval_batch([0, 1, 2, 3], segs, [0, 0, 0, 0])
    for i, s in enumerate(segs):
        chk(logits[i], orcs[i][0].eval(s, 0), orcs[i][1].eval(s, 0), f"eval_batch {i}")
    past = [len(s) for s in segs]
    toks = [3, 9, 27, 81]
    logits, nxt = eng.decode_batch([0, 1, 2, 3], toks, past)
    for i in range(4):
        chk(logits[i], orcs[i][0].eval([toks[i]], past[i]), orcs[i][1].eval([toks[i]], past[i]), f"decode_batch {i}")
    past = [p + 1 for p in past]
    first = [int(t) for t in nxt]
    out = eng.generate_batch([0, 1, 2, 3], first, past, 4)
    for i in range(4):
        t, pos = first[i], past[i]
        for g in out[i]:
            want = orcs[i][0].eval([t], pos)
            chk.running(want, orcs[i][1].eval([t], pos))
            if unambiguous(want, 2 * bar(chk.running.floor)):
                assert int(g) == greedy(want), i
            t, pos = int(g), pos + 1
    eng.close()
    # eval_all: every row's log-prob of its target and argmax, against the graph's rows
    eng = m.engine(n_seq=2)
    segs = [[int(t) for t in rng.integers(0, 320, n)] for n in (9, 14)]
    tg = [[int(t) for t in rng.integers(0, 320, len(s))] for s in segs]
    lp, am, lg = eng.eval_all([0, 1], segs, [0, 0], targets=tg, want_logits=True)
    for i, s in enumerate(segs):
        g, j = m.graph(), m.graph(jig=True)
        for r, t in enumerate(s):
            want, jw = g.eval([t], r), j.eval([t], r)
            chk(lg[i][r], want, jw, f"eval_all {i}:{r}")
            assert am[i][r] == int(np.flatnonzero(lg[i][r] == lg[i][r].max())[0]) and np.isfinite(lp[i][r])
    eng.close()
    worst, b = chk.check()
    print(f"Qwen2 batched {n_head}/{n_head_kv}: worst {worst:.2e}, bar {b:.2e}")


@pytest.mark.parametrize("n_head,n_head_kv", [(4, 4), (2, 1)])
def test_q8_0_cache_against_the_qwen2_q8_0_graph(n_head, n_head_kv):
    """a Q8_0 KV cache holds K in P order: its blocks of 32 group P-order elements, as the CPU graph quantises them"""
    m = qwen2_models.toy(n_head, n_head_kv, seed=30 + n_head, n_ctx=96)
    chk = Checked()
    eng = m.engine()
    eng.set_kv_type("q8_0")
    eng.set_exact_prefill(True)  # the 40-token prompt in pieces of 32 on the integer tensor cores: every pass under the bar
    orc, jig = m.graph_q8(), m.graph_q8(jig=True)
    rng = np.random.default_rng(9)
    pos = 0
    for n in (5, 12, 1, 1, 40, 1):
        toks = [int(t) for t in rng.integers(0, 320, n)]
        got, _ = eng.eval(toks, pos)
        chk(got, orc.eval(toks, pos), jig.eval(toks, pos), f"q8_0 {n}")
        pos += n
    eng.close()
    worst, b = chk.check()
    print(f"Qwen2 Q8_0 cache {n_head}/{n_head_kv}: worst {worst:.2e}, bar {b:.2e}")


# ------------------------------------------------------------------------------------------------------------ real shapes
def test_qwen2_7b_shaped_against_the_reference_engine():
    """Qwen2-7B's shapes (n_embd 3584, 28 heads over 4 KV heads of 128, n_ff 18944, vocab 151936; two Q4_0 layers and the full head)
    against the reference engine's qwen2 graph (oracle.qwen2.RefNeQwen2; the CPU graph where oracle/_ref is absent): a 6-token prompt
    token by token, then 6 greedy steps fed from the reference; logits within the running bar of the reference against its jig,
    greedy ids equal where the margin exceeds it"""
    rng = np.random.default_rng(2025)
    m = qwen2_models.qwen2_7b_shaped(rng, n_ctx=32)
    m.tok_jig = _moved(m.tok, rng.integers(0, 2, m.tok.shape, dtype=np.int8).astype(np.int32) * 2 - 1)
    eng = m.engine()
    ref = m.reference()
    if ref_ne_qwen2() is None:
        ref_jig = m.graph(jig=True)
    else:
        ref_jig = RefNeQwen2(m.hp, m.tok_jig, m.out_norm, m.out_rows, m.layers)
    prompt = [int(t) for t in rng.integers(3, m.hp["n_vocab"], 6)]
    pos, t, running, agree, checked, worst = 0, prompt[0], RunningBar(), 0, 0, 0.0
    for step in range(12):
        want = ref.eval([t], pos)
        tol = running(want, ref_jig.eval([t], pos))
        got, nxt = eng.eval([t], pos)
        d = distance(got, want)
        worst = max(worst, d)
        assert d <= tol, (step, d, running.floor)
        if unambiguous(want, 2 * tol):
            checked += 1
            agree += int(nxt == greedy(want))
        pos += 1
        t = prompt[pos] if pos < len(prompt) else greedy(want)
    print(f"Qwen2-7B shape: worst {worst:.2e}, floor {running.floor:.2e}, ids {agree}/{checked}, scale {scale(want):.2f}")
    assert checked >= 4 and agree == checked, (agree, checked)
    eng.close()
    close(ref, ref_jig)


# ------------------------------------------------------------------------------------------------------ launch structure
@pytest.mark.parametrize("n_head,n_head_kv", CONFIGS)
def test_decode_step_launches_what_the_llama_step_launches(n_head, n_head_kv):
    """the first one-token step enqueues the eager pass and the captured one; later steps replay the graph and enqueue nothing"""
    m = qwen2_models.toy(n_head, n_head_kv, seed=1, n_ctx=32)
    L = ns.lib()
    counts = []
    for eng in (m.engine(), m.llama_twin()):
        eng.eval([1, 2, 3], 0)
        c = []
        for pos, t in enumerate((5, 6, 7), start=3):
            before = L.ns_launch_count()
            eng.eval([t], pos)
            c.append(L.ns_launch_count() - before)
        before = L.ns_launch_count()
        eng.generate(8, 6, 5)
        c.append(L.ns_launch_count() - before)
        counts.append(c)
        eng.close()
    assert counts[0] == counts[1], counts
    assert counts[0][0] > 0 and counts[0][1:] == [0, 0, 0], counts


def test_batched_step_launches_what_the_llama_step_launches_gqa():
    m = qwen2_models.toy(4, 2, seed=2, n_ctx=32)
    L = ns.lib()
    counts = []
    for eng in (m.engine(n_seq=3), m.llama_twin(n_seq=3)):
        eng.eval_batch([0, 1, 2], [[1, 2], [3], [4, 5, 6]], [0, 0, 0])
        c = []
        for step in range(2):
            before = L.ns_launch_count()
            eng.decode_batch([0, 1, 2], [7, 8, 9], [2 + step, 1 + step, 3 + step])
            c.append(L.ns_launch_count() - before)
        counts.append(c)
        eng.close()
    assert counts[0] == counts[1] and counts[0][1] == 0, counts


# -------------------------------------------------------------------------------------------------------------- refusals
def _create(rope_scale=1.0):
    return ns.Llama(320, 256, 4, 2, 1, 512, 32, rope_scale=rope_scale)


def test_refusals_return_their_codes_and_launch_nothing():
    L = ns.lib()
    E, kvd = 256, 128
    # rope_scale != 1
    eng = _create(rope_scale=2.0)
    assert L.ns_llama_set_arch(eng.h, ARCH_QWEN2) == E_UNSUPPORTED
    eng.close()
    # streaming, either order
    eng = _create()
    assert L.ns_llama_set_streaming(eng.h, 4) == 0
    assert L.ns_llama_set_arch(eng.h, ARCH_QWEN2) == E_UNSUPPORTED
    assert L.ns_llama_set_streaming(eng.h, -1) == 0
    assert L.ns_llama_set_arch(eng.h, ARCH_QWEN2) == 0
    assert L.ns_llama_set_streaming(eng.h, 4) == E_UNSUPPORTED
    eng.close()
    # an unknown architecture
    eng = _create()
    assert L.ns_llama_set_arch(eng.h, 7) == E_INVALID
    # biases on a Llama context
    b = np.ones(E, np.float32)
    assert L.ns_llama_set_f32(eng.h, ns.Llama.BQ, 0, b.ctypes.data_as(C.c_void_p), E) == E_INVALID
    # set_arch after a weight
    w = ns.Weight.from_q4_0_host(oracle.quantize_q4_0(np.zeros((E, E), np.float32)), E, E)
    eng.set_weight(ns.Llama.WO, 0, w)
    assert L.ns_llama_set_arch(eng.h, ARCH_QWEN2) == E_INVALID
    eng.close()
    # a Qwen2 context: a bias of the wrong size or layer, then eval with one bias missing
    m = qwen2_models.toy(4, 2, seed=3, n_ctx=32)
    eng = m.engine()
    bk = np.ones(kvd, np.float32)
    assert L.ns_llama_set_f32(eng.h, ns.Llama.BK, 0, bk.ctypes.data_as(C.c_void_p), E) == E_INVALID
    assert L.ns_llama_set_f32(eng.h, ns.Llama.BK, 5, bk.ctypes.data_as(C.c_void_p), kvd) == E_INVALID
    assert L.ns_llama_set_arch(eng.h, 0) == E_INVALID  # weights are set
    eng.close()
    eng = ns.Llama(320, 256, 4, 2, 2, 512, 32, arch="qwen2")  # every tensor but layer 1's b_v
    q4 = lambda n, k: ns.Weight.from_q4_0_host(oracle.quantize_q4_0(np.full((n, k), 0.01, np.float32)), n, k)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, m.tok)
    eng.set_f32(ns.Llama.OUT_NORM, 0, m.out_norm)
    eng.set_weight(ns.Llama.OUTPUT, 0, q4(320, E))
    for il in range(2):
        eng.set_f32(ns.Llama.ATTN_NORM, il, m.layers[0]["attn_norm"])
        eng.set_f32(ns.Llama.FFN_NORM, il, m.layers[0]["ffn_norm"])
        for tid, n, k in ((ns.Llama.WQ, E, E), (ns.Llama.WK, kvd, E), (ns.Llama.WV, kvd, E), (ns.Llama.WO, E, E),
                          (ns.Llama.W1, 512, E), (ns.Llama.W2, E, 512), (ns.Llama.W3, 512, E)):
            eng.set_weight(tid, il, q4(n, k))
        eng.set_f32(ns.Llama.BQ, il, m.layers[0]["bq"])
        eng.set_f32(ns.Llama.BK, il, m.layers[0]["bk"])
        if il == 0:
            eng.set_f32(ns.Llama.BV, il, m.layers[0]["bv"])
    toks = np.array([1, 2, 3], np.int32)
    before = L.ns_launch_count()
    assert L.ns_llama_eval(eng.h, toks.ctypes.data_as(C.c_void_p), 3, 0, None, None) == E_INVALID
    out = np.zeros(4, np.int32)
    assert L.ns_llama_generate(eng.h, 1, 0, 4, out.ctypes.data_as(C.c_void_p)) == E_INVALID
    assert L.ns_launch_count() == before
    eng.set_f32(ns.Llama.BV, 1, m.layers[0]["bv"])  # complete: it runs
    assert L.ns_llama_eval(eng.h, toks.ctypes.data_as(C.c_void_p), 3, 0, None, None) == 0
    assert L.ns_launch_count() > before
    eng.close()

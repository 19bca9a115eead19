"""Phi-3 in the eval step (ns_llama_set_arch(NS_LLAMA_ARCH_PHI3)): NeoX RoPE as the mode-0 kernels on W_q / W_k rows in the
interleaved head order P, no biases, head size 96 on the split decode and tensor-core prompt attention (include/ns_b200.h).

1. identity: a Phi-3 context is bit-identical to a Llama context whose W_q / W_k rows were permuted on the host, through eval,
   generate, decode_batch, eval_batch and beam search;
2. the engine against the Phi-3 CPU graph (tests/phi3_models.py) under the running bar, on every pass kind;
3. a Phi-3-mini-shaped model against the reference engine's graph;
4. a Phi-3 decode step launches what the Llama step launches and replays one graph;
5. a synthetic phi3 GGUF file through to device logits;
6. refusals return their codes and launch nothing."""
import ctypes as C

import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
import oracle
import phi3_models
from llama_models import RunningBar, _moved, bar, distance, scale, unambiguous
from neural_speed_b200 import gguf_loader
from oracle.llama_model import greedy
from oracle.phi3 import OraclePhi3
from test_gpu_qwen2 import TC_TOL, Checked

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4
ARCH_PHI3 = 2


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


CONFIGS = [(4, 4), (4, 2), (2, 1)]  # MHA / GQA at head size 96


# ------------------------------------------------------------------------------------------------------------- identity
@pytest.mark.parametrize("n_head,n_head_kv", CONFIGS)
def test_phi3_is_the_llama_step_on_interleaved_rows(n_head, n_head_kv):
    """eval (prompts of 1, 5, 12 and 40 tokens, then single tokens), generate, eval_batch, decode_batch and beam search:
    np.array_equal"""
    m = phi3_models.toy(n_head, n_head_kv, seed=n_head + n_head_kv, n_ctx=96)
    p, l = m.engine(), m.llama_twin()
    rng = np.random.default_rng(3)
    pos = 0
    for n in (1, 5, 12, 40):
        toks = [int(t) for t in rng.integers(0, 320, n)]
        (a, na), (b, nb) = p.eval(toks, pos), l.eval(toks, pos)
        assert np.array_equal(a, b) and na == nb, n
        pos += n
    for t in (4, 77, 300):
        (a, na), (b, nb) = p.eval([t], pos), l.eval([t], pos)
        assert np.array_equal(a, b) and na == nb
        pos += 1
    assert np.array_equal(p.generate(9, pos, 8), l.generate(9, pos, 8))
    p.close(), l.close()
    p, l = m.engine(n_seq=4), m.llama_twin(n_seq=4)
    segs = [[int(t) for t in rng.integers(0, 320, n)] for n in (7, 1, 20, 3)]
    (a, na), (b, nb) = p.eval_batch([0, 1, 2, 3], segs, [0, 0, 0, 0]), l.eval_batch([0, 1, 2, 3], segs, [0, 0, 0, 0])
    assert np.array_equal(a, b) and np.array_equal(na, nb)
    past = [7, 1, 20, 3]
    (a, na), (b, nb) = p.decode_batch([0, 1, 2, 3], [5, 6, 7, 8], past), l.decode_batch([0, 1, 2, 3], [5, 6, 7, 8], past)
    assert np.array_equal(a, b) and np.array_equal(na, nb)
    prompts = [[int(t) for t in rng.integers(0, 320, 6)], [int(t) for t in rng.integers(0, 320, 3)]]
    ba = p.beam_search(prompts, num_beams=2, max_new_tokens=5)
    bb = l.beam_search(prompts, num_beams=2, max_new_tokens=5)
    assert all(np.array_equal(x[0], y[0]) and x[1] == y[1] for x, y in zip(ba, bb)), (ba, bb)
    p.close(), l.close()


# ------------------------------------------------------------------------------------------------- against the CPU graph
@pytest.mark.parametrize("n_head,n_head_kv", CONFIGS)
def test_engine_against_the_phi3_graph(n_head, n_head_kv):
    """prompts of 1, 5, 12 and 40 tokens (GEMV, integer tensor-core and wgmma matmuls; split decode and tensor-core attention),
    single steps and generate; in exact-prefill mode every pass under the bar, else the 40-token prompt and the steps after it
    (bf16 KV rows) under TC_TOL"""
    m = phi3_models.toy(n_head, n_head_kv, seed=10 + n_head_kv, n_ctx=128)
    chk = Checked()
    rng = np.random.default_rng(n_head_kv)
    for exact in (True, False):
        eng, orc, jig = m.engine(), m.graph(), m.graph(jig=True)
        eng.set_exact_prefill(exact)
        pos, tol = 0, None
        for n in (1, 5, 12, 40):
            toks = [int(t) for t in rng.integers(0, 320, n)]
            tol = TC_TOL if n > 32 and not exact else tol
            got, _ = eng.eval(toks, pos)
            chk(got, orc.eval(toks, pos), jig.eval(toks, pos), f"prompt {n} exact={exact}", tol)
            pos += n
        t = 11
        for _ in range(4):
            got, _ = eng.eval([t], pos)
            want = orc.eval([t], pos)
            chk(got, want, jig.eval([t], pos), f"step exact={exact}", tol)
            t, pos = greedy(want), pos + 1
        gen = eng.generate(t, pos, 6)
        for g in gen:
            want = orc.eval([t], pos)
            chk.running(want, jig.eval([t], pos))
            if unambiguous(want, 2 * (tol or bar(chk.running.floor))):
                assert int(g) == greedy(want)
            t, pos = int(g), pos + 1
        eng.close()
    worst, b = chk.check()
    print(f"Phi-3 {n_head}/{n_head_kv}: worst {worst:.2e}, bar {b:.2e}, floor {chk.running.floor:.2e}")


@pytest.mark.parametrize("n_head,n_head_kv", [(4, 4), (4, 2)])
def test_batched_passes_against_the_phi3_graph(n_head, n_head_kv):
    """decode_batch, generate_batch, a mixed eval_batch and eval_all on several KV blocks (beam search runs these passes: its
    logits are held by the identity with the Llama step above)"""
    m = phi3_models.toy(n_head, n_head_kv, seed=20 + n_head, n_ctx=96)
    chk = Checked()
    eng = m.engine(n_seq=4)
    orcs = [(m.graph(), m.graph(jig=True)) for _ in range(4)]
    rng = np.random.default_rng(5)
    segs = [[int(t) for t in rng.integers(0, 320, n)] for n in (6, 1, 17, 5)]
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
    eng = m.engine(n_seq=2)
    segs = [[int(t) for t in rng.integers(0, 320, n)] for n in (9, 14)]
    tg = [[int(t) for t in rng.integers(0, 320, len(s))] for s in segs]
    lp, am, lg = eng.eval_all([0, 1], segs, [0, 0], targets=tg, want_logits=True)
    for i, s in enumerate(segs):
        g, j = m.graph(), m.graph(jig=True)
        for r, t in enumerate(s):
            chk(lg[i][r], g.eval([t], r), j.eval([t], r), f"eval_all {i}:{r}")
            assert am[i][r] == int(np.flatnonzero(lg[i][r] == lg[i][r].max())[0]) and np.isfinite(lp[i][r])
    eng.close()
    worst, b = chk.check()
    print(f"Phi-3 batched {n_head}/{n_head_kv}: worst {worst:.2e}, bar {b:.2e}")


# ------------------------------------------------------------------------------------------------------------ real shapes
def test_phi3_mini_shaped_against_the_reference_engine():
    """Phi-3-mini's shapes (n_embd 3072, 32 heads of 96, n_ff 8192, vocab 32064; two Q4_0 layers and the full head) against the
    reference engine's graph (oracle.phi3.RefNePhi3; the CPU graph where oracle/_ref is absent): a 6-token prompt token by token,
    then 6 greedy steps fed from the reference; logits within the running bar of the reference against its jig, greedy ids equal
    where the margin exceeds it"""
    rng = np.random.default_rng(2026)
    m = phi3_models.phi3_mini_shaped(rng, n_ctx=32)
    m.tok_jig = _moved(m.tok, rng.integers(0, 2, m.tok.shape, dtype=np.int8).astype(np.int32) * 2 - 1)
    eng = m.engine()
    ref = m.reference()
    ref_jig = m.reference(jig=True)
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
    print(f"Phi-3-mini shape: worst {worst:.2e}, floor {running.floor:.2e}, ids {agree}/{checked}, scale {scale(want):.2f}")
    assert checked >= 4 and agree == checked, (agree, checked)
    eng.close()
    for g in (ref, ref_jig):
        if hasattr(g, "close"):
            g.close()


# ------------------------------------------------------------------------------------------------------ launch structure
@pytest.mark.parametrize("n_head,n_head_kv", CONFIGS)
def test_decode_step_launches_what_the_llama_step_launches(n_head, n_head_kv):
    """the first one-token step enqueues the eager pass and the captured one; later steps replay the graph and enqueue nothing"""
    m = phi3_models.toy(n_head, n_head_kv, seed=1, n_ctx=32)
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
        before = L.ns_launch_count()
        eng.eval([1, 2, 3, 4, 5, 6, 7, 8, 9], 11)  # a prompt pass: rope_kv_kernel + attn_mma_kernel per layer, as Llama's
        c.append(L.ns_launch_count() - before)
        counts.append(c)
        eng.close()
    assert counts[0] == counts[1], counts
    assert counts[0][0] > 0 and counts[0][1:4] == [0, 0, 0], counts


def test_batched_step_launches_what_the_llama_step_launches_gqa():
    m = phi3_models.toy(4, 2, seed=2, n_ctx=32)
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


# ------------------------------------------------------------------------------------------------------------- file
def test_phi3_gguf_file_to_device_logits(tmp_path):
    """a synthetic phi3 GGUF (fused attn_qkv and gate / up) through gguf_loader.parse and load_into_engine: a Phi-3 context whose
    logits are within the running bar of the CPU graph on the parsed tensors"""
    pytest.importorskip("gguf")
    import test_phi3_cpu
    path = str(tmp_path / "phi3.gguf")
    test_phi3_cpu._write(path, n_head_kv=4)
    model = gguf_loader.parse(path)
    assert model.arch == "phi3"
    eng = gguf_loader.load_into_engine(model)
    assert eng.arch == "phi3"
    layers = [{k: v[1] if isinstance(v, tuple) else v for k, v in L.items()} for L in model.layers]
    orc = OraclePhi3(model.hparams, model.tok_embd, model.out_norm, model.output[1], layers)
    signs = (np.random.default_rng(99).integers(0, 2, model.tok_embd.shape) * 2 - 1).astype(np.int32)
    jig = OraclePhi3(model.hparams, _moved(model.tok_embd, signs), model.out_norm, model.output[1], layers)
    chk = Checked()
    pos = 0
    for toks in ([1, 2, 3, 4, 5], [6], [7]):
        got, _ = eng.eval(toks, pos)
        chk(got, orc.eval(toks, pos), jig.eval(toks, pos), f"file {len(toks)}")
        pos += len(toks)
    chk.check()
    eng.close()


# -------------------------------------------------------------------------------------------------------------- refusals
def test_refusals_return_their_codes_and_launch_nothing():
    L = ns.lib()
    E = 384  # 4 heads of 96
    before = L.ns_launch_count()
    # rope_scale != 1
    eng = ns.Llama(320, E, 4, 2, 1, 512, 32, rope_scale=2.0)
    assert L.ns_llama_set_arch(eng.h, ARCH_PHI3) == E_UNSUPPORTED
    eng.close()
    # streaming, either order
    eng = ns.Llama(320, 256, 4, 2, 1, 512, 32)  # streaming needs head size 64 / 128
    assert L.ns_llama_set_streaming(eng.h, 4) == 0
    assert L.ns_llama_set_arch(eng.h, ARCH_PHI3) == E_UNSUPPORTED
    assert L.ns_llama_set_streaming(eng.h, -1) == 0
    assert L.ns_llama_set_arch(eng.h, ARCH_PHI3) == 0
    assert L.ns_llama_set_streaming(eng.h, 4) == E_UNSUPPORTED and "Phi-3" in ns.last_error()
    eng.close()
    # biases on a Phi-3 context
    eng = ns.Llama(320, E, 4, 2, 1, 512, 32, arch="phi3")
    b = np.ones(E, np.float32)
    for tid, n in ((ns.Llama.BQ, E), (ns.Llama.BK, 192), (ns.Llama.BV, 192)):
        assert L.ns_llama_set_f32(eng.h, tid, 0, b.ctypes.data_as(C.c_void_p), n) == E_INVALID
    # the Q8_0 KV cache and streaming at head size 96 stay refused
    assert L.ns_llama_set_kv_type(eng.h, 1) == E_UNSUPPORTED
    assert L.ns_llama_set_arch(eng.h, 3) == E_INVALID
    # set_arch after a weight
    w = ns.Weight.from_q4_0_host(oracle.quantize_q4_0(np.zeros((E, E), np.float32)), E, E)
    eng.set_weight(ns.Llama.WO, 0, w)
    n0 = L.ns_launch_count()
    assert L.ns_llama_set_arch(eng.h, 0) == E_INVALID and L.ns_llama_set_arch(eng.h, ARCH_PHI3) == E_INVALID
    assert L.ns_launch_count() == n0
    eng.close()
    eng = ns.Llama(320, E, 4, 2, 1, 512, 32)
    eng.set_weight(ns.Llama.WQ, 0, w)
    n0 = L.ns_launch_count()
    assert L.ns_llama_set_arch(eng.h, ARCH_PHI3) == E_INVALID
    assert L.ns_launch_count() == n0
    eng.close()
    # a Llama context at head size 96 takes several sequences now; head size 80 still does not
    eng = ns.Llama(320, E, 4, 4, 1, 512, 32)
    assert L.ns_llama_set_sequences(eng.h, 2) == 0
    eng.close()
    eng = ns.Llama(320, 320, 4, 4, 1, 512, 32)
    assert L.ns_llama_set_sequences(eng.h, 2) == E_UNSUPPORTED and "head size 80" in ns.last_error()
    eng.close()
    assert before <= L.ns_launch_count()

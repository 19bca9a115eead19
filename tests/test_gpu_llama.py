"""Device-resident Llama eval step (SURVEY §8 f.1) against the CPU restatement of the reference graph (oracle/llama_model.py).
North-star bar: logits within 1e-2, greedy token ids equal (checked wherever the oracle's top-2 margin exceeds the tolerance)."""
import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
from llama_models import RunningBar, bar, check_logits, close, distance, llama2_7b_shaped, scale, smooth, toy, unambiguous
from oracle.llama_model import greedy

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


@pytest.mark.parametrize("n_head,n_head_kv,out_fmt", [(4, 4, "q4_0"), (4, 2, "q4_0"), (4, 4, "q6_K"), (2, 2, "q4_0"), (2, 1, "q4_0"),
                                                       (8, 8, "q4_0")])
def test_token_by_token_decode_matches_the_cpu_graph(n_head, n_head_kv, out_fmt):
    """head sizes 64 and 128 take the fused rope + KV-append + attention kernel, 32 the generic one"""
    m = toy(n_head, n_head_kv, out_fmt, seed=n_head_kv)
    orc, eng = m.graph(), m.engine()
    toks = [1, 17, 300, 5, 123, 77, 9]
    for pos, t in enumerate(toks):
        want = orc.eval([t], pos)
        got, nxt = eng.eval([t], pos)
        check_logits(got, want)
        assert nxt == int(np.argmax(got)) or got[nxt] == got.max()   # device argmax: lowest index among maxima
        assert nxt == int(np.flatnonzero(got == got.max())[0])
    eng.close()


def test_small_prompt_eval_then_decode():
    """a 3-token prompt in one eval (M <= 4: the exact-integer GEMV path), then two single-token steps"""
    m = toy(seed=5)
    orc, eng = m.graph(), m.engine()
    prompt = [1, 200, 31]
    check_logits(eng.eval(prompt, 0)[0], orc.eval(prompt, 0))
    check_logits(eng.eval([8], 3)[0], orc.eval([8], 3))
    check_logits(eng.eval([250], 4)[0], orc.eval([250], 4))
    eng.close()


@pytest.mark.parametrize("n_head", [4, 2])
def test_long_prompt_goes_through_the_tensor_core_gemm(n_head):
    """M > 16 rows take the bf16 wgmma GEMM: same graph, bf16 matmul numerics (looser bar), KV cache usable afterwards"""
    m = toy(n_head, n_head, seed=6)
    orc, eng = m.graph(), m.engine()
    prompt = list(np.random.default_rng(1).integers(3, m.hp["n_vocab"], 24))
    check_logits(eng.eval(prompt, 0)[0], orc.eval(prompt, 0), tol=4e-2)
    check_logits(eng.eval([42], 24)[0], orc.eval([42], 24), tol=4e-2)
    eng.close()


def test_exact_prefill_mode_keeps_reference_numerics_for_long_prompts():
    """a 70-token prompt: default = bf16 tensor-core GEMM (looser bar); exact mode = pieces of 32 on the integer tensor cores,
    held to the north-star 1e-2, and the KV cache it leaves serves the following single-token steps"""
    m = toy(seed=12, n_ctx=96)
    orc, jig, eng = m.graph(), m.graph(jig=True), m.engine()
    prompt = [int(t) for t in np.random.default_rng(3).integers(3, m.hp["n_vocab"], 70)]
    want = orc.eval(prompt, 0)
    # 70 positions of Q8_0 rounding decisions: the CPU graph against itself with inputs moved by +-64 ulp differs by 1.6e-2 here
    # (+-4 ulp: 0.9e-2) -- the per-step bar on that measured floor
    tol = bar(distance(jig.eval(prompt, 0), want))
    eng.set_exact_prefill(True)
    check_logits(eng.eval(prompt, 0)[0], want, tol=tol)
    check_logits(eng.eval([9], 70)[0], orc.eval([9], 70), tol=tol)
    eng.close()


def test_generate_feeds_the_argmax_on_device():
    m = toy(seed=7)
    orc, eng = m.graph(), m.engine()
    first, n_new = 11, 10
    out = eng.generate(first, 0, n_new)
    # the same steps through ns_llama_eval, one host round trip per token: identical kernels, identical picks
    eng2 = m.engine()
    t, ref = first, []
    for pos in range(n_new):
        _, t = eng2.eval([t], pos, want_logits=False)
        ref.append(t)
    assert list(out) == ref
    # and against the CPU graph while the pick is unambiguous
    t = first
    for pos in range(n_new):
        want = orc.eval([t], pos)
        if not unambiguous(want):
            break
        assert int(out[pos]) == greedy(want)
        t = int(out[pos])
    eng.close()
    eng2.close()


def test_argument_checks():
    m = toy(seed=8, n_ctx=16)
    eng = m.engine()
    rc = ns.lib().ns_llama_eval(eng.h, np.zeros(20, np.int32).ctypes.data, 20, 0, None, None)
    assert rc != 0 and "n_ctx" in ns.last_error()
    eng2 = ns.Llama(**m.hp)
    with pytest.raises(RuntimeError):
        eng2.eval([1], 0)                      # no tensors set: refuses instead of reading null pointers
    eng.close()
    eng2.close()


def test_llama2_7b_shaped_greedy_decode_matches_the_reference_engine():
    """North-star parity at the model's real shapes: n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000, Q4_0 weights (two
    decoder layers + the full output head keep the CPU side to a few minutes).  A 12-token prompt evaluated token by token, then
    16 greedy steps against the REFERENCE's own graph engine (oracle.RefNeLlama = core/ne_layers.c compiled where it lies; the
    numpy restatement -- bit-identical to it -- when that library is absent).  Token ids must be identical wherever the
    reference's top-2 margin exceeds the bound; ids are fed from the reference so one near-tie cannot derail the rest.

    The logit bound.  Every matmul of the step is within 4e-7 of the oracle at these shapes (profiles/diag_7b_stages.py; the
    residue is fp32 summation order), but each Q8_0 activation quantisation is a rounding DISCONTINUITY: one code that lands
    on the other side of .5 moves that element by 1/127 of its block maximum, and the next quantisation amplifies that
    again.  The reference run against ITSELF with every embedding value moved by +-64 ulp (4e-6 relative) differs by
    1.4e-2 max / 3e-3 rms of max|logit| on this model, and does not grow further with a larger perturbation: that is the
    conditioning floor of the Q4_0 x Q8_0 path at this width, measured below in the same loop (`self_err`).  The CUDA
    step has to stay within max(1e-2, 1.5 x the largest self_err seen so far) of the reference at every step, and within 2.5e-2 outright."""
    rng = np.random.default_rng(2024)
    m = llama2_7b_shaped(rng, n_ctx=64)
    m.draw_jig(rng)
    ref, ref_jig = m.reference(), m.reference(jig=True)  # the same engine, inputs moved by +-64 ulp
    eng = m.engine()
    prompt = [1] + [int(t) for t in rng.integers(3, m.hp["n_vocab"], 11)]
    pos, agree, checked, worst, running = 0, 0, 0, 0.0, RunningBar()
    t = prompt[0]
    for step in range(len(prompt) + 16):
        want = ref.eval([t], pos)
        tol = running(want, ref_jig.eval([t], pos))
        got, nxt = eng.eval([t], pos)
        s, err = scale(want), float(np.abs(got - want).max())
        assert err <= tol * s, (step, err / s, running.floor)
        worst = max(worst, err / s)
        if unambiguous(want, 2 * tol):
            checked += 1
            agree += int(nxt == greedy(want))
        pos += 1
        t = prompt[pos] if pos < len(prompt) else greedy(want)
    print(f"7B-shape decode: worst |dlogit|/max|logit| {worst:.2e}; the reference against itself (+-64 ulp inputs) {running.floor:.2e}; "
          f"ids {agree}/{checked}")
    assert checked >= 8 and agree == checked, (agree, checked)
    eng.close()
    close(ref, ref_jig)


@pytest.mark.parametrize("n_head,n_head_kv", [(4, 4), (2, 2), (4, 2)])
def test_tensor_core_prompt_attention_matches_the_scalar_kernel(n_head, n_head_kv, monkeypatch):
    """Prompts of >= 8 tokens run the causal attention on mma.sync (attn_mma_kernel: 64 query rows per CTA, K/V tiles of 64 keys):
    several q tiles, several key tiles, ragged last tiles and a non-zero n_past (chunked prompt), head sizes 64 and 128, GQA.
    Compared with the decode-shaped scalar kernel (NS_ATTN_SCALAR=1, itself held to the CPU graph by the tests above) on an engine
    whose matmuls are smooth (fp32 compute): only the fp16 rounding of the probabilities differs (5e-4 relative)."""
    eng = smooth(n_head, n_head_kv, n_ctx=400, seed=21).engine()
    rng = np.random.default_rng(8)
    p1 = [int(t) for t in rng.integers(3, 320, 37)]
    p2 = [int(t) for t in rng.integers(3, 320, 141)]
    p3 = [int(t) for t in rng.integers(3, 320, 200)]

    def run():
        return [eng.eval(p1, 0)[0], eng.eval(p2, len(p1))[0], eng.eval([11], len(p1) + len(p2))[0], eng.eval(p3, len(p1) + len(p2) + 1)[0]]

    a = run()
    monkeypatch.setenv("NS_ATTN_SCALAR", "1")
    b = run()
    monkeypatch.delenv("NS_ATTN_SCALAR")
    for x, y in zip(a, b):
        assert np.isfinite(x).all()
        # bf16 activation rounding in the tensor-core GEMMs of both runs turns 5e-4 into a few 1e-3; a layout bug would be O(1)
        assert float(np.abs(x - y).max()) <= 1e-2 * max(1.0, float(np.abs(y).max())), float(np.abs(x - y).max())
    eng.close()


def test_tensor_core_prompt_attention_against_the_cpu_graph():
    """a 37 + 90 token chunked prompt in exact-prefill mode (integer matmuls as the reference, attention on mma.sync) against the
    CPU graph, bar = north star or 1.5 x the graph's own conditioning floor (see the exact-prefill test)"""
    m = toy(seed=23, n_ctx=160)
    orc, jig, eng = m.graph(), m.graph(jig=True), m.engine()
    eng.set_exact_prefill(True)
    rng = np.random.default_rng(9)
    p1 = [int(t) for t in rng.integers(3, m.hp["n_vocab"], 37)]
    p2 = [int(t) for t in rng.integers(3, m.hp["n_vocab"], 90)]
    w1, w2 = orc.eval(p1, 0), orc.eval(p2, len(p1))
    j1, j2 = jig.eval(p1, 0), jig.eval(p2, len(p1))
    tol = bar(max(distance(j1, w1), distance(j2, w2)))
    check_logits(eng.eval(p1, 0)[0], w1, tol=tol)
    check_logits(eng.eval(p2, len(p1))[0], w2, tol=tol)
    eng.close()


@pytest.mark.parametrize("n_head,n_head_kv", [(4, 4), (2, 1)])
def test_split_context_decode_attention_matches_the_single_cta_kernel(n_head, n_head_kv, monkeypatch):
    """decode attention with K / V staged by TMA and the context split into ranges of 256 positions (attn_decode_kernel) against the
    one-CTA-per-head kernel with dependent row loads (NS_ATTN_OLD_DECODE=1), token by token across the 256 and 512 boundaries
    (1, 2 and 3 active ranges; a range holding only the new token), head sizes 64 and 128, GQA; smooth fp32-compute engine"""
    rng = np.random.default_rng(5)
    prompt = [int(t) for t in rng.integers(3, 320, 250)]
    steps = [int(t) for t in rng.integers(3, 320, 12)]
    jump = [int(t) for t in rng.integers(3, 320, 250)]

    def run(old):
        if old:
            monkeypatch.setenv("NS_ATTN_OLD_DECODE", "1")
        eng = smooth(n_head, n_head_kv, n_ctx=600, seed=31).engine()
        outs = [eng.eval(prompt, 0)[0]]
        n_past = len(prompt)
        for t in steps:  # positions 250 .. 261: crosses into the second range
            outs.append(eng.eval([t], n_past)[0])
            n_past += 1
        outs.append(eng.eval(jump, n_past)[0])  # to position 512
        n_past += len(jump)
        gen = eng.generate(7, n_past, 6)        # three ranges, through the decode graph
        eng.close()
        if old:
            monkeypatch.delenv("NS_ATTN_OLD_DECODE")
        return outs, gen

    a, ga = run(False)
    b, gb = run(True)
    for i, (x, y) in enumerate(zip(a, b)):
        assert np.isfinite(x).all()
        assert float(np.abs(x - y).max()) <= 1e-2 * max(1.0, float(np.abs(y).max())), (i, float(np.abs(x - y).max()))
    assert len(ga) == 6 and len(gb) == 6  # (greedy ids may part at a near-tie; the logits above are the check)


def test_long_context_decode_against_the_cpu_graph():
    """300-token prompt (tensor-core prompt attention), then single-token steps with two active ranges, against the CPU graph"""
    m = toy(seed=33, n_ctx=320)
    orc, jig, eng = m.graph(), m.graph(jig=True), m.engine()
    eng.set_exact_prefill(True)
    rng = np.random.default_rng(11)
    prompt = [int(t) for t in rng.integers(3, m.hp["n_vocab"], 300)]
    want = orc.eval(prompt, 0)
    check_logits(eng.eval(prompt, 0)[0], want, tol=bar(distance(jig.eval(prompt, 0), want)))
    n_past = len(prompt)
    for t in (9, 200, 31):
        want = orc.eval([t], n_past)
        check_logits(eng.eval([t], n_past)[0], want, tol=bar(distance(jig.eval([t], n_past), want)))
        n_past += 1
    eng.close()

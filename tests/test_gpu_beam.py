"""Beam search in the eval step (ns_llama_beam_search, include/ns_b200.h): the reference's beam_search_flow over per-beam KV blocks,
candidates scored on the device.

1. The candidates kernel equals its host restatement (ns_beam_candidates_row_host) bit for bit: vocab 320 / 32000 / 128256, k 4
   .. 64, 1 .. 32 rows, ties, -inf entries and EOS-masked rows, a poisoned workspace whose tickets are zero again afterwards.
2. ns_llama_kv_copy: the copied bytes equal their source and every other block and position is unchanged; a sequence forked by the
   copy decodes bit-identically to the original; pair lists that overlap are refused without a launch.
3. Engine identity: on the toy models of tests/llama_models.py (GQA 4 on 2, Q4_0 and Q6_K lm_head), ns_llama_beam_search equals
   oracle/beam_search.cpp with the library's row arithmetic, driven by a second engine's own eval_batch / decode_batch logits for
   the same running rows (its KV blocks kept by the same rule: a beam continues in its source's block or a copy of it), bit for bit
   in tokens and scores -- num_beams 2 / 4 / 8, 1-4 requests, passes of 2 and of 3 or more rows.
4. (Not here: the oracle flow on the toy models' CPU-graph logits.  Their running bar is 2.5e-2 of max |logit|, wider than the
   gap between a request's B-th and (B+1)-th candidate in nearly every search, so such a comparison would cover almost no step;
   DESIGN.md section 4 says so.)
5. Llama-2-7B shapes (head size 128, vocab 32000): the first step's candidates against the reference engine's prompt logits
   (oracle/_ref's engine where built, else the CPU graph) under the same bar, and the identity of 3 over a few steps.
6. Launch structure, from the CUDA activity torch.profiler records: per step one replay of the decode graph, one candidates
   launch, one device-to-host copy and at most one KV copy launch; refusals launch nothing; blocks from n num_beams up are
   untouched; a greedy generate afterwards equals one before."""
import ctypes as C

import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
from llama_models import bar, bits, close, distance, llama2_7b_shaped, rows, scale, toy
from test_beam_cpu import oracle_search, orc  # noqa: F401 -- the oracle fixture
from torch.profiler import ProfilerActivity, profile

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


# ------------------------------------------------------------------------------------------------------------- 1. kernel
def _rows(rng, n, V):
    x = (rng.standard_normal((n, V)) * rng.choice([1e-2, 1.0, 30.0], (n, 1))).astype(np.float32)
    for r in range(n):
        kind = r % 4
        if kind == 1:
            x[r] = np.round(x[r] * 2) / 2  # many equal logits
        elif kind == 2:
            x[r, ::3] = -np.inf
        elif kind == 3:
            x[r, rng.integers(0, V, 5)] = x[r].max() + 1  # a five-way tie for the max
    return x


@pytest.mark.parametrize("V", [320, 32000, 128256])
def test_kernel_equals_the_host_restatement(V):
    rng = np.random.default_rng(V)
    wsb = ns.lib().ns_llama_beam_candidates_workspace_bytes(32, 64)
    ws = torch.full((wsb,), 0xFF, dtype=torch.uint8, device="cuda")
    ws[:128] = 0
    cases = [(1, 4), (2, 8), (3, 6), (7, 16), (13, 64), (32, 8), (32, 64)] if V == 320 else [(1, 64), (5, 4), (32, 16)]
    for n, k in cases:
        x = _rows(rng, n, V)
        prev = (rng.standard_normal(n) * 5).astype(np.float32)
        mask = (rng.integers(0, 2, n)).astype(np.int32)
        eos = int(np.argmax(x[0])) if n > 1 else 2  # the row's best token is EOS: the mask moves the selection
        K = min(k, V)
        out = torch.zeros((n, K, 2), dtype=torch.int32, device="cuda")
        xd = torch.from_numpy(x).cuda()
        torch.cuda.synchronize()
        rc = ns.beam_candidates(xd.data_ptr(), n, V, k, prev, mask, eos, out.data_ptr(), ws.data_ptr())
        assert rc == 0, ns.last_error()
        torch.cuda.synchronize()
        assert torch.count_nonzero(ws[:128]).item() == 0, (n, k)
        got = out.cpu().numpy()
        for r in range(n):
            ids, sc = ns.beam_candidates_row_host(x[r], k, float(prev[r]), bool(mask[r]), eos)
            assert np.array_equal(got[r, :, 0], ids), (n, k, r)
            assert np.array_equal(got[r, :, 1].view(np.uint32), bits(sc)), (n, k, r)


# ------------------------------------------------------------------------------------------------------------- 2. kv_copy
def _kv(eng):
    """the whole fp16 K and V caches on the host, [n_layer][n_seq][n_head_kv][n_ctx][hd] each"""
    k, v = eng.kv_cache()
    hp = eng.hp
    hd = hp.n_embd // hp.n_head
    n_seq = eng.kv_bytes() // (2 * hp.n_layer * hp.n_head_kv * hp.n_ctx * hd * 2)
    shape = (hp.n_layer, n_seq, hp.n_head_kv, hp.n_ctx, hd)
    out = []
    for p in (k, v):
        a = np.empty(shape, np.float16)
        ns.lib().bestla_device_memcpy_sync(a.ctypes.data, C.c_void_p(p), a.nbytes, None)
        out.append(a)
    return out


def test_kv_copy_bytes_and_forks():
    eng = toy(4, 2, n_ctx=96).engine(n_seq=6)
    rng = np.random.default_rng(3)
    prompts = [rng.integers(0, 320, 9 + 3 * s).tolist() for s in range(4)]
    eng.eval_batch([0, 1, 2, 3], prompts, [0, 0, 0, 0])
    k0, v0 = _kv(eng)
    eng.kv_copy([1, 3], [4, 5], 2, 11)
    k1, v1 = _kv(eng)
    for a0, a1 in ((k0, k1), (v0, v1)):
        want = a0.copy()
        want[:, 4, :, 2:11] = a0[:, 1, :, 2:11]
        want[:, 5, :, 2:11] = a0[:, 3, :, 2:11]
        assert np.array_equal(want.view(np.uint16), a1.view(np.uint16))
    # a fork decodes as the original: block 2's 15 positions into block 4, then the same token on both
    eng.kv_copy([2], [4], 0, 15)
    lg, _ = eng.decode_batch([2, 4], [7, 7], [15, 15])
    assert np.array_equal(bits(lg[0]), bits(lg[1]))
    before = eng.kv_bytes()
    n0 = ns.lib().ns_launch_count()
    for src, dst, p0, p1 in [([1, 4], [4, 5], 0, 4), ([1, 2], [3, 3], 0, 4), ([1], [1], 0, 4), ([1], [6], 0, 4), ([1], [2], 3, 2),
                             ([1], [2], 0, 97)]:
        with pytest.raises(RuntimeError):
            eng.kv_copy(src, dst, p0, p1)
    assert ns.lib().ns_launch_count() == n0 and eng.kv_bytes() == before
    eng.close()


# ------------------------------------------------------------------------------------------------------------- 3. identity
class EngineModel:
    """the logits of the rows the oracle asks for, from a second engine: the prompts in one eval_batch pass into blocks r B, then
    one decode_batch pass over every running beam, each beam in its source's block or, after the first, in a block no beam
    continues in, receiving a copy of its source's positions"""

    def __init__(self, eng, B):
        self.eng, self.B, self.where, self.rows = eng, B, {}, []

    def __call__(self, req, hists):
        self.rows.append(len(hists))
        B = self.B
        if not self.where:
            lg, _ = self.eng.eval_batch([r * B for r in req], hists, [0] * len(req))
            self.where = {(r, tuple(h)): r * B for r, h in zip(req, hists)}
            return lg
        blocks = [None] * len(hists)
        taken = set()
        for i, (r, h) in enumerate(zip(req, hists)):
            src = self.where[(r, tuple(h[:-1]))]
            if src not in taken:
                taken.add(src)
                blocks[i] = src
        for i, (r, h) in enumerate(zip(req, hists)):
            if blocks[i] is None:
                free = min(b for b in range(r * B, r * B + B) if b not in taken)
                taken.add(free)
                self.eng.kv_copy([self.where[(r, tuple(h[:-1]))]], [free], 0, len(h) - 1)
                blocks[i] = free
        lg, _ = self.eng.decode_batch(blocks, [h[-1] for h in hists], [len(h) - 1 for h in hists])
        self.where = {(r, tuple(h)): b for r, h, b in zip(req, hists, blocks)}
        return lg


@pytest.mark.parametrize("out_fmt", ["q4_0", "q6_K"])
def test_engine_equals_the_oracle_on_its_own_logits(orc, out_fmt):  # noqa: F811
    m = toy(4, 2, out_fmt, n_ctx=96)
    eng, ref = m.engine(n_seq=32), m.engine(n_seq=32)
    rng = np.random.default_rng(11)
    V, eos = 320, 5
    row_counts = set()
    for B, n, max_new, min_new, lp, early in [(2, 1, 8, 0, 1.0, False), (2, 2, 6, 2, 0.5, True), (4, 1, 7, 0, 2.0, True),
                                              (4, 4, 5, 3, 1.0, False), (8, 2, 6, 0, -1.0, False), (8, 4, 4, 1, 0.0, True),
                                              (2, 3, 9, 0, 1.0, True)]:
        prompts = [rng.integers(0, V, int(rng.integers(1, 20))).tolist() for _ in range(n)]
        got = eng.beam_search(prompts, B, max_new, min_new, lp, early, eos)
        model = EngineModel(ref, B)
        want = oracle_search(orc, V, prompts, model, B, max_new, min_new, lp, early, eos)
        row_counts.update(model.rows)
        for (gt, gs), (wt, ws) in zip(got, want):
            assert np.array_equal(gt, wt), (B, n, got, want)
            assert bits(np.float32(gs)) == bits(np.float32(ws)), (B, n, got, want)
    assert {2, 4} <= row_counts and max(row_counts) == 32  # GEMV-tile and tensor-core passes
    eng.close()
    ref.close()


# ------------------------------------------------------------------------------------------------------------- 5. 7B shapes
def test_llama2_7b_shaped_candidates_and_identity(orc):  # noqa: F811
    """synthetic Llama-2-7B weights (tests/llama_models.py: Q4_0, two layers, the full output head); the first step's candidates
    under the per-step bar of the reference against its +-64 ulp jig"""
    rng = np.random.default_rng(2025)
    m = llama2_7b_shaped(rng, n_ctx=64)
    V = m.hp["n_vocab"]
    prompts = [[1] + [int(t) for t in rng.integers(3, V, 9)], [1] + [int(t) for t in rng.integers(3, V, 6)]]
    m.draw_jig(rng)
    last = {}
    for which in ("ref", "jig"):
        r = m.reference(jig=which == "jig")
        last[which] = [rows(r, p, 0)[-1] for p in prompts]  # the prompt evaluated token by token, as the 7B logits_all test
        close(r)
    eng, ref = m.engine(8), m.engine(8)
    B = 4
    # the first step's candidates: the candidates kernel on the engine's prompt logits against float64 log_softmax of the
    # reference's, where the reference's own margins clear the bar
    lg, _ = eng.eval_batch([0, B], prompts, [0, 0])
    xd = torch.from_numpy(np.ascontiguousarray(lg)).cuda()
    ws = torch.zeros(ns.lib().ns_llama_beam_candidates_workspace_bytes(2, B), dtype=torch.uint8, device="cuda")
    out = torch.zeros((2, B, 2), dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    assert ns.beam_candidates(xd.data_ptr(), 2, V, B, np.zeros(2, np.float32), np.zeros(2, np.int32), 2, out.data_ptr(), ws.data_ptr()) == 0
    torch.cuda.synchronize()
    cand = out.cpu().numpy()
    checked = 0
    for r in range(2):
        want, self_w = last["ref"][r].astype(np.float64), last["jig"][r]
        sc, bound = scale(want), bar(distance(self_w, want))
        order = np.lexsort((np.arange(V), -want))
        lsm = want - (want.max() + np.log(np.exp(want - want.max()).sum()))
        scores = cand[r, :, 1].view(np.float32)
        for j in range(B):
            assert abs(float(scores[j]) - lsm[cand[r, j, 0]]) <= 2 * bound * sc, (r, j, scores[j], lsm[cand[r, j, 0]])
            if want[order[j]] - want[order[j + 1]] > 2 * bound * sc and (j == 0 or want[order[j - 1]] - want[order[j]] > 2 * bound * sc):
                assert cand[r, j, 0] == order[j], (r, j)
                checked += 1
    print(f"7B-shape first-step candidates: {checked} of {2 * B} ranks clear of the bar and equal")
    # the identity of 3 over a few steps: 8 rows (integer tensor cores) and 2 rows (GEMV), head size 128, vocab 32000
    for Bq, ps in ((4, prompts), (2, prompts[:1])):
        got = eng.beam_search(ps, Bq, 4, 0, 1.0, False, 2)
        want = oracle_search(orc, V, ps, EngineModel(ref, Bq), Bq, 4, 0, 1.0, False, 2)
        for (gt, gs), (wt, wsc) in zip(got, want):
            assert np.array_equal(gt, wt) and bits(np.float32(gs)) == bits(np.float32(wsc)), (Bq, got, want)
    eng.close()
    ref.close()


# ------------------------------------------------------------------------------------------------------------- 6. structure
def test_launches_refusals_and_untouched_blocks():
    m = toy(4, 2, n_ctx=96)
    eng = m.engine(n_seq=12)
    rng = np.random.default_rng(5)
    # a greedy generate before and after, on block 0
    eng.eval([1, 2, 3], 0)
    g0 = eng.generate(4, 3, 6)
    eng.eval_batch([8, 9, 10, 11], [rng.integers(0, 320, 7).tolist() for _ in range(4)], [0] * 4)
    prompts = [rng.integers(0, 320, 10).tolist() for _ in range(2)]
    B, T = 4, 6
    eng.beam_search(prompts, B, T)  # captures the graphs
    kb, vb = _kv(eng)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eng.beam_search(prompts, B, T)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events()]
    count = {k: sum(k in nm for nm in names) for k in ("beam_candidates_kernel", "kv_copy_kernel", "argmax_kernel", "embed_kernel",
                                                        "Memcpy DtoH")}
    # the prompt pass and T - 1 decode steps, each ending in its argmax (the graph's last node); one candidates launch and one copy
    # of the candidates to the host per step; the prompt into the other beams' blocks before the first decode, then at most one KV
    # copy launch per later step
    assert count["embed_kernel"] == T and count["argmax_kernel"] == T, count
    assert count["beam_candidates_kernel"] == T and count["Memcpy DtoH"] == T, count
    assert 1 <= count["kv_copy_kernel"] <= T - 1, count
    ka, va = _kv(eng)
    assert np.array_equal(kb[:, 8:].view(np.uint16), ka[:, 8:].view(np.uint16))  # blocks n B .. untouched
    assert np.array_equal(vb[:, 8:].view(np.uint16), va[:, 8:].view(np.uint16))
    eng.eval([1, 2, 3], 0)
    assert np.array_equal(eng.generate(4, 3, 6), g0)
    # refusals launch nothing
    L = ns.lib()
    n0 = L.ns_launch_count()
    for kw, ps in [(dict(num_beams=1), prompts), (dict(num_beams=8), prompts), (dict(num_beams=4, max_new_tokens=90), prompts),
                   (dict(min_new_tokens=-1), prompts), (dict(eos_token_id=320), prompts), (dict(length_penalty=float("nan")), prompts),
                   (dict(), [[1]] * 4), (dict(), [[]])]:
        with pytest.raises(RuntimeError):
            eng.beam_search(ps, **kw)
    eng.set_sampling(top_k=4, seed=1)
    with pytest.raises(RuntimeError, match="sampling"):
        eng.beam_search(prompts, 2, 3)
    eng.set_sampling(None)
    assert L.ns_launch_count() == n0
    eng.close()
    one = m.engine()
    one.set_streaming(4)
    with pytest.raises(RuntimeError, match="streaming"):
        one.beam_search([[1, 2]], 2, 3)
    one.close()

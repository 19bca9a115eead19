"""Generation past n_ctx (ns_llama_set_streaming): the ring variant of the split decode attention on its own
(ns_llama_attention_ring) and the whole eval step, against the ring mode of the CPU graph (oracle/llama_model.py, itself bit-exact
with the reference's engine: tests/test_streaming_cpu.py)."""
import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
from llama_models import RunningBar, close, llama2_7b_shaped, scale, toy, unambiguous
from oracle import llama_model as lm
from oracle import streaming as sm
from oracle.llama_model import greedy

pytestmark = pytest.mark.gpu

# Output bars relative to max|V|.  The split decode kernel sums e in fp32 in its own order and rounds p = e / sum to fp16, where the
# reference sums in double: now and then one p lands on the other side of an fp16 rounding boundary, which moves the output by one
# fp16 ulp of p times V -- at most 2^-11 max|V|.  Over the thousands of steps of a ring run that happens (measured on an H100 80GB
# HBM3: 1.1e-4 at one step of the hd 64, group 4, n_ctx 48 case), so a step is held to that one-ulp bound, and the mean error
# over the run to the mean bar of tests/test_gpu_attention.py's split decode (1e-6).
STEP_MAX, RUN_MEAN = 2.0 ** -11, 1e-6


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


# ------------------------------------------------------------------------------------------------------------- the kernel
def _ring_step(q, k, v, kc, vc, H, HK, hd, n_ctx, n_keep, n_total, ws):
    out = torch.full((H * hd,), float("nan"), device="cuda")
    torch.cuda.synchronize()
    rc = ns.lib().ns_llama_attention_ring(q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), H, HK, hd, n_ctx, n_keep,
                                          n_total, 10000.0, out.data_ptr(), ws.data_ptr(), None)
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    return out


def _gpu_q_rot(q, H, HK, hd, pos):
    """q rotated at pos by the device's sincosf (rope_kv_kernel of the generic path leaves it in place), so that the output check
    measures the attention, not sincosf against libm"""
    q = q.clone()
    kc = torch.zeros((HK, pos + 1, hd), dtype=torch.float16, device="cuda")
    vc = kc.clone()
    k = torch.zeros((HK * hd,), device="cuda")
    out = torch.empty((H * hd,), device="cuda")
    ws = torch.zeros(ns.lib().ns_llama_attention_workspace_bytes(H, hd, pos + 1), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc = ns.lib().ns_llama_attention(ns.ATTN_GENERIC, q.data_ptr(), k.data_ptr(), k.data_ptr(), kc.data_ptr(), vc.data_ptr(), H, HK, hd,
                                     pos + 1, pos, 1, 10000.0, 1.0, out.data_ptr(), ws.data_ptr(), None)
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    return q.cpu().numpy().reshape(1, H, hd)


RING_CASES = [(64, 1, 48, 0), (128, 2, 48, 4), (64, 4, 48, 1), (128, 4, 48, 0),
              (128, 1, 300, 256), (64, 2, 300, 4), (128, 4, 300, 1), (64, 1, 300, 0),
              (64, 1, 520, 1), (128, 2, 520, 256), (128, 4, 520, 4), (64, 4, 520, 0), (128, 1, 520, 0)]


@pytest.mark.parametrize("hd,group,n_ctx,n_keep", RING_CASES)
def test_ring_step_against_the_shift_of_its_own_cache(hd, group, n_ctx, n_keep):
    """A full cache, then 2 (n_ctx - n_keep) ring steps (the slot wraps twice and crosses every range boundary).  After each step:
    every cache row but the new one is bit-identical to rope_shift_f16 of the cache before the step (sinks unchanged), the new K
    row within 1 fp16 ulp of its pair's magnitude plus 1 ulp of its own of the oracle's (RoPE at n_ctx leaves 1 ulp -- CUDA sincosf
    is not glibc's -- which the shift turns between the pair's two elements, then rounds once more),
    the new V row exact, the output
    against the attention over all n_ctx slots (STEP_MAX, RUN_MEAN), the tickets zero again."""
    HK = 2
    H = HK * group
    r = np.random.default_rng(hd + group + n_ctx + n_keep)
    g = torch.Generator(device="cuda").manual_seed(n_ctx + n_keep)
    kc = torch.randn((HK, n_ctx, hd), generator=g, device="cuda").half()
    vc = torch.randn((HK, n_ctx, hd), generator=g, device="cuda").half()
    ws = torch.zeros(ns.lib().ns_llama_attention_workspace_bytes(H, hd, n_ctx), dtype=torch.uint8, device="cuda")
    table = sm.shift_table(hd)
    worst, means, past = 0.0, [], 0
    for n_total in range(n_ctx, n_ctx + 2 * (n_ctx - n_keep)):
        q = r.normal(0, 2, (H * hd,)).astype(np.float32)
        k = r.normal(0, 1, (HK, hd)).astype(np.float32)
        v = r.normal(0, 1, (HK, hd)).astype(np.float32)
        prev_k, prev_v = kc.cpu().numpy(), vc.cpu().numpy()
        qd = torch.from_numpy(q).cuda()
        out = _ring_step(qd, torch.from_numpy(k.ravel()).cuda(), torch.from_numpy(v.ravel()).cuda(), kc, vc, H, HK, hd, n_ctx, n_keep,
                         n_total, ws).cpu().numpy().reshape(1, H, hd)
        got_k, got_v = kc.cpu().numpy(), vc.cpu().numpy()
        s = sm.ring_slot(n_total, n_ctx, n_keep)
        want_k = sm.rope_shift_f16(prev_k, n_keep, table)
        rows = np.arange(n_ctx) != s
        assert np.array_equal(got_k[:, rows].view(np.uint16), want_k[:, rows].view(np.uint16)), (n_total, "shifted K rows")
        assert np.array_equal(got_k[:, :n_keep].view(np.uint16), prev_k[:, :n_keep].view(np.uint16)), (n_total, "sinks")
        new = sm.rope_shift_f16(lm.rope_mode0(k, n_ctx, hd).astype(np.float16)[:, None], 0, table)[:, 0].astype(np.float32)
        pair = np.sqrt(new[:, 0::2] ** 2 + new[:, 1::2] ** 2).repeat(2, axis=-1)
        tol = (np.spacing(pair.astype(np.float16)) + np.spacing(np.abs(new).astype(np.float16))).astype(np.float32)
        assert (np.abs(got_k[:, s].astype(np.float32) - new) <= tol).all(), (n_total, "new K row")
        want_v = prev_v.copy()
        want_v[:, s] = v.astype(np.float16)
        assert np.array_equal(got_v.view(np.uint16), want_v.view(np.uint16)), (n_total, "V cache")
        assert (ws[16:16 + 4 * H].view(torch.int32).cpu().numpy() == 0).all(), "tickets"
        assert np.isfinite(out).all()
        q_rot = _gpu_q_rot(qd, H, HK, hd, n_ctx - 1)
        ref = lm.attention_reference(q_rot, got_k, got_v, n_ctx - 1)  # m = 1 at n_past = n_ctx - 1: all n_ctx slots, no mask
        stated = lm.attention_stated(q_rot, got_k, got_v, n_ctx - 1, "split") if n_ctx > lm.SPLIT_KEYS else ref
        vmax = float(np.abs(got_v.astype(np.float32)).max())
        d = np.abs(out.astype(np.float64) - stated)
        emax, emean = float(d.max()) / vmax, float(d.mean()) / vmax
        assert emax <= STEP_MAX, (n_total, emax, emean)
        assert float(np.abs(out - ref).max()) <= 1e-3 * float(np.abs(ref).max()), n_total
        worst = max(worst, emax)
        means.append(emean)
        past += emax > 5e-5
    assert np.mean(means) <= RUN_MEAN, np.mean(means)
    print(f"ring hd{hd} group{group} ctx{n_ctx} keep{n_keep}: {len(means)} steps, max {worst:.2e}, mean {np.mean(means):.2e} (x max|V|); "
          f"steps past 5e-5: {past}")


def test_ring_entry_argument_checks():
    L = ns.lib()
    assert L.ns_llama_attention_ring(1, 1, 1, 1, 1, 4, 2, 32, 64, 4, 70, 10000.0, 1, 1, None) == -4  # head size 32: nothing launched
    for n_keep in (-1, 64):
        assert L.ns_llama_attention_ring(1, 1, 1, 1, 1, 4, 2, 64, 64, n_keep, 70, 10000.0, 1, 1, None) == -1
    assert L.ns_llama_attention_ring(1, 1, 1, 1, 1, 4, 3, 64, 64, 4, 70, 10000.0, 1, 1, None) == -1


# ------------------------------------------------------------------------------------------------------------- the engine
def _ring_graph(m, n_keep, jig=False):
    """the CPU graph of a toy model in ring mode"""
    return sm.OracleLlamaRing(m.hp, m.tok_jig if jig else m.tok, m.out_norm, m.out_rows, m.layers, n_keep)


def _ring_engine(m, n_keep):
    eng = m.engine()
    eng.set_streaming(n_keep)
    return eng


@pytest.mark.parametrize("n_head,n_head_kv,n_keep", [(4, 4, 4), (4, 2, 1), (2, 1, 0), (2, 2, 4)])
def test_ring_decode_matches_the_cpu_graph(n_head, n_head_kv, n_keep):
    """a 4-token prompt, then single tokens to 2.5 n_ctx (n_ctx 48), teacher-forced: logits at every step within the north star
    of OracleLlamaRing (or 1.5 x the CPU graph's own floor, measured with +-64 ulp inputs, where that is larger), ids
    equal wherever the top-2 margin exceeds the bound; head sizes 64 and 128, MHA and GQA"""
    m = toy(n_head, n_head_kv, seed=40 + n_keep)
    orc, jig, eng = _ring_graph(m, n_keep), _ring_graph(m, n_keep, jig=True), _ring_engine(m, n_keep)
    n_ctx = m.hp["n_ctx"]
    seq = [int(t) for t in np.random.default_rng(n_head).integers(3, m.hp["n_vocab"], int(2.5 * n_ctx))]
    steps = [(seq[:4], 0)] + [([seq[t]], t) for t in range(4, len(seq))]
    worst, running = 0.0, RunningBar()
    for toks, pos in steps:
        want = orc.eval(toks, pos)
        tol = running(want, jig.eval(toks, pos))
        got, nxt = eng.eval(toks, pos)
        s, err = scale(want), float(np.abs(got - want).max())
        assert err <= tol * s, (pos, err, running.floor)
        worst = max(worst, err / s)
        if unambiguous(want, 2 * tol):
            assert nxt == greedy(want), pos
    print(f"ring decode H{n_head}/{n_head_kv} keep{n_keep}: worst |dlogit|/max|logit| {worst:.2e}, CPU graph floor {running.floor:.2e}")
    eng.close()


def test_before_the_wrap_streaming_is_bit_identical_to_plain():
    for n_head_kv in (4, 2):
        m = toy(4, n_head_kv, seed=50)
        plain, ring = m.engine(), _ring_engine(m, 4)
        seq = [int(t) for t in np.random.default_rng(2).integers(3, 320, 48)]
        steps = [(seq[:20], 0)] + [([seq[t]], t) for t in range(20, 48)]
        for toks, pos in steps:
            a, b = plain.eval(toks, pos)[0], ring.eval(toks, pos)[0]
            assert np.array_equal(a.view(np.int32), b.view(np.int32)), pos
        plain.close()
        ring.close()


def test_a_ring_step_launches_as_many_kernels_as_a_plain_step():
    L = ns.lib()
    counts = []
    for n_keep in (None, 4):
        eng = toy(4, 2, seed=51).engine()
        if n_keep is not None:
            eng.set_streaming(n_keep)
        eng.eval([1, 2, 3], 0)
        before = L.ns_launch_count()
        eng.eval([5], 3)  # builds the decode graph: one eager pass and the captured one
        counts.append(L.ns_launch_count() - before)
        eng.close()
    assert counts[0] == counts[1] and counts[0] > 0, counts


def test_generate_across_two_wraps_matches_the_eval_loop():
    m = toy(4, 2, seed=52)
    a, b = _ring_engine(m, 4), _ring_engine(m, 4)
    prompt = [3, 14, 15, 92, 65]
    n_new = 2 * 48 + 30  # the record buffer (n_ctx picks) drains three times
    a.eval(prompt, 0)
    gen = a.generate(35, len(prompt), n_new)
    _, t = b.eval(prompt, 0)
    t, ref = 35, []
    for i in range(n_new):
        _, t = b.eval([t], len(prompt) + i, want_logits=False)
        ref.append(t)
    assert list(gen) == ref
    # and the context continues where generate left it
    pos = len(prompt) + n_new
    assert np.array_equal(a.eval([7], pos)[0], b.eval([7], pos)[0])
    a.close()
    b.close()


def test_streaming_argument_checks():
    L = ns.lib()
    m = toy(4, 2, seed=53, n_ctx=16)
    hp, eng = dict(m.hp), m.engine()
    toks = np.arange(16, dtype=np.int32)
    ev = lambda n, past: L.ns_llama_eval(eng.h, toks.ctypes.data, n, past, None, None)
    assert ev(1, 16) == -1 and "n_ctx" in ns.last_error()          # streaming off: past n_ctx stays invalid
    assert L.ns_llama_set_streaming(eng.h, 16) == -1               # n_keep must be < n_ctx
    assert L.ns_llama_set_streaming(eng.h, -2) == -1
    eng.set_streaming(2)
    assert ev(16, 0) == 0
    assert ev(2, 16) == -4                                         # N > 1 past n_ctx (llama.cpp:467)
    assert ev(1, 17) == -1                                         # not the next position
    assert ev(1, 16) == 0 and ev(1, 17) == 0                       # the ring wraps
    assert ev(1, 10) == -1                                         # a rewind into rotated slots
    assert ev(1, 18) == 0
    assert ev(3, 2) == 0 and ev(1, 5) == 0                          # a restart that keeps the sinks
    eng.set_streaming(-1)
    assert ev(1, 16) == -1
    eng.close()
    e2 = toy(2, 2, seed=54).engine()
    assert L.ns_llama_set_streaming(e2.h, 4) == 0
    e2.close()
    hp["rope_scale"] = 2.0
    e3 = ns.Llama(**hp)
    assert L.ns_llama_set_streaming(e3.h, 4) == -4                 # scaled RoPE: the reference disagrees with itself
    e3.close()
    hp["rope_scale"], hp["n_head"], hp["n_head_kv"] = 1.0, 8, 8
    e4 = ns.Llama(**hp)                                            # head size 32
    assert L.ns_llama_set_streaming(e4.h, 4) == -4
    e4.close()


def test_llama2_7b_shaped_ring_against_the_reference_engine():
    """n_embd 4096, 32 heads of 128, two layers, vocab 32000, Q4_0, n_ctx 256, n_keep 4: a 240-token prompt (exact prefill), then
    single teacher-forced tokens to position 300, against the reference's engine running the shift-RoPE-K graph
    (oracle.streaming.RefNeLlamaRing) where oracle/_ref was built, else against OracleLlamaRing.  Bound: max(1e-2, 1.5 x the
    reference's own floor with +-64 ulp inputs, running maximum), at most 2.5e-2 (tests/llama_models.py)."""
    rng = np.random.default_rng(2025)
    n_keep = 4
    m = llama2_7b_shaped(rng, n_ctx=256)
    m.draw_jig(rng)
    if sm.ref_ne_ring() is not None:
        table = sm.shift_table(128)
        ref, ref_jig = (sm.RefNeLlamaRing(m.hp, t_, m.out_norm, m.out_rows, m.layers, n_keep, table) for t_ in (m.tok, m.tok_jig))
    else:
        ref, ref_jig = _ring_graph(m, n_keep), _ring_graph(m, n_keep, jig=True)
    eng = m.engine()
    eng.set_exact_prefill(True)
    eng.set_streaming(n_keep)
    seq = [1] + [int(t) for t in rng.integers(3, m.hp["n_vocab"], 299)]
    steps = [(seq[:240], 0)] + [([seq[t]], t) for t in range(240, 300)]
    worst, running, checked, agree = 0.0, RunningBar(), 0, 0
    for toks, pos in steps:
        want = ref.eval(toks, pos)
        tol = running(want, ref_jig.eval(toks, pos))
        got, nxt = eng.eval(toks, pos)
        s, err = scale(want), float(np.abs(got - want).max())
        assert err <= tol * s, (pos, err, running.floor)
        worst = max(worst, err / s)
        if unambiguous(want, 2 * tol):
            checked += 1
            agree += int(nxt == greedy(want))
    print(f"7B-shape ring: worst |dlogit|/max|logit| {worst:.2e}; the reference against itself (+-64 ulp) {running.floor:.2e}; ids "
          f"{agree}/{checked}")
    assert agree == checked
    eng.close()
    close(ref, ref_jig)

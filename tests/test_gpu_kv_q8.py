"""The Q8_0 KV cache on the device (include/ns_b200.h, NS_KV_Q8_0; neural_speed_b200/csrc/kv_cache.cuh).

1. store: every new V row, and K at position 0 (angle 0: RoPE is exact), byte for byte the runtime quantize_row_q8_0 of the row;
   K at other positions within one fp16 ulp of d and one code of quantising the CPU graph's rotated row -- for the append
   kernel (prompt rows) and the decode kernel (its own new row); nothing else of the cache changes.
2. equivalences, bit for bit: the Q8_0 prompt kernel (single and ragged) and the fp16 prompt kernel on an fp16 cache holding
   deq(C); each batched decode row and the single-sequence decode on its block; each ragged segment and its own NS_ATTN_MMA call.
3. the decode kernel against attention_stated("split") on the dequantised cache it left (its own new row included), at the bars
   tests/test_gpu_attention.py holds the fp16 decode kernel to.
4. the engine against the CPU graph with a Q8_0 cache (tests/test_kv_q8_cpu.py) under the running bar on that graph's own jig: eval /
   generate, decode_batch, eval_batch with chunked prompts and eval_all on the toy models (MHA and GQA, Q4_0 and Q6_K heads),
   and the 7B-shaped model.
5. beam search: kv_copy moves both planes; a Q8_0 engine's search is the oracle flow driven by its own logits.
6. refusals launch nothing; kv_bytes follows the layout; a type change restarts every block and drops the graphs."""
import ctypes as C

import numpy as np
import pytest
import torch

import neural_speed_b200 as ns
import oracle
from llama_models import bar, bits, distance, llama2_7b_shaped, toy
from oracle import llama_model as lm
from test_beam_cpu import oracle_search, orc  # noqa: F401 -- the oracle fixture
from test_gpu_beam import EngineModel
from test_kv_q8_cpu import graph_q8

pytestmark = pytest.mark.gpu

E_INVALID, E_UNSUPPORTED = -1, -4
SPLIT, ROWS, MMA, GENERIC = ns.ATTN_SPLIT_DECODE, ns.ATTN_ROWS, ns.ATTN_MMA, ns.ATTN_GENERIC
SPLIT_BARS = (5e-5, 1e-6)  # test_gpu_attention.py's bars of the split decode kernel: max and mean |d| / max|V|


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    ns.lib().bestla_init()
    yield


# ------------------------------------------------------------------------------------------------------------- host layout
def quantize(rows):
    """runtime quantize_row_q8_0 of rows [..., hd] -> (codes [..., hd] int8, d [..., hd / 32] float16)"""
    r = np.ascontiguousarray(rows, np.float32)
    hd = r.shape[-1]
    b = oracle.quantize_q8_0(r.reshape(-1, hd), variant="runtime").reshape(-1, hd // 32, 34)
    d = b[:, :, :2].copy().view(np.float16)[..., 0].reshape(r.shape[:-1] + (hd // 32,))
    return b[:, :, 2:].copy().view(np.int8).reshape(r.shape), d


def deq(codes, d):
    """fp16(q * d): what the kernels read"""
    hd = codes.shape[-1]
    return (codes.astype(np.float32) * np.repeat(d.astype(np.float32), 32, axis=-1)).astype(np.float16).reshape(codes.shape[:-1] + (hd,))


class Planes:
    """one layer's Q8_0 caches of n_seq blocks on the device: codes [n_seq][HK][n_ctx][hd] int8, scales [n_seq][HK][stride] fp16"""

    def __init__(self, n_seq, HK, n_ctx, hd):
        self.shape, self.stride = (n_seq, HK, n_ctx, hd), ns.kv_d_stride(n_ctx, hd)
        self.kq = torch.zeros(self.shape, dtype=torch.int8, device="cuda")
        self.vq = torch.zeros_like(self.kq)
        self.kd = torch.zeros((n_seq, HK, self.stride), dtype=torch.float16, device="cuda")
        self.vd = torch.zeros_like(self.kd)

    def fill(self, rng, n_fill):
        """positions [0, n_fill[s]) of block s: quantised random rows"""
        for s, L in enumerate(n_fill):
            for q, d in ((self.kq, self.kd), (self.vq, self.vd)):
                c, sc = quantize(rng.normal(0, 1, (self.shape[1], L, self.shape[3])).astype(np.float32))
                q[s, :, :L] = torch.from_numpy(c).cuda()
                d[s, :, :L * (self.shape[3] // 32)] = torch.from_numpy(sc.reshape(self.shape[1], -1)).cuda()
        return self

    def clone(self):
        p = Planes.__new__(Planes)
        p.shape, p.stride = self.shape, self.stride
        p.kq, p.vq, p.kd, p.vd = (x.clone() for x in (self.kq, self.vq, self.kd, self.vd))
        return p

    def ptrs(self, s=0):
        return tuple(x[s].data_ptr() for x in (self.kq, self.kd, self.vq, self.vd))

    def host(self, s):
        """block s on the host: (K codes, K scales [HK][n_ctx][hd / 32], V codes, V scales)"""
        HK, n_ctx, hd = self.shape[1:]
        out = []
        for q, d in ((self.kq, self.kd), (self.vq, self.vd)):
            out += [q[s].cpu().numpy(), d[s, :, :n_ctx * (hd // 32)].cpu().numpy().reshape(HK, n_ctx, hd // 32)]
        return out

    def deq(self, s):
        kq, kd, vq, vd = self.host(s)
        return deq(kq, kd), deq(vq, vd)

    def same(self, other):
        return all(torch.equal(a, b) for a, b in zip((self.kq, self.vq, self.kd, self.vd), (other.kq, other.vq, other.kd, other.vd)))


def _inputs(rng, m, H, HK, hd):
    return (rng.normal(0, 2, (m, H, hd)).astype(np.float32), rng.normal(0, 1, (m, HK, hd)).astype(np.float32),
            rng.normal(0, 1, (m, HK, hd)).astype(np.float32))


def _dev(*arrays):
    return [torch.from_numpy(np.ascontiguousarray(a).reshape(a.shape[0], -1)).cuda() for a in arrays]


def run_q8(kernel, planes, q, k, v, H, HK, hd, n_ctx, n_past, rope_scale=1.0, s=0):
    """one ns_llama_attention_q8_0 call on block s of planes -> (out [m][H][hd], q after the call)"""
    m = q.shape[0]
    qd, kd, vd = _dev(q, k, v)
    out = torch.full((m, H * hd), float("nan"), device="cuda")
    ws = torch.zeros(ns.lib().ns_llama_attention_workspace_bytes(H, hd, n_ctx), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc = ns.attention_q8_0(kernel, qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), planes.ptrs(s), H, HK, hd, n_ctx, n_past, m,
                           out.data_ptr(), ws.data_ptr(), rope_scale=rope_scale)
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(m, H, hd), qd.cpu().numpy().reshape(m, H, hd)


def run_f16(kernel, kc, vc, q, k, v, H, HK, hd, n_ctx, n_past, rope_scale=1.0):
    m = q.shape[0]
    qd, kd, vd = _dev(q, k, v)
    kc, vc = torch.from_numpy(kc).cuda(), torch.from_numpy(vc).cuda()
    out = torch.full((m, H * hd), float("nan"), device="cuda")
    ws = torch.zeros(ns.lib().ns_llama_attention_workspace_bytes(H, hd, n_ctx), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc = ns.lib().ns_llama_attention(kernel, qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), kc.data_ptr(), vc.data_ptr(), H, HK, hd, n_ctx,
                                     n_past, m, 10000.0, rope_scale, out.data_ptr(), ws.data_ptr(), None)
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    return out.cpu().numpy().reshape(m, H, hd), kc.cpu().numpy()


# ------------------------------------------------------------------------------------------------------------- 1. store, 3. decode
def check_store(before, after, k, v, pos, hd):
    """the new rows at positions pos: V and K at position 0 byte-exact, other K within 1 ulp of d / 1 code; the rest untouched"""
    kq0, kd0, vq0, vd0 = before
    kq1, kd1, vq1, vd1 = after
    k_rot = lm.rope_mode0_rows(k, pos, hd)
    wkq, wkd = quantize(k_rot)
    wvq, wvd = quantize(v)
    untouched = np.ones(kq0.shape[1], bool)
    untouched[pos] = False
    for a0, a1 in ((kq0, kq1), (kd0, kd1), (vq0, vq1), (vd0, vd1)):
        assert np.array_equal(a0[:, untouched].view(np.uint8), a1[:, untouched].view(np.uint8)), "rows other than the new ones"
    assert np.array_equal(vq1[:, pos], wvq.transpose(1, 0, 2)) and np.array_equal(bits16(vd1[:, pos]), bits16(wvd.transpose(1, 0, 2)))
    gq, gd = kq1[:, pos].astype(np.int32), kd1[:, pos]
    wq, wd = wkq.transpose(1, 0, 2).astype(np.int32), wkd.transpose(1, 0, 2)
    at0 = np.asarray(pos) == 0
    if at0.any():
        assert np.array_equal(gq[:, at0], wq[:, at0]) and np.array_equal(bits16(gd[:, at0]), bits16(wd[:, at0])), "K at position 0"
    assert (np.abs(gq - wq) <= 1).all(), "K codes beyond one step"
    ulp = np.spacing(np.abs(wd)).astype(np.float32)
    assert (np.abs(gd.astype(np.float32) - wd.astype(np.float32)) <= ulp).all(), "K scales beyond one fp16 ulp"


def bits16(a):
    return np.ascontiguousarray(a, np.float16).view(np.uint16)


DECODE = [(128, 8, 1, 2048, p) for p in (0, 1, 255, 256, 1023, 2047)] + [(64, 4, 2, 2048, p) for p in (0, 300, 2047)] + \
         [(128, 32, 32, 600, 599), (64, 32, 8, 300, 17)]


@pytest.mark.parametrize("hd,H,HK,n_ctx,n_past", DECODE)
def test_decode_store_and_stated_arithmetic(hd, H, HK, n_ctx, n_past):
    """1-8 ranges, MHA and GQA, head sizes 64 and 128"""
    rng = np.random.default_rng(n_past + hd)
    planes = Planes(1, HK, n_ctx, hd).fill(rng, [n_past])
    before = planes.host(0)
    q, k, v = _inputs(rng, 1, H, HK, hd)
    after_planes = planes.clone()
    out, _ = run_q8(SPLIT, after_planes, q, k, v, H, HK, hd, n_ctx, n_past)
    check_store(before, after_planes.host(0), k, v, [n_past], hd)
    # the q the kernels rotate (rope_kv_kernel's, as test_gpu_attention.py takes it): the MMA path rotates q in place
    _, q_rot = run_q8(MMA, planes.clone(), q, k, v, H, HK, hd, n_ctx, n_past)
    kc, vc = after_planes.deq(0)
    L = n_past + 1
    stated = lm.attention_stated(q_rot, kc[:, :L], vc[:, :L], n_past, "split")
    vmax = float(np.abs(vc[:, :L].astype(np.float32)).max())
    d = np.abs(out.astype(np.float64) - stated)
    assert np.isfinite(out).all()
    assert d.max() / vmax <= SPLIT_BARS[0] and d.mean() / vmax <= SPLIT_BARS[1], (d.max() / vmax, d.mean() / vmax)


# ------------------------------------------------------------------------------------------------------------- 2. equivalences
IDENTITY = 1e30  # rope_scale: every angle below 1e-26, so RoPE leaves fp16 values as they are (the fp16 side can append deq(C))


@pytest.mark.parametrize("hd,H,HK,n_past,m", [(128, 8, 2, 0, 64), (128, 8, 8, 37, 3), (64, 4, 1, 100, 130), (64, 8, 2, 255, 7),
                                              (128, 4, 4, 500, 12)])
def test_prompt_kernel_store_and_equivalence(hd, H, HK, n_past, m):
    n_ctx = 768
    rng = np.random.default_rng(m + n_past)
    planes = Planes(1, HK, n_ctx, hd).fill(rng, [n_past])
    before = planes.host(0)
    q, k, v = _inputs(rng, m, H, HK, hd)
    p1 = planes.clone()
    run_q8(MMA, p1, q, k, v, H, HK, hd, n_ctx, n_past)
    check_store(before, p1.host(0), k, v, list(range(n_past, n_past + m)), hd)
    # equivalence: identity rotation on both sides; the fp16 kernel appends fp16(deq) rows, i.e. deq(C) itself
    p2 = planes.clone()
    out_q8, _ = run_q8(MMA, p2, q, k, v, H, HK, hd, n_ctx, n_past, rope_scale=IDENTITY)
    kc, vc = p2.deq(0)
    new = slice(n_past, n_past + m)
    kin, vin = kc[:, new].transpose(1, 0, 2).astype(np.float32), vc[:, new].transpose(1, 0, 2).astype(np.float32)
    out_f16, kc_after = run_f16(MMA, kc, vc, q, kin, vin, H, HK, hd, n_ctx, n_past, rope_scale=IDENTITY)
    assert np.array_equal(kc_after[:, new].astype(np.float32), kc[:, new].astype(np.float32))  # the fp16 side read deq(C)
    assert np.array_equal(out_q8, out_f16)


def _batch_ws(n, H, hd, n_ctx):
    return torch.zeros(ns.lib().ns_llama_attention_batch_workspace_bytes(n, H, hd, n_ctx), dtype=torch.uint8, device="cuda")


@pytest.mark.parametrize("hd,H,HK", [(128, 8, 2), (64, 4, 4)])
def test_batched_decode_rows_equal_single_sequence_decode(hd, H, HK):
    n_ctx, n_seq = 1100, 6
    rng = np.random.default_rng(hd)
    fill = [0, 5, 256, 700, 1099, 300]
    planes = Planes(n_seq, HK, n_ctx, hd).fill(rng, fill)
    seqs, past = [3, 0, 4, 1, 2], [700, 0, 1099, 5, 256]
    n = len(seqs)
    q, k, v = _inputs(rng, n, H, HK, hd)
    pb = planes.clone()
    qd, kd, vd = _dev(q, k, v)
    out = torch.full((n, H * hd), float("nan"), device="cuda")
    torch.cuda.synchronize()
    rc = ns.attention_batch_q8_0(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), pb.ptrs(0), n_seq, seqs, past, H, HK, hd, n_ctx,
                                 out.data_ptr(), _batch_ws(n, H, hd, n_ctx).data_ptr())
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    out = out.cpu().numpy().reshape(n, H, hd)
    ps = planes.clone()
    for i, (s, p) in enumerate(zip(seqs, past)):
        o, _ = run_q8(SPLIT, ps, q[i:i + 1], k[i:i + 1], v[i:i + 1], H, HK, hd, n_ctx, p, s=s)
        assert np.array_equal(bits(o[0]), bits(out[i])), (i, s, p)
    assert ps.same(pb)


@pytest.mark.parametrize("hd,H,HK", [(128, 8, 2), (64, 4, 1)])
def test_ragged_segments_equal_their_own_calls(hd, H, HK):
    n_ctx, n_seq = 512, 4
    rng = np.random.default_rng(7 + hd)
    planes = Planes(n_seq, HK, n_ctx, hd).fill(rng, [40, 0, 200, 7])
    seqs, n_tok, past = [2, 0, 3, 1], [70, 5, 1, 64], [200, 40, 7, 0]
    T = sum(n_tok)
    q, k, v = _inputs(rng, T, H, HK, hd)
    pr = planes.clone()
    qd, kd, vd = _dev(q, k, v)
    out = torch.full((T, H * hd), float("nan"), device="cuda")
    ws = torch.zeros(ns.lib().ns_llama_attention_ragged_workspace_bytes(len(seqs), T), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    rc = ns.attention_ragged_q8_0(qd.data_ptr(), kd.data_ptr(), vd.data_ptr(), pr.ptrs(0), n_seq, seqs, n_tok, past, H, HK, hd, n_ctx,
                                  out.data_ptr(), ws.data_ptr())
    assert rc == 0, ns.last_error()
    torch.cuda.synchronize()
    out = out.cpu().numpy().reshape(T, H, hd)
    ps, r0 = planes.clone(), 0
    for s, m, p in zip(seqs, n_tok, past):
        o, _ = run_q8(MMA, ps, q[r0:r0 + m], k[r0:r0 + m], v[r0:r0 + m], H, HK, hd, n_ctx, p, s=s)
        assert np.array_equal(bits(o), bits(out[r0:r0 + m])), (s, m, p)
        r0 += m
    assert ps.same(pr)


# ------------------------------------------------------------------------------------------------------------- 4. engine
class Held:
    """device logits and the Q8_0 CPU graph's, held to the bar on the largest distance of that graph to its jig over the whole
    test (RunningBar's floor, taken once every step of the test has been evaluated: a code that lands on the other side of a
    rounding boundary moves a K / V value by a Q8_0 step, and the floor is a property of the model, not of one step)"""

    def __init__(self):
        self.rows, self.floor = [], 0.0

    def add(self, got, want, jig_want, what):
        self.floor = max(self.floor, distance(jig_want, want))
        self.rows.append((distance(got, want), what))

    def check(self):
        b = bar(self.floor)
        worst = max(d for d, _ in self.rows)
        bad = [(d, w) for d, w in self.rows if d > b]
        assert not bad, (bad[:5], b)
        return worst, b


class Q8Oracle:
    """one sequence on the Q8_0 CPU graph and its jig; eval() records the device logits against both"""

    def __init__(self, model, held):
        self.orc, self.jig, self.held = graph_q8(model), graph_q8(model, jig=True), held

    def eval(self, got, tokens, n_past, what=""):
        want = self.orc.eval(tokens, n_past)
        self.held.add(got, want, self.jig.eval(tokens, n_past), what)
        return want


def q8_engine(model, n_seq=1):
    eng = model.engine(n_seq)
    eng.set_kv_type("q8_0")
    assert eng.kv_type() == "q8_0"
    return eng


@pytest.mark.parametrize("HK,out_fmt", [(4, "q4_0"), (1, "q6_K"), (2, "q4_0")])
def test_engine_against_the_q8_0_graph(HK, out_fmt):
    m = toy(4, HK, out_fmt, seed=HK, n_ctx=64)
    rng = np.random.default_rng(HK)
    held = Held()
    # eval / generate: a 12-token prompt, then 16 greedy steps
    eng = q8_engine(m)
    prompt = rng.integers(0, 320, 12).tolist()
    o = Q8Oracle(m, held)
    got, tok = eng.eval(prompt, 0)
    o.eval(got, prompt, 0, "prompt")
    picks = []
    for i in range(16):
        picks.append(tok)
        got, tok = eng.eval([picks[-1]], 12 + i)
        o.eval(got, [picks[-1]], 12 + i, f"step {i}")
    eng.eval(prompt, 0)
    gen = eng.generate(picks[0], 12, 16)
    assert np.array_equal(gen[:15], np.array(picks[1:], np.int32))
    # eval_seq of 2 .. 7 rows (the tensor-core prompt kernel under Q8_0)
    got, _ = eng.eval_seq(0, prompt[:5], 0)
    Q8Oracle(m, held).eval(got, prompt[:5], 0, "eval_seq 5 rows")
    eng.close()
    # decode_batch / eval_batch (chunked prompts) / eval_all over three sequences
    eng = q8_engine(m, 3)
    prompts = [rng.integers(0, 320, L).tolist() for L in (9, 1, 20)]
    orcs = [Q8Oracle(m, held) for _ in prompts]
    past = [0, 0, 0]
    chunks = [[p[:6], p[6:]] if len(p) > 6 else [p] for p in prompts]
    for c in range(2):
        seqs = [s for s in range(3) if c < len(chunks[s])]
        lg, nxt = eng.eval_batch(seqs, [chunks[s][c] for s in seqs], [past[s] for s in seqs])
        for j, s in enumerate(seqs):
            orcs[s].eval(lg[j], chunks[s][c], past[s], f"eval_batch chunk {c} seq {s}")
            past[s] += len(chunks[s][c])
    toks = [7, 11, 13]
    for i in range(16):
        lg, nxt = eng.decode_batch([0, 1, 2], toks, past)
        for s in range(3):
            orcs[s].eval(lg[s], [toks[s]], past[s], f"decode_batch {i} seq {s}")
            past[s] += 1
        toks = [int(t) for t in nxt]
    # eval_all: a scoring pass appending one more segment to each sequence
    segs = [rng.integers(0, 320, L).tolist() for L in (3, 1, 4)]
    _, am, lgs = eng.eval_all([0, 1, 2], segs, past, want_logits=True)
    for s in range(3):
        for j, t in enumerate(segs[s]):
            orcs[s].eval(lgs[s][j], [t], past[s] + j, f"eval_all seq {s} row {j}")
    eng.close()
    worst, b = held.check()
    print(f"HK {HK} {out_fmt}: worst distance {worst:.3e}, bar {b:.3e} (floor {held.floor:.3e})")


def test_llama2_7b_shaped_against_the_q8_0_graph():
    rng = np.random.default_rng(77)
    m = llama2_7b_shaped(rng, n_ctx=64)
    m.draw_jig(rng)
    held = Held()
    o = Q8Oracle(m, held)
    eng = q8_engine(m)
    f16 = m.engine()
    prompt = [1] + [int(t) for t in rng.integers(3, 32000, 11)]
    got, tok = eng.eval(prompt, 0)
    ref16, _ = f16.eval(prompt, 0)
    o.eval(got, prompt, 0, "prompt")
    gap = distance(got, ref16)
    for i in range(16):
        t = tok
        got, tok = eng.eval([t], 12 + i)
        ref16, _ = f16.eval([t], 12 + i)
        o.eval(got, [t], 12 + i, f"step {i}")
        gap = max(gap, distance(got, ref16))
    worst, b = held.check()
    print(f"7B-shaped: worst distance {worst:.3e}, bar {b:.3e}; Q8_0 vs fp16 engine logit distance {gap:.3e} (measured, not asserted)")
    eng.close()
    f16.close()


# ------------------------------------------------------------------------------------------------------------- 5. beam search
def _planes_host(eng):
    """the four planes on the host: codes [n_layer][n_seq][HK][n_ctx][hd] int8, scales [n_layer][n_seq][HK][stride] fp16"""
    hp = eng.hp
    hd = hp.n_embd // hp.n_head
    n_seq = eng.kv_bytes() // ns.kv_bytes("q8_0", hp.n_layer, 1, hp.n_head_kv, hp.n_ctx, hd)
    k, kd, v, vd = eng.kv_planes()
    out = []
    for p, shape, dt in ((k, (hp.n_ctx, hd), np.int8), (kd, (ns.kv_d_stride(hp.n_ctx, hd),), np.float16), (v, (hp.n_ctx, hd), np.int8),
                         (vd, (ns.kv_d_stride(hp.n_ctx, hd),), np.float16)):
        a = np.empty((hp.n_layer, n_seq, hp.n_head_kv) + shape, dt)
        ns.lib().bestla_device_memcpy_sync(a.ctypes.data, C.c_void_p(p), a.nbytes, None)
        out.append(a)
    return out


def test_kv_copy_moves_both_planes():
    eng = q8_engine(toy(4, 2, n_ctx=96), 6)
    hd = 64
    rng = np.random.default_rng(3)
    eng.eval_batch([0, 1, 2, 3], [rng.integers(0, 320, 9 + 3 * s).tolist() for s in range(4)], [0, 0, 0, 0])
    before = _planes_host(eng)
    eng.kv_copy([1, 3], [4, 5], 2, 11)
    after = _planes_host(eng)
    for i, (a0, a1) in enumerate(zip(before, after)):
        want = a0.copy()
        per = hd // 32 if i % 2 else None  # scale planes: hd / 32 halves per position
        sl = slice(2 * per, 11 * per) if per else slice(2, 11)
        want[:, 4, :, sl] = a0[:, 1, :, sl]
        want[:, 5, :, sl] = a0[:, 3, :, sl]
        assert np.array_equal(want.view(np.uint8), a1.view(np.uint8)), i
    assert before[1][:, 1, :, :22].any()  # the copied scales are not zeros
    eng.kv_copy([2], [4], 0, 15)
    lg, _ = eng.decode_batch([2, 4], [7, 7], [15, 15])
    assert np.array_equal(bits(lg[0]), bits(lg[1]))
    eng.close()


def test_beam_search_equals_the_oracle_on_its_own_logits(orc):  # noqa: F811
    m = toy(4, 2, "q4_0", n_ctx=96)
    eng, ref = q8_engine(m, 32), q8_engine(m, 32)
    rng = np.random.default_rng(12)
    V, eos = 320, 5
    for B, n, max_new, min_new, lp, early in [(2, 2, 6, 2, 0.5, True), (4, 4, 5, 3, 1.0, False), (8, 3, 6, 0, -1.0, False)]:
        prompts = [rng.integers(0, V, int(rng.integers(1, 20))).tolist() for _ in range(n)]
        got = eng.beam_search(prompts, B, max_new, min_new, lp, early, eos)
        want = oracle_search(orc, V, prompts, EngineModel(ref, B), B, max_new, min_new, lp, early, eos)
        for (gt, gs), (wt, ws) in zip(got, want):
            assert np.array_equal(gt, wt), (B, n, got, want)
            assert bits(np.float32(gs)) == bits(np.float32(ws)), (B, n, got, want)
    eng.close()
    ref.close()


# ------------------------------------------------------------------------------------------------------------- 6. refusals
def test_refusals_bytes_and_reset():
    L = ns.lib()
    m = toy(4, 2, n_ctx=48)
    eng = m.engine(2)
    hd, HK, n_layer, n_ctx = 64, 2, 2, 48
    assert eng.kv_bytes() == ns.kv_bytes("f16", n_layer, 2, HK, n_ctx, hd)
    n0 = L.ns_launch_count()
    for bad in (2, -1, 7):
        assert L.ns_llama_set_kv_type(eng.h, bad) == E_INVALID
    assert eng.kv_type() == "f16"
    # streaming and Q8_0, in both orders (streaming needs one block)
    eng.set_sequences(1)
    eng.set_streaming(4)
    assert L.ns_llama_set_kv_type(eng.h, 1) == E_UNSUPPORTED and eng.kv_type() == "f16"
    eng.set_streaming(-1)
    eng.set_kv_type("q8_0")
    assert L.ns_llama_set_streaming(eng.h, 4) == E_UNSUPPORTED
    assert L.ns_llama_kv_cache(eng.h, C.byref(C.c_void_p()), C.byref(C.c_void_p())) == E_UNSUPPORTED
    assert eng.kv_bytes() == ns.kv_bytes("q8_0", n_layer, 1, HK, n_ctx, hd)
    eng.set_sequences(3)
    assert eng.kv_bytes() == ns.kv_bytes("q8_0", n_layer, 3, HK, n_ctx, hd) and eng.kv_type() == "q8_0"
    assert L.ns_launch_count() == n0
    # head sizes other than 64 / 128
    for E, H in ((256, 8), (320, 4), (384, 4)):
        other = ns.Llama(320, E, H, H, 1, 512, 32)
        assert L.ns_llama_set_kv_type(other.h, 1) == E_UNSUPPORTED, E // H
        other.close()
    # NS_ATTN_ROWS / NS_ATTN_GENERIC and head size 96 on the parity entries
    for kernel, H, hd_ in ((ROWS, 4, 64), (GENERIC, 4, 128), (SPLIT, 4, 96), (MMA, 4, 80)):
        planes = Planes(1, 4, 64, max(hd_, 64))
        t = torch.zeros(4 * 4 * hd_, device="cuda")
        ws = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
        rc = ns.attention_q8_0(kernel, t.data_ptr(), t.data_ptr(), t.data_ptr(), planes.ptrs(0), H, 4, hd_, 64, 3, 1, t.data_ptr(),
                               ws.data_ptr())
        assert rc == E_UNSUPPORTED, (kernel, hd_)
    assert L.ns_launch_count() == n0
    # a type change restarts every block and drops the graphs: the same steps give the same logits as a fresh Q8_0 engine
    fresh = q8_engine(m)
    eng.set_sequences(1)
    eng.generate(3, 0, 5)
    eng.set_kv_type("f16")
    eng.generate(3, 0, 5)
    eng.set_kv_type("q8_0")
    assert not any(a.any() for a in _planes_host(eng))
    for e in (eng, fresh):
        e.eval([3, 9, 27], 0)
    a, b = eng.generate(4, 3, 6), fresh.generate(4, 3, 6)
    assert np.array_equal(a, b)
    la, _ = eng.eval([a[-1]], 9)
    lb, _ = fresh.eval([b[-1]], 9)
    assert np.array_equal(bits(la), bits(lb))
    eng.close()
    fresh.close()

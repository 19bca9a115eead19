"""CPU restatements for ggml Q8_0 weights, shared by the Q8_0 tests.

* `quantize_weights`: ne_quantize_q8_0's rows (quantize_row_q8_0_reference, core/ne_layers.c:13029), the weight quantiser of
  the reference's converters.
* `vec_dot` / `mul_mat`: ne_vec_dot_q8_0_q8_0's AVX2 body (core/layers/vec_dot.h:594-621) inside
  ne_compute_forward_mul_mat_q_f32 (ne_layers.c:7085-7203): the activations are quantised by quantize_row_q8_0 (x86 body, the
  pinned oracle), and per 32-block i the eight fp32 lanes take acc[l] = fma(fp32(d_w * d_a), (float)sum_{j<4} w[4l+j] a[4l+j],
  acc[l]); the lanes are summed in hsum_float_8's order ((a0+a4)+(a2+a6)) + ((a1+a5)+(a3+a7)).  mul_sum_i8_pairs_float is
  exact for every code pair a file can hold: maddubs sees |w| <= 128 and a code of at most 127 in magnitude, so no pair sum
  reaches the int16 limit.
* `ring_stated`: the ring GEMV's stated arithmetic for 8-bit codes (DESIGN.md section 4), without oracle.ring_stated's 4-bit
  chunk bound.
* `OracleLlamaQ8` / `RefNeLlamaQ8`: oracle/llama_model.OracleLlama with every matmul Q8_0, and the reference's own engine on
  NE_TYPE_Q8_0 tensors.
"""
import numpy as np

import llama_models as lm
import oracle
from oracle.llama_model import OracleLlama, _fmaf

BLOCK = 34  # sizeof(block_q8_0), core/data_types.h:107-111
NE_TYPE_Q8_0 = 8


def quantize_weights(w):
    """fp32 [N, K] -> block_q8_0 rows uint8 [N, K/32*34]"""
    return oracle.quantize_q8_0(np.ascontiguousarray(w, np.float32), variant="reference")


def split(rows, k):
    """block_q8_0 rows -> (codes int32 [N, K], d fp32 [N, K/32])"""
    b = np.ascontiguousarray(rows, np.uint8).reshape(rows.shape[0], k // 32, BLOCK)
    q = b[:, :, 2:].copy().view(np.int8).reshape(rows.shape[0], k).astype(np.int32)
    d = b[:, :, :2].copy().view(np.float16).reshape(rows.shape[0], k // 32).astype(np.float32)
    return q, d


def join(q, d):
    """(codes int [N, K], d fp16-representable [N, K/32]) -> block_q8_0 rows"""
    n, k = q.shape
    b = np.zeros((n, k // 32, BLOCK), np.uint8)
    b[:, :, :2] = np.asarray(d, np.float16).reshape(n, k // 32, 1).view(np.uint8)
    b[:, :, 2:] = np.asarray(q, np.int8).reshape(n, k // 32, 32).view(np.uint8)
    return b.reshape(n, k // 32 * BLOCK)


def dequantize(rows, k):
    """dequantize_row_q8_0 (vectors/cpu/quantize.h:780): fp32(d) * q"""
    q, d = split(rows, k)
    return (q.astype(np.float32).reshape(q.shape[0], k // 32, 32) * d[:, :, None]).reshape(q.shape[0], k)


def _hsum8(acc):
    """hsum_float_8 over the last axis, in fp32"""
    r = [(acc[..., i + 4] + acc[..., i]).astype(np.float32) for i in range(4)]
    return ((r[0] + r[2]).astype(np.float32) + (r[1] + r[3]).astype(np.float32)).astype(np.float32)


def dots(wq, wd, aq, ad, row_chunk=512):
    """ne_vec_dot_q8_0_q8_0 of every (activation row m, weight row n): codes int [N, K] / [M, K], scales [N, nb] / [M, nb]
    -> fp32 [M, N]"""
    n, k = wq.shape
    m = aq.shape[0]
    nb = k // 32
    out = np.empty((m, n), np.float32)
    a4 = aq.reshape(m, nb, 8, 4).astype(np.int32)
    for r0 in range(0, n, row_chunk):
        w4 = wq[r0:r0 + row_chunk].reshape(-1, nb, 8, 4).astype(np.int32)
        for mi in range(m):
            si = (w4 * a4[mi][None]).sum(axis=3)                                        # [n', nb, 8] exact int
            d = (wd[r0:r0 + row_chunk] * ad[mi][None, :]).astype(np.float32)            # fp32(d_w * d_a) [n', nb]
            acc = np.zeros((si.shape[0], 8), np.float32)
            for b in range(nb):
                acc = _fmaf(np.broadcast_to(d[:, b:b + 1], acc.shape), si[:, b].astype(np.float32), acc)
            out[mi, r0:r0 + row_chunk] = _hsum8(acc)
    return out


def quantize_act(a):
    """quantize_row_q8_0 (x86 body) of every row: (codes int32 [M, K], d fp32 [M, K/32])"""
    a = np.ascontiguousarray(a, np.float32)
    return split(oracle.quantize_q8_0(a), a.shape[1])


def vec_dot(wrow, arow, k):
    """ne_vec_dot_q8_0_q8_0 on one pair of block_q8_0 rows"""
    wq, wd = split(np.asarray(wrow, np.uint8).reshape(1, -1), k)
    aq, ad = split(np.asarray(arow, np.uint8).reshape(1, -1), k)
    return np.float32(dots(wq, wd, aq, ad)[0, 0])


def mul_mat(rows, a):
    """ne_compute_forward_mul_mat_q_f32 for NE_TYPE_Q8_0: rows uint8 [N, K/32*34], a fp32 [M, K] -> fp32 [M, N]"""
    a = np.ascontiguousarray(a, np.float32)
    wq, wd = split(rows, a.shape[1])
    aq, ad = quantize_act(a)
    return dots(wq, wd, aq, ad)


def ring_stated(a, rows, lanes=False):
    """The ring GEMV on Q8_0 weights (gemv_ring_kernel, DESIGN.md section 4): per 32-chunk c, isum_c = sum a*q (exact),
    t_c = fp32(a_d * w_d); lane L runs acc = fmaf(isum_c, t_c, acc) over c = L, L + 32, ... from +0, and lane 0 of the xor
    butterfly (16, 8, 4, 2, 1) is the output.  a fp32 [M, K] (quantised here), rows block_q8_0 [N, K/32*34] -> fp32 [M, N]."""
    a = np.ascontiguousarray(a, np.float32)
    m, k = a.shape
    aq, ad = quantize_act(a)
    wq, wd = split(rows, k)
    nch = k // 32
    isum = np.einsum("mcj,ncj->cmn", aq.reshape(m, nch, 32).astype(np.int64), wq.reshape(-1, nch, 32).astype(np.int64))
    t = (ad.T[:, :, None] * wd.T[:, None, :]).astype(np.float32)                       # [nch, M, N]
    acc = np.zeros((32, m, wq.shape[0]), np.float32)
    for j in range(-(-nch // 32)):
        c0, c1 = 32 * j, min(32 * j + 32, nch)
        acc[:c1 - c0] = _fmaf(isum[c0:c1].astype(np.float32), t[c0:c1], acc[:c1 - c0])
    out = oracle.warp_butterfly(acc)
    return (out, acc) if lanes else out


def imma_stated(a, rows, ksplit, cols=None):
    """The integer tensor-core GEMM on Q8_0 weights (gemm_imma_kernel, DESIGN.md section 4.3) with K split into ksplit slice ranges:
    K is cut into slices of 256, split s takes slices [S s / ksplit, S (s + 1) / ksplit).  Inside a split, per 32-block b in
    order: acc = fmaf(isum_b, fp32(a_d * w_d), acc) from +0 (isum_b exact).  One split is the result; several are summed in split
    order in fp32 from +0.  a fp32 [M, K] (quantised here), rows block_q8_0 [N, K/32*34]; cols: the weight rows to restate."""
    a = np.ascontiguousarray(a, np.float32)
    m, k = a.shape
    aq, ad = quantize_act(a)
    wq, wd = split(rows, k)
    if cols is not None:
        wq, wd = wq[cols], wd[cols]
    nb = k // 32
    isum = np.einsum("mbj,nbj->bmn", aq.reshape(m, nb, 32).astype(np.int64), wq.reshape(-1, nb, 32).astype(np.int64))
    t = (ad.T[:, :, None] * wd.T[:, None, :]).astype(np.float32)                       # [nb, M, N']
    nsl = -(-k // 256)
    parts = []
    for sp in range(ksplit):
        b0, b1 = (nsl * sp // ksplit) * 8, min((nsl * (sp + 1) // ksplit) * 8, nb)
        acc = np.zeros(isum.shape[1:], np.float32)
        for b in range(b0, b1):
            acc = _fmaf(isum[b].astype(np.float32), t[b], acc)
        parts.append(acc)
    if ksplit == 1:
        return parts[0]
    out = np.zeros_like(parts[0])
    for p in parts:
        out = (out + p).astype(np.float32)
    return out


def imma_split_of(got, a, rows, cols):
    """the split count in 1..16 whose imma_stated equals got [M, len(cols)] bit for bit, or None"""
    gb = np.ascontiguousarray(got, np.float32).view(np.uint32)
    for ks in range(1, 17):
        if np.array_equal(np.ascontiguousarray(imma_stated(a, rows, ks, cols)).view(np.uint32), gb):
            return ks
    return None


class OracleLlamaQ8(OracleLlama):
    """The CPU graph of oracle/llama_model.py with Q8_0 rows for every matmul (layers and lm_head)"""

    def __init__(self, hp, tok_embd, out_norm, output_rows, layers):
        super().__init__(hp, tok_embd, out_norm, output_rows, layers, fmt="q8_0")

    @staticmethod
    def _mm(rows, a):
        return mul_mat(rows, a)


class RefNeLlamaQ8(oracle.RefNeLlama):
    """The reference's own graph engine with NE_TYPE_Q8_0 weight tensors (ne_mul_mat -> ne_vec_dot_q8_0_q8_0)"""

    NE_TYPE_Q4_0 = NE_TYPE_Q8_0  # the weight type RefNeLlama's constructor hands to the engine


def write_gguf(path, hp, tok_rows, out_norm, out_rows, layers):
    """A llama GGUF file with every 2-D tensor Q8_0 (token_embd.weight included), as llama.cpp writes a "Q8_0" model.
    hp: n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx, norm_eps; layers as tests/llama_models.py keeps them."""
    import gguf
    w = gguf.GGUFWriter(path, "llama")
    w.add_context_length(hp["n_ctx"])
    w.add_embedding_length(hp["n_embd"])
    w.add_block_count(hp["n_layer"])
    w.add_feed_forward_length(hp["n_ff"])
    w.add_head_count(hp["n_head"])
    w.add_head_count_kv(hp["n_head_kv"])
    w.add_layer_norm_rms_eps(hp["norm_eps"])
    w.add_rope_freq_base(hp.get("rope_theta", 10000.0))
    T = gguf.GGMLQuantizationType
    w.add_tensor("token_embd.weight", tok_rows, raw_dtype=T.Q8_0)
    w.add_tensor("output_norm.weight", np.asarray(out_norm, np.float32))
    w.add_tensor("output.weight", out_rows, raw_dtype=T.Q8_0)
    names = dict(wq="attn_q", wk="attn_k", wv="attn_v", wo="attn_output", w1="ffn_gate", w2="ffn_down", w3="ffn_up")
    for il, L in enumerate(layers):
        w.add_tensor(f"blk.{il}.attn_norm.weight", np.asarray(L["attn_norm"], np.float32))
        w.add_tensor(f"blk.{il}.ffn_norm.weight", np.asarray(L["ffn_norm"], np.float32))
        for ours, g in names.items():
            w.add_tensor(f"blk.{il}.{g}.weight", L[ours], raw_dtype=T.Q8_0)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()


def toy(seed=5, n_head=4, n_head_kv=4, n_layer=2, n_ctx=48):
    """the toy Llama of tests/llama_models.py (vocab 320, n_embd 256, n_ff 512) with Q8_0 layers and a Q8_0 lm_head; also
    returns the Q8_0 rows of the embedding table, whose dequantised values are the model's fp32 table"""
    rng = np.random.default_rng(seed)
    hp = lm._hparams(320, 256, n_head, n_head_kv, n_layer, 512, n_ctx)
    E, V = 256, 320

    def w(n, k):
        return quantize_weights(rng.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32))

    tok_rows = quantize_weights(rng.normal(0, 1, (V, E)).astype(np.float32))
    tok = dequantize(tok_rows, E)
    out_norm = lm._norm(rng, E)
    layers = []
    for _ in range(n_layer):
        L = dict(attn_norm=lm._norm(rng, E), ffn_norm=lm._norm(rng, E))
        for name, (n, k) in lm._shapes(hp).items():
            L[name] = w(n, k)
        layers.append(L)
    m = Q8Llama(hp, tok, out_norm, w(V, E), layers)
    m.tok_jig = lm._moved(tok, (np.random.default_rng(99).integers(0, 2, tok.shape) * 2 - 1).astype(np.int32))
    return m, tok_rows


class Q8Llama(lm.Llama):
    """tests/llama_models.Llama with Q8_0 payloads everywhere: its CPU graph is OracleLlamaQ8, its reference RefNeLlamaQ8"""

    def __init__(self, hp, tok, out_norm, out_rows, layers):
        super().__init__(hp, tok, out_norm, out_rows, layers, out_fmt="q8_0", fmt="q8_0")

    def graph(self, jig=False):
        return OracleLlamaQ8(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers)

    def reference(self, jig=False):
        if oracle.ref_ne() is None:
            return self.graph(jig)
        return RefNeLlamaQ8(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers)


def llama2_7b_shaped(rng, n_ctx):
    """tests/llama_models.llama2_7b_shaped's model (two layers of Llama-2-7B's shapes, vocab 32000) with Q8_0 weights"""
    hp = lm._hparams(32000, 4096, 32, 32, 2, 11008, n_ctx)
    E, V = 4096, 32000

    def qw(n, k):
        return quantize_weights(rng.standard_normal((n, k), dtype=np.float32) * np.float32(1.0 / np.sqrt(k)))

    tok = rng.standard_normal((V, E), dtype=np.float32)
    out_norm = lm._norm(rng, E)
    layers = []
    for _ in range(hp["n_layer"]):
        L = dict(attn_norm=lm._norm(rng, E), ffn_norm=lm._norm(rng, E))
        for name, (n, k) in lm._shapes(hp).items():
            L[name] = qw(n, k)
        layers.append(L)
    return Q8Llama(hp, tok, out_norm, qw(V, E), layers)

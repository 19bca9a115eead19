"""oracle/qwen2.py -- TEST INFRASTRUCTURE ONLY.  The version-2 graph of the reference's qwen architecture (models/qwen/qwen.cpp;
Qwen1.5 / Qwen2 / Qwen2.5), restated on top of oracle/llama_model.py, and the reference's own engine running it.

  rope_neox_rows     ne_rope_inplace(mode 2), the NeoX rotation of the pairs (i, i + hd/2) (core/ne_layers.c:9396-9423)
  interleave_perm    the per-head order P of the Qwen2 eval step: (P x)[2i] = x[i], (P x)[2i + 1] = x[i + hd/2]
  OracleQwen2        OracleLlama with q / k / v biases (ne_add(ne_repeat(bias), cur), qwen.cpp:193-203) and NeoX RoPE (:206-209),
                     in the reference's natural head order; qwen_ff's up * silu(gate) is the same fp32 product as Llama's FFN
  RefNeQwen2         the reference's engine running that graph (oracle/ref_ne_qwen2.c -> oracle/_ref/libref_ne_qwen2.so, built by
                     Makefile.qwen2 where the reference sources are present)

Parity status: PINNED (tests/test_qwen2_cpu.py): rope_neox_rows and OracleQwen2 bit for bit against the reference's engine, or
against tests/golden/qwen2_tiny.npz where it is not built.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

import oracle
from oracle.llama_model import OracleLlama, _fmaf, _libm

_HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference"


def rope_neox_rows(x, pos, hd, freq_base=10000.0, rope_scale=1.0):
    """ne_rope_inplace(mode 2) of x [T, n_head, hd] with row t at position pos[t] (ne_layers.c:9396-9423): theta_base = p * freq_scale,
    then per pair i (dims i and i + hd/2) angle = freq_scale * theta_base (rope_yarn) and theta_base *= theta_scale in fp32;
    dst_i = x_i*cos - x_{i+hd/2}*sin, dst_{i+hd/2} = x_i*sin + x_{i+hd/2}*cos, with the default build's contractions
    fma(x0, cos, -(x1*sin)) and fma(x0, sin, x1*cos) as in llama_model.rope_mode0_rows.  The pair's angle sequence is mode 0's for
    the pair (2i, 2i+1), so at rope_scale 1 rope_mode0_rows(P x) == P rope_neox_rows(x) (interleave_heads)."""
    x = np.asarray(x, np.float32)
    pos = np.asarray(pos, np.int64).reshape(-1)
    assert x.shape[0] == pos.size and x.shape[-1] == hd
    theta_scale = np.float32(_libm.powf(float(np.float32(freq_base)), float(np.float32(-2.0) / np.float32(hd))))
    freq_scale = np.float32(1.0) / np.float32(rope_scale)
    upos, inv = np.unique(pos, return_inverse=True)
    th = np.empty((upos.size, hd // 2), np.float32)
    theta = (upos.astype(np.float32) * freq_scale).astype(np.float32)
    for i in range(hd // 2):
        th[:, i] = freq_scale * theta
        theta = (theta * theta_scale).astype(np.float32)
    cosf, sinf = _libm.cosf, _libm.sinf
    c = np.array([cosf(float(t)) for t in th.ravel()], np.float32).reshape(th.shape)[inv][:, None, :]
    s = np.array([sinf(float(t)) for t in th.ravel()], np.float32).reshape(th.shape)[inv][:, None, :]
    x0, x1 = x[..., :hd // 2], x[..., hd // 2:]
    out = np.empty_like(x)
    out[..., :hd // 2] = _fmaf(x0, c, -(x1 * s))
    out[..., hd // 2:] = _fmaf(x0, s, x1 * c)
    return out


def interleave_perm(hd):
    """the interleaved head order P of the Qwen2 eval step as an index array: (P x)[j] = x[interleave_perm(hd)[j]]"""
    j = np.arange(hd)
    return np.where(j % 2 == 0, j // 2, hd // 2 + j // 2)


def interleave_heads(x, hd):
    """P applied to every head of x's last axis (its length a multiple of hd)"""
    x = np.asarray(x)
    n = x.shape[-1]
    idx = (np.arange(n) // hd * hd) + interleave_perm(hd)[np.arange(n) % hd]
    return x[..., idx]


class OracleQwen2(OracleLlama):
    """OracleLlama's constructor arguments; the layers also hold bq, bk, bv (f32 [n_embd] / [kvd] / [kvd]).  OracleLlama.eval
    computes each projection with _mm and rotates q and k with _rope: the overrides add the layer's bias to its q / k / v projection
    and rotate NeoX-style."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self._bias = {}
        for L in self.layers:
            for w, b in (("wq", "bq"), ("wk", "bk"), ("wv", "bv")):
                self._bias[id(L[w])] = L[b]

    def _mm(self, rows, a):
        out = OracleLlama._mm(rows, a)
        b = self._bias.get(id(rows))
        return out if b is None else out + b

    def _rope(self, x, pos):
        return rope_neox_rows(x[None], [pos], self.hd, self.hp.get("rope_theta", 10000.0), self.hp.get("rope_scale", 1.0))[0]


# ---------------------------------------------------------------------------------------------------- the reference's engine
_lib = None


def ref_ne_qwen2():
    """oracle/_ref/libref_ne_qwen2.so (built here when the reference sources are present) or None"""
    global _lib
    if _lib is None:
        p = os.path.join(_HERE, "_ref", "libref_ne_qwen2.so")
        if os.path.isdir(os.path.join(REF, "neural_speed")):
            try:
                subprocess.run(["make", "-C", _HERE, "-s", "-f", "Makefile.qwen2", f"REF={REF}"], check=True)
            except Exception:
                pass
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        L.ref_ne_rope_neox.restype = None
        L.ref_ne_rope_neox.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float]
        L.ref_ne_rope.restype = None
        L.ref_ne_rope.argtypes = L.ref_ne_rope_neox.argtypes
        L.ref_ne_qwen2_create.restype = C.c_void_p
        L.ref_ne_qwen2_create.argtypes = [C.c_int] * 7 + [C.c_float] * 3
        L.ref_ne_qwen2_set.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
        L.ref_ne_qwen2_set_bias.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
        L.ref_ne_qwen2_eval.restype = None
        L.ref_ne_qwen2_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.ref_ne_qwen2_free.restype = None
        L.ref_ne_qwen2_free.argtypes = [C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def ref_rope(x, hd, n_past, freq_base, neox):
    """the engine's rope of x [T, n_head, hd] fp32 at positions n_past .., mode 2 (neox) or 0; a new array"""
    y = np.ascontiguousarray(x, np.float32).copy()
    L = ref_ne_qwen2()
    (L.ref_ne_rope_neox if neox else L.ref_ne_rope)(_p(y), hd, y.shape[1], y.shape[0], n_past, freq_base, 1.0)
    return y


class RefNeQwen2:
    """A Qwen2 model (OracleQwen2's constructor arguments, Q4_0 weights, the biases in the natural head order) evaluated by the
    reference's engine.  Only available where oracle/_ref/libref_ne_qwen2.so is built."""

    NAMES = ["attn_norm", "wq", "wk", "wv", "wo", "ffn_norm", "w1", "w2", "w3"]

    def __init__(self, hp, tok_embd, out_norm, output_rows, layers):
        L = ref_ne_qwen2()
        if L is None:
            raise RuntimeError("oracle/_ref/libref_ne_qwen2.so not built")
        self.L, self.n_vocab = L, hp["n_vocab"]
        self.h = C.c_void_p(L.ref_ne_qwen2_create(hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["n_ff"],
                                                  hp["n_ctx"], hp.get("norm_eps", 1e-6), hp.get("rope_theta", 10000.0),
                                                  hp.get("rope_scale", 1.0)))

        def put(layer, which, arr, dt):
            a = np.ascontiguousarray(arr, dt)
            assert L.ref_ne_qwen2_set(self.h, layer, which, _p(a), a.nbytes) == 0, (layer, which, a.nbytes)

        put(0, -1, tok_embd, np.float32)
        put(0, -2, out_norm, np.float32)
        put(0, -3, output_rows, np.uint8)
        for il, lay in enumerate(layers):
            for j, name in enumerate(self.NAMES):
                put(il, j, lay[name], np.float32 if "norm" in name else np.uint8)
            for j, name in enumerate(("bq", "bk", "bv")):
                b = np.ascontiguousarray(lay[name], np.float32)
                assert L.ref_ne_qwen2_set_bias(self.h, il, j, _p(b), b.nbytes) == 0, (il, name)

    def eval(self, tokens, n_past):
        t = np.ascontiguousarray(tokens, np.int32)
        logits = np.zeros(self.n_vocab, np.float32)
        self.L.ref_ne_qwen2_eval(self.h, _p(t), t.size, n_past, _p(logits))
        return logits

    def close(self):
        if self.h:
            self.L.ref_ne_qwen2_free(self.h)
            self.h = None

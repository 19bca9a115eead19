"""oracle/streaming.py -- TEST INFRASTRUCTURE ONLY.  The shift-RoPE-K ("StreamingLLM") ring of the reference, for the fp16 KV cache
and batch 1, restated on top of oracle/llama_model.py, and the reference's own engine running the same graphs.

  shift_table        kv_self.cossin (models/model_utils/model_utils.cpp:165-192)
  rope_shift_f16     ne_rope_shift_inplace on the fp16 K cache (core/ne_layers.c:9495-9532)
  OracleLlamaRing    OracleLlama with the ring of models/llama/llama.cpp:102-107, 351-354, 430-470
  RefNeLlamaRing     the reference's engine running that graph (oracle/ref_ne_ring.c -> oracle/_ref/libref_ne_ring.so, built by
                     Makefile.ring where the reference sources are present)
  check              golden.check against tests/golden/streaming_digests.json (bit-exact with the engine where it is built, the
                     stored digests of its results elsewhere; NS_RECORD_GOLDEN=1 rewrites them)

Parity status: PINNED (tests/test_streaming_cpu.py): the table, the shift and whole toy-model ring runs, bit for bit.
"""
from __future__ import annotations

import atexit
import ctypes as C
import json
import os
import subprocess

import numpy as np

import oracle
from oracle import golden
from oracle.llama_model import OracleLlama, _f16, _fmaf, _libm, soft_max_f16table, vec_dot_f16_rows

_HERE = os.path.dirname(os.path.abspath(__file__))
DIGESTS = os.path.join(os.path.dirname(_HERE), "tests", "golden", "streaming_digests.json")
REF = "/root/reference"


def shift_table(hd, freq_base=10000.0):
    """kv_self.cossin of the shift-RoPE-K mode (model_utils.cpp:165-192 with freq_scale 1): theta = -1, then theta *= theta_scale
    per pair in fp32, theta_scale = powf(freq_base, -2 / hd); cosf / sinf from libm rounded to fp16.  -> [hd] fp16 (cos, sin)"""
    theta_scale = np.float32(_libm.powf(float(np.float32(freq_base)), float(np.float32(-2.0) / np.float32(hd))))
    theta = np.float32(-1.0)
    out = np.empty(hd, np.float32)
    for i in range(0, hd, 2):
        out[i], out[i + 1] = _libm.cosf(float(theta)), _libm.sinf(float(theta))
        theta = np.float32(theta * theta_scale)
    return out.astype(np.float16)


def rope_shift_f16(kc, n_keep, table):
    """ne_rope_shift_inplace on the fp16 K cache (ne_layers.c:9507-9529): every row of kc [..., slots, hd] at or past slot n_keep
    shifted one position back, dst0 = x0*cos - x1*sin, dst1 = x1*cos + x0*sin in fp32 from fp16 x and table, rounded to fp16.
    The reference's build (-O3 -mfma) contracts these to fma(x0, cos, -(x1*sin)) and fma(x1, cos, x0*sin); the products of two
    fp16 values are exact in fp32, so every contraction rounds once and gives the same bits (pinned against the engine)."""
    kc = np.asarray(kc, np.float16)
    out = kc.copy()
    x = kc[..., n_keep:, :].astype(np.float32)
    t = np.asarray(table, np.float16).astype(np.float32)
    c, s = t[0::2], t[1::2]
    x0, x1 = x[..., 0::2], x[..., 1::2]
    y = np.empty_like(x)
    y[..., 0::2] = _fmaf(x0, c, -(x1 * s))
    y[..., 1::2] = _fmaf(x1, c, x0 * s)
    out[..., n_keep:, :] = y.astype(np.float16)
    return out


def ring_slot(n_total, n_ctx, n_keep):
    """the cache slot of the token evaluated after n_total others: n_total until the cache is full, then the sinks [0, n_keep) stay
    and slots n_keep .. n_ctx - 1 are reused in token order (the n_past of application/main_run.cpp:474-494)"""
    return n_total if n_total < n_ctx else n_keep + (n_total - n_ctx) % (n_ctx - n_keep)


class OracleLlamaRing(OracleLlama):
    """OracleLlama in the ring mode of the reference's shift-RoPE-K inference with n_keep sink slots.  eval's n_past is n_total,
    the number of tokens evaluated so far; one-token steps may pass n_ctx.  Until the cache is full a step is OracleLlama.eval
    (the reference drops the mask for one new token, where it has no effect).  After that (llama.cpp:351-354, 430-470): q is
    rotated at n_ctx - 1, the new k at n_ctx and stored with v in ring_slot(), every cached key at or past n_keep is shifted back
    by rope_shift_f16 (the write comes first), and attention covers all n_ctx slots unmasked."""

    def __init__(self, hp: dict, tok_embd, out_norm, output_rows, layers, n_keep, fmt="q4_0"):
        super().__init__(hp, tok_embd, out_norm, output_rows, layers, fmt=fmt)
        assert 0 <= n_keep < hp["n_ctx"] and hp.get("rope_scale", 1.0) == 1.0
        self.n_keep = n_keep
        self.table = shift_table(self.hd, hp.get("rope_theta", 10000.0))

    def eval(self, tokens, n_past):
        hp = self.hp
        n_ctx = hp["n_ctx"]
        if n_past < n_ctx:
            assert n_past + len(tokens) <= n_ctx, "past n_ctx: one token per step"
            return super().eval(tokens, n_past)
        assert len(tokens) == 1, "past n_ctx: one token per step"
        E, H, HK, hd = hp["n_embd"], hp["n_head"], hp["n_head_kv"], self.hd
        s = ring_slot(n_past, n_ctx, self.n_keep)
        x = self.tok_embd[np.asarray(tokens)].astype(np.float32)
        scale = np.float32(1.0) / np.float32(np.sqrt(np.float32(hd)))
        for il, L in enumerate(self.layers):
            cur = self._rms(x, L["attn_norm"])
            q = self._rope(self._mm(L["wq"], cur).reshape(H, hd), n_ctx - 1)
            k = self._mm(L["wk"], cur).reshape(HK, hd)
            v = self._mm(L["wv"], cur).reshape(HK, hd)
            self.kc[il, :, s, :] = self._rope(k, n_ctx).astype(np.float16)
            self.vc[il, :, s, :] = v.astype(np.float16)
            self.kc[il] = rope_shift_f16(self.kc[il], self.n_keep, self.table)
            attn = np.zeros((1, H, hd), np.float32)
            for h in range(H):
                hk = h // (H // HK)
                sc = vec_dot_f16_rows(self.kc[il, hk].astype(np.float32), _f16(q[h])) * scale
                p = soft_max_f16table(sc)
                vt = np.ascontiguousarray(self.vc[il, hk].astype(np.float32).T)
                attn[0, h] = vec_dot_f16_rows(vt, _f16(p))
            inp_ff = self._mm(L["wo"], attn.reshape(1, E)) + x
            cur = self._rms(inp_ff, L["ffn_norm"])
            g = self._mm(L["w1"], cur)
            silu = np.array([[oracle.lib().orc_silu(float(z)) for z in row] for row in g], np.float32)
            x = self._mm(L["w2"], silu * self._mm(L["w3"], cur)) + inp_ff
        last = self._rms(x[-1:], self.out_norm)
        if self.out_fmt == "q6_K":
            return oracle.mul_mat_q6_K_f32(self.output_rows, last)[0]
        return self._mm(self.output_rows, last)[0]


# ---------------------------------------------------------------------------------------------------- the reference's engine
_ring = None


def ref_ne_ring():
    """oracle/_ref/libref_ne_ring.so (built here when the reference sources are present) or None"""
    global _ring
    if _ring is None:
        p = os.path.join(_HERE, "_ref", "libref_ne_ring.so")
        if os.path.isdir(os.path.join(REF, "neural_speed")):
            try:
                subprocess.run(["make", "-C", _HERE, "-s", "-f", "Makefile.ring", f"REF={REF}"], check=True)
            except Exception:
                pass
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        oracle._bind_llama(L)
        L.ref_ne_llama_eval_ring.restype = None
        L.ref_ne_llama_eval_ring.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.ref_ne_rope_shift.restype = None
        L.ref_ne_rope_shift.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_float, C.c_float]
        _ring = L
    return _ring


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def ref_rope_shift(kc, n_keep, table, freq_base=10000.0):
    """the engine's shift of kc [n_head][slots][hd] fp16 (its layout: [slots][n_head][hd]); table None: the op's own table"""
    k = np.ascontiguousarray(np.asarray(kc, np.float16).transpose(1, 0, 2))
    H, S, hd = kc.shape
    t = None if table is None else np.ascontiguousarray(table, np.float16)
    ref_ne_ring().ref_ne_rope_shift(_p(k), hd, H, S, n_keep, None if t is None else _p(t), freq_base, 1.0)
    return k.transpose(1, 0, 2)


class RefNeLlamaRing:
    """A Llama model (OracleLlama's constructor arguments, Q4_0 weights) evaluated by the reference's engine in shift-RoPE-K mode
    with n_keep sink slots.  eval(tokens, n_total) as OracleLlamaRing; the cache slot passed to the graph is ring_slot()."""

    NAMES = ["attn_norm", "wq", "wk", "wv", "wo", "ffn_norm", "w1", "w2", "w3"]
    NE_TYPE_Q4_0 = 2  # core/data_types.h:32-55

    def __init__(self, hp, tok_embd, out_norm, output_rows, layers, n_keep, table=None):
        """table: the fp16 shift table handed to the graph as kv_self.cossin (None: the op builds its own)"""
        L = ref_ne_ring()
        if L is None:
            raise RuntimeError("oracle/_ref/libref_ne_ring.so not built")
        self.L, self.n_vocab, self.n_ctx, self.n_keep = L, hp["n_vocab"], hp["n_ctx"], n_keep
        self.table = None if table is None else np.ascontiguousarray(table, np.float16)
        self.h = C.c_void_p(L.ref_ne_llama_create_ex(hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["n_ff"],
                                                     hp["n_ctx"], hp.get("norm_eps", 1e-6), hp.get("rope_theta", 10000.0),
                                                     hp.get("rope_scale", 1.0), self.NE_TYPE_Q4_0, None, 0, 1))

        def put(layer, which, arr, dt):
            a = np.ascontiguousarray(arr, dt)
            assert L.ref_ne_llama_set(self.h, layer, which, _p(a), a.nbytes) == 0, (layer, which, a.nbytes)

        put(0, -1, tok_embd, np.float32)
        put(0, -2, out_norm, np.float32)
        put(0, -3, output_rows, np.uint8)
        for il, lay in enumerate(layers):
            for j, name in enumerate(self.NAMES):
                put(il, j, lay[name], np.float32 if "norm" in name else np.uint8)

    def eval(self, tokens, n_total):
        t = np.ascontiguousarray(tokens, np.int32)
        logits = np.zeros(self.n_vocab, np.float32)
        self.L.ref_ne_llama_eval_ring(self.h, _p(t), t.size, ring_slot(n_total, self.n_ctx, self.n_keep), n_total, self.n_keep,
                                      None if self.table is None else _p(self.table), _p(logits))
        return logits

    def close(self):
        if self.h:
            self.L.ref_ne_llama_free(self.h)
            self.h = None


# ---------------------------------------------------------------------------------------------------- stored digests
_stored = None
_recorded = {}


def _write():
    merged = dict(_load())
    merged.update(_recorded)
    with open(DIGESTS, "w") as f:
        json.dump(dict(sorted(merged.items())), f, indent=0)
        f.write("\n")


def _load():
    global _stored
    if _stored is None:
        try:
            with open(DIGESTS) as f:
                _stored = json.load(f)
        except FileNotFoundError:
            _stored = {}
    return _stored


def check(key: str, ours, ref_fn, have_ref: bool):
    """golden.check's rule for tests/golden/streaming_digests.json: assert ours == the engine's result (computed where the engine is
    built, else known by its digest); return that result"""
    ours = np.ascontiguousarray(ours)
    if have_ref:
        want = np.ascontiguousarray(ref_fn())
        assert ours.dtype == want.dtype and ours.shape == want.shape, key
        assert np.array_equal(ours, want, equal_nan=ours.dtype.kind in "fc"), key
        if os.environ.get("NS_RECORD_GOLDEN"):
            if not _recorded:
                atexit.register(_write)
            _recorded[key] = golden.digest(want)
        return want
    stored = _load()
    assert key in stored, f"{key}: no stored reference digest in {DIGESTS}"
    assert golden.digest(ours) == stored[key], key
    return ours

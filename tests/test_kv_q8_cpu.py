"""The Q8_0 KV cache's stated arithmetic on the CPU (include/ns_b200.h, NS_KV_Q8_0; neural_speed_b200/csrc/kv_cache.cuh).

Every appended row r -- K after RoPE, V as projected, fp32 -- is stored as ggml Q8_0 blocks of 32 (the runtime quantize_row_q8_0 the
NS_COMP_Q8_0 matmuls use), and every kernel reads fp16(q * d) where it read an fp16 value.  So a Q8_0 engine is the CPU graph
with every appended row replaced by fp16(dequantize_q8_0(quantize_q8_0(r))): `OracleQ8` is that graph, OracleLlama with its two
cache arrays behind a store that takes the fp32 row the graph just computed instead of its fp16 rounding."""
import numpy as np

import neural_speed_b200 as ns
import oracle
from llama_models import toy
from oracle.llama_model import OracleLlama


def q8_round_trip(rows):
    """fp16(dequantize_q8_0(quantize_q8_0(r))) of every row of rows [..., hd] fp32, as float16"""
    r = np.ascontiguousarray(rows, np.float32)
    flat = r.reshape(-1, r.shape[-1])
    deq = oracle.dequantize_q8_0(oracle.quantize_q8_0(flat, variant="runtime"), flat.shape[1])
    return deq.astype(np.float16).reshape(r.shape)


class _Store:
    """an fp16 cache array whose row stores take the graph's fp32 row (`source()`), checked against the fp16 value the graph
    would have stored, through the Q8_0 round trip; reads are the array's"""

    def __init__(self, a, source, log):
        self.a, self.source, self.log = a, source, log

    def __getitem__(self, key):
        return self.a[key]

    def __setitem__(self, key, value):
        r = self.source()
        assert np.array_equal(r.astype(np.float16).view(np.uint16), np.asarray(value, np.float16).view(np.uint16))
        stored = q8_round_trip(r)
        self.a[key] = stored
        self.log.append((r.copy(), stored))

    @property
    def shape(self):
        return self.a.shape


class OracleQ8(OracleLlama):
    """OracleLlama with a Q8_0 KV cache.  OracleLlama.eval stores rope(k[t]) and v[t] (computed by _rope and _mm just before each
    store); the overrides hand the fp32 rows to the stores."""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.log = []
        self._rot = None
        self._v, self._vt = None, 0
        self._wv = {id(L["wv"]) for L in self.layers}
        self.kc = _Store(self.kc, lambda: self._rot, self.log)
        self.vc = _Store(self.vc, self._next_v, self.log)

    def _next_v(self):
        r = self._v[self._vt]
        self._vt += 1
        return r

    def _rope(self, x, pos):
        self._rot = super()._rope(x, pos)
        return self._rot

    def _mm(self, rows, a):
        out = OracleLlama._mm(rows, a)
        if id(rows) in self._wv:  # this layer's V rows, stored in token order
            self._v, self._vt = out.reshape(out.shape[0], self.hp["n_head_kv"], self.hd), 0
        return out


def graph_q8(model, jig=False):
    """the toy model's CPU graph with a Q8_0 KV cache (llama_models.Llama.graph's arguments)"""
    return OracleQ8(model.hp, model.tok_jig if jig else model.tok, model.out_norm, model.out_rows, model.layers, fmt=model.out_fmt)


def test_every_stored_row_is_the_round_trip_of_the_row_computed():
    m = toy(4, 1, seed=1, n_ctx=24)
    g = graph_q8(m)
    rng = np.random.default_rng(5)
    prompt = rng.integers(0, 320, 6).tolist()
    g.eval(prompt, 0)
    g.eval([7], 6)
    hd, HK = g.hd, m.hp["n_head_kv"]
    n_layer = m.hp["n_layer"]
    assert len(g.log) == 2 * n_layer * 7  # K and V of 7 positions per layer
    for r, stored in g.log:
        assert r.shape == (HK, hd) and r.dtype == np.float32
        assert np.array_equal(stored.view(np.uint16), q8_round_trip(r).view(np.uint16))
    # what the cache holds is what was stored, and it differs from the fp16 rounding of the same rows
    kc = g.kc.a
    assert np.array_equal(kc[n_layer - 1, :, 6].view(np.uint16), g.log[-2][1].view(np.uint16))
    assert any(not np.array_equal(s, r.astype(np.float16)) for r, s in g.log)


def test_round_trip_is_ggml_q8_0():
    """blocks of 32, d = fp16(amax / 127), codes round-half-even of x * 127 / amax, read back as fp16(q * d)"""
    rng = np.random.default_rng(0)
    x = (rng.standard_normal((5, 128)) * rng.choice([1e-3, 1.0, 50.0], (5, 1))).astype(np.float32)
    x[1, :32] = 0.0  # an all-zero block: d = 0, codes 0
    blocks = oracle.quantize_q8_0(x, variant="runtime").reshape(5, 4, 34)
    d = blocks[:, :, :2].copy().view(np.float16)[..., 0].astype(np.float32)
    q = blocks[:, :, 2:].view(np.int8).astype(np.float32)
    amax = np.abs(x.reshape(5, 4, 32)).max(-1)
    assert np.array_equal(d, (amax / np.float32(127)).astype(np.float16).astype(np.float32))
    assert np.array_equal(q8_round_trip(x), (q * d[..., None]).astype(np.float16).reshape(5, 128))
    assert not q8_round_trip(x)[1, :32].any()


def test_plane_sizes():
    """the layout ns_llama_kv_bytes follows: a code plane of n_ctx x hd bytes and a scale plane of n_ctx x hd / 32 halves, padded
    to a multiple of 8 halves, per (layer, block, kv head), for K and V"""
    for n_ctx, hd, want in [(48, 128, 192), (47, 128, 192), (45, 64, 96), (4096, 128, 16384), (2, 64, 8), (1, 128, 8)]:
        assert ns.kv_d_stride(n_ctx, hd) == want, (n_ctx, hd)
        assert ns.kv_d_stride(n_ctx, hd) * 2 % 16 == 0
    L, S, HK, n_ctx, hd = 32, 32, 32, 4096, 128
    f16 = ns.kv_bytes("f16", L, S, HK, n_ctx, hd)
    q8 = ns.kv_bytes("q8_0", L, S, HK, n_ctx, hd)
    assert f16 == 2 * L * S * HK * n_ctx * hd * 2
    assert q8 == 2 * L * S * HK * (n_ctx * hd + n_ctx * hd // 16)
    assert q8 * 256 == f16 * 136  # 136 B against 256 B per row at head size 128

"""The synthetic Qwen2 models of the Qwen2 eval-step tests.

A Qwen2 model is a Llama model (tests/llama_models.py) with q / k / v biases and NeoX RoPE.  `toy` has the Llama toy's shapes
(vocab 320, n_embd 256, n_ff 512, Q4_0 layers and head) with rope base 1e6 and biases drawn at about the projections' scale;
`qwen2_7b_shaped` has Qwen2-7B's shapes (n_embd 3584, 28 heads over 4 KV heads of 128, n_ff 18944, vocab 151936) with two Q4_0
layers and the full Q4_0 head.  Each has its CPU graph (oracle.qwen2.OracleQwen2), the jig graph of the running bar, the reference
engine where oracle/_ref is built (oracle.qwen2.RefNeQwen2), the device engine loaded through gguf_loader.load_into_engine, and a
Llama twin: the same model with W_q / W_k rows in the interleaved order P and no biases, which a Qwen2 context with zero biases
must reproduce bit for bit."""
import numpy as np

import oracle
from llama_models import _moved, _norm, _shapes
from neural_speed_b200 import gguf_loader
from oracle.qwen2 import OracleQwen2, RefNeQwen2, interleave_perm, ref_ne_qwen2


def row_perm(n, hd):
    """the row order of an [n, k] weight whose output rows are heads of hd: row r of the result is row perm[r]"""
    r = np.arange(n)
    return r // hd * hd + interleave_perm(hd)[r % hd]


class Qwen2:
    tok_jig = None

    def __init__(self, hp, tok, out_norm, out_rows, layers):
        self.hp, self.tok, self.out_norm, self.out_rows, self.layers = hp, tok, out_norm, out_rows, layers

    @property
    def hd(self):
        return self.hp["n_embd"] // self.hp["n_head"]

    def graph(self, jig=False):
        """a fresh CPU graph of the Qwen2 model, on the jig table with jig=True"""
        return OracleQwen2(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers)

    def graph_q8(self, jig=False):
        """the CPU graph with the engine's Q8_0 KV cache (OracleQwen2Q8)"""
        return OracleQwen2Q8(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers)

    def reference(self):
        """the reference's own graph engine where oracle/_ref is built, else the CPU graph (bit-identical to it)"""
        if ref_ne_qwen2() is None:
            return self.graph()
        return RefNeQwen2(self.hp, self.tok, self.out_norm, self.out_rows, self.layers)

    def _model(self, arch, layers):
        return gguf_loader.GGUFLlama(self.hp, self.tok, self.out_norm, ("q4_0", self.out_rows), layers, arch=arch)

    def engine(self, n_seq=1, zero_bias=False):
        """a device Qwen2 engine with every tensor set (biases zeroed with zero_bias), and n_seq KV blocks"""
        layers = []
        for L in self.layers:
            d = {k: (np.zeros_like(v) if zero_bias else v) if k in ("bq", "bk", "bv") else v if k.endswith("norm") else ("q4_0", v)
                 for k, v in L.items()}
            layers.append(d)
        eng = gguf_loader.load_into_engine(self._model("qwen2", layers))
        if n_seq != 1:
            eng.set_sequences(n_seq)
        return eng

    def llama_twin(self, n_seq=1):
        """a device Llama engine of the same model with the W_q / W_k rows in P order, host-permuted, and no biases"""
        hd, layers = self.hd, []
        for L in self.layers:
            d = {k: v if k.endswith("norm") else ("q4_0", v) for k, v in L.items() if k not in ("bq", "bk", "bv")}
            d["wq"] = ("q4_0", np.ascontiguousarray(L["wq"][row_perm(L["wq"].shape[0], hd)]))
            d["wk"] = ("q4_0", np.ascontiguousarray(L["wk"][row_perm(L["wk"].shape[0], hd)]))
            layers.append(d)
        eng = gguf_loader.load_into_engine(self._model("llama", layers))
        if n_seq != 1:
            eng.set_sequences(n_seq)
        return eng


def _hparams(n_vocab, n_embd, n_head, n_head_kv, n_layer, n_ff, n_ctx):
    return dict(n_vocab=n_vocab, n_embd=n_embd, n_head=n_head, n_head_kv=n_head_kv, n_layer=n_layer, n_ff=n_ff, n_ctx=n_ctx,
                norm_eps=1e-6, rope_theta=1000000.0, rope_scale=1.0)


def _biases(rng, hp, scale):
    E = hp["n_embd"]
    kvd = E // hp["n_head"] * hp["n_head_kv"]
    return dict(bq=rng.normal(0, scale, E).astype(np.float32), bk=rng.normal(0, scale, kvd).astype(np.float32),
                bv=rng.normal(0, scale, kvd).astype(np.float32))


def toy(n_head=4, n_head_kv=4, seed=0, n_layer=2, n_ctx=64):
    rng = np.random.default_rng(seed)
    hp = _hparams(320, 256, n_head, n_head_kv, n_layer, 512, n_ctx)
    E, V = 256, 320

    def w(n, k):
        return rng.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32)

    tok = rng.normal(0, 1, (V, E)).astype(np.float32)
    out_norm = _norm(rng, E)
    layers = []
    for _ in range(n_layer):
        L = dict(attn_norm=_norm(rng, E), ffn_norm=_norm(rng, E))
        for name, (n, k) in _shapes(hp).items():
            L[name] = oracle.quantize_q4_0(w(n, k))
        L.update(_biases(rng, hp, 0.5))
        layers.append(L)
    m = Qwen2(hp, tok, out_norm, oracle.quantize_q4_0(w(V, E)), layers)
    m.tok_jig = _moved(tok, (np.random.default_rng(99).integers(0, 2, tok.shape) * 2 - 1).astype(np.int32))
    return m


def qwen2_7b_shaped(rng, n_ctx):
    """Qwen2-7B's shapes, two Q4_0 layers and the full Q4_0 head, drawn from rng"""
    hp = _hparams(151936, 3584, 28, 4, 2, 18944, n_ctx)
    E, V = hp["n_embd"], hp["n_vocab"]

    def qw(n, k):
        return oracle.quantize_q4_0(rng.standard_normal((n, k), dtype=np.float32) * np.float32(1.0 / np.sqrt(k)))

    tok = rng.standard_normal((V, E), dtype=np.float32)
    out_norm = _norm(rng, E)
    layers = []
    for _ in range(hp["n_layer"]):
        L = dict(attn_norm=_norm(rng, E), ffn_norm=_norm(rng, E))
        for name, (n, k) in _shapes(hp).items():
            L[name] = qw(n, k)
        L.update(_biases(rng, hp, 0.5))
        layers.append(L)
    return Qwen2(hp, tok, out_norm, qw(V, E), layers)


class _KStore:
    """a cache array whose row stores take the graph's fp32 row through a Q8_0 round trip in the order `perm` (per head)"""

    def __init__(self, a, source, hd, interleaved):
        self.a, self.source, self.hd, self.interleaved = a, source, hd, interleaved

    def __getitem__(self, key):
        return self.a[key]

    def __setitem__(self, key, value):
        from test_kv_q8_cpu import q8_round_trip
        r = self.source()
        assert np.array_equal(r.astype(np.float16).view(np.uint16), np.asarray(value, np.float16).view(np.uint16))
        if self.interleaved:  # the engine's K rows are in P order: its Q8_0 blocks group P-order elements
            inv = np.argsort(interleave_perm(self.hd))
            self.a[key] = q8_round_trip(r[..., interleave_perm(self.hd)])[..., inv]
        else:
            self.a[key] = q8_round_trip(r)

    @property
    def shape(self):
        return self.a.shape


class OracleQwen2Q8(OracleQwen2):
    """the Qwen2 CPU graph with the engine's Q8_0 KV cache: K after RoPE quantised in blocks of 32 of the P-order row (what the
    engine stores), V as projected (bias added) in natural order, both read back as fp16(q * d)"""

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self._rot = None
        self._v, self._vt = None, 0
        self._wv = {id(L["wv"]) for L in self.layers}
        self.kc = _KStore(self.kc, lambda: self._rot, self.hd, True)
        self.vc = _KStore(self.vc, self._next_v, self.hd, False)

    def _next_v(self):
        r = self._v[self._vt]
        self._vt += 1
        return r

    def _rope(self, x, pos):
        self._rot = super()._rope(x, pos)
        return self._rot

    def _mm(self, rows, a):
        out = super()._mm(rows, a)
        if id(rows) in self._wv:  # this layer's V rows (bias added), stored in token order
            self._v, self._vt = out.reshape(out.shape[0], self.hp["n_head_kv"], self.hd), 0
        return out

"""The synthetic Phi-3 models of the Phi-3 eval-step tests.

A Phi-3 model is a Llama model (tests/llama_models.py) with NeoX RoPE and, for Phi-3-mini, head size 96.  `toy` has heads of 96
(n_embd 96 x n_head), vocab 320, n_ff 512, Q4_0 layers and head, rope base 1e4; `phi3_mini_shaped` has Phi-3-mini's shapes
(n_embd 3072, 32 heads of 96, n_ff 8192, vocab 32064) with two Q4_0 layers and the full Q4_0 head.  Each has its CPU graph
(oracle.phi3.OraclePhi3), the jig graph of the running bar, the reference engine where oracle/_ref is built (oracle.phi3.RefNePhi3),
the device engine loaded through gguf_loader.load_into_engine, and a Llama twin: the same model with W_q / W_k rows in the
interleaved order P, which a Phi-3 context must reproduce bit for bit."""
import numpy as np

import oracle
from llama_models import _hparams, _moved, _norm, _shapes
from neural_speed_b200 import gguf_loader
from oracle.phi3 import OraclePhi3, RefNePhi3, ref_ne_phi3
from qwen2_models import row_perm


class Phi3:
    tok_jig = None

    def __init__(self, hp, tok, out_norm, out_rows, layers):
        self.hp, self.tok, self.out_norm, self.out_rows, self.layers = hp, tok, out_norm, out_rows, layers

    @property
    def hd(self):
        return self.hp["n_embd"] // self.hp["n_head"]

    def graph(self, jig=False):
        """a fresh CPU graph of the Phi-3 model, on the jig table with jig=True"""
        return OraclePhi3(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers)

    def reference(self, jig=False):
        """the reference's own graph engine where oracle/_ref is built, else the CPU graph (bit-identical to it)"""
        if ref_ne_phi3() is None:
            return self.graph(jig)
        return RefNePhi3(self.hp, self.tok_jig if jig else self.tok, self.out_norm, self.out_rows, self.layers)

    def _engine(self, arch, layers, n_seq):
        model = gguf_loader.GGUFLlama(self.hp, self.tok, self.out_norm, ("q4_0", self.out_rows), layers, arch=arch)
        eng = gguf_loader.load_into_engine(model)
        if n_seq != 1:
            eng.set_sequences(n_seq)
        return eng

    def engine(self, n_seq=1):
        """a device Phi-3 engine with every tensor set, and n_seq KV blocks"""
        return self._engine("phi3", [{k: v if k.endswith("norm") else ("q4_0", v) for k, v in L.items()} for L in self.layers], n_seq)

    def llama_twin(self, n_seq=1):
        """a device Llama engine of the same model with the W_q / W_k rows in P order, host-permuted"""
        layers = []
        for L in self.layers:
            d = {k: v if k.endswith("norm") else ("q4_0", v) for k, v in L.items()}
            for name in ("wq", "wk"):
                d[name] = ("q4_0", np.ascontiguousarray(L[name][row_perm(L[name].shape[0], self.hd)]))
            layers.append(d)
        return self._engine("llama", layers, n_seq)


def toy(n_head=4, n_head_kv=4, seed=0, n_layer=2, n_ctx=64, hd=96):
    rng = np.random.default_rng(seed)
    E, V = hd * n_head, 320
    hp = _hparams(V, E, n_head, n_head_kv, n_layer, 512, n_ctx)

    def w(n, k):
        return rng.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32)

    tok = rng.normal(0, 1, (V, E)).astype(np.float32)
    out_norm = _norm(rng, E)
    layers = []
    for _ in range(n_layer):
        L = dict(attn_norm=_norm(rng, E), ffn_norm=_norm(rng, E))
        for name, (n, k) in _shapes(hp).items():
            L[name] = oracle.quantize_q4_0(w(n, k))
        layers.append(L)
    m = Phi3(hp, tok, out_norm, oracle.quantize_q4_0(w(V, E)), layers)
    m.tok_jig = _moved(tok, (np.random.default_rng(99).integers(0, 2, tok.shape) * 2 - 1).astype(np.int32))
    return m


def phi3_mini_shaped(rng, n_ctx, n_layer=2):
    """Phi-3-mini's shapes, n_layer Q4_0 layers and the full Q4_0 head, drawn from rng"""
    hp = _hparams(32064, 3072, 32, 32, n_layer, 8192, n_ctx)
    E, V = hp["n_embd"], hp["n_vocab"]

    def qw(n, k):
        return oracle.quantize_q4_0(rng.standard_normal((n, k), dtype=np.float32) * np.float32(1.0 / np.sqrt(k)))

    tok = rng.standard_normal((V, E), dtype=np.float32)
    out_norm = _norm(rng, E)
    layers = []
    for _ in range(n_layer):
        L = dict(attn_norm=_norm(rng, E), ffn_norm=_norm(rng, E))
        for name, (n, k) in _shapes(hp).items():
            L[name] = qw(n, k)
        layers.append(L)
    return Phi3(hp, tok, out_norm, qw(V, E), layers)

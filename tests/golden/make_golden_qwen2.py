"""Writes tests/golden/qwen2_tiny.npz from the reference's own graph engine (oracle/_ref/libref_ne_qwen2.so; needs the reference sources):

  rope.{hd}.{base}.x / .y   ne_rope_inplace(mode 2) of a [T, 2, hd] input at positions 8180 .. 8191 (ref_ne_rope_neox)
  {kind}.*                  a tiny Qwen2 model, kind "mha" or "gqa" (layers l{il}.*, biases l{il}.bq / bk / bv), and the logits
                            the reference computes for the graph of models/qwen/qwen.cpp (version 2) for a 4-token prompt and
                            three single-token steps (oracle.qwen2.RefNeQwen2)

Run: python tests/golden/make_golden_qwen2.py"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import oracle  # noqa: E402
from oracle.qwen2 import RefNeQwen2, ref_ne_qwen2  # noqa: E402

STEPS = [[1, 40, 7, 91], [13], [55], [2]]
ROPE_POS0, ROPE_T = 8180, 12


def tiny(rm, n_head_kv):
    hp = dict(n_vocab=96, n_embd=128, n_head=2, n_head_kv=n_head_kv, n_layer=2, n_ff=192, n_ctx=16, norm_eps=1e-6,
              rope_theta=1000000.0, rope_scale=1.0)
    E, FF, V = hp["n_embd"], hp["n_ff"], hp["n_vocab"]
    kvd = E // hp["n_head"] * n_head_kv
    qw = lambda n, k: oracle.quantize_q4_0(rm.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32), "ref")
    mdl = dict(tok=rm.normal(0, 1, (V, E)).astype(np.float32), out_norm=rm.uniform(0.5, 1.5, E).astype(np.float32), output=qw(V, E))
    layers = []
    for _ in range(hp["n_layer"]):
        layers.append(dict(attn_norm=rm.uniform(0.5, 1.5, E).astype(np.float32), ffn_norm=rm.uniform(0.5, 1.5, E).astype(np.float32),
                           wq=qw(E, E), wk=qw(kvd, E), wv=qw(kvd, E), wo=qw(E, E), w1=qw(FF, E), w2=qw(E, FF), w3=qw(FF, E),
                           bq=rm.normal(0, 0.5, E).astype(np.float32), bk=rm.normal(0, 0.5, kvd).astype(np.float32),
                           bv=rm.normal(0, 0.5, kvd).astype(np.float32)))
    return hp, mdl, layers


def main():
    ne = ref_ne_qwen2()
    assert ne is not None, "oracle/_ref/libref_ne_qwen2.so is not built"
    out = {}
    rr = np.random.default_rng(77)
    for hd in (64, 128):
        for base in (10000.0, 1000000.0):
            x = rr.standard_normal((ROPE_T, 2, hd)).astype(np.float32)
            y = x.copy()
            ne.ref_ne_rope_neox(y.ctypes.data_as(C.c_void_p), hd, 2, ROPE_T, ROPE_POS0, base, 1.0)
            out[f"rope.{hd}.{int(base)}.x"], out[f"rope.{hd}.{int(base)}.y"] = x, y
    rm = np.random.default_rng(4343)
    for kind, hk in (("mha", 2), ("gqa", 1)):
        hp, mdl, layers = tiny(rm, hk)
        ref = RefNeQwen2(hp, mdl["tok"], mdl["out_norm"], mdl["output"], layers)
        pos = 0
        for i, t in enumerate(STEPS):
            out[f"{kind}.logits{i}"] = ref.eval(t, pos)
            pos += len(t)
        ref.close()
        for k, v in mdl.items():
            out[f"{kind}.{k}"] = v
        for il, L in enumerate(layers):
            for k, v in L.items():
                out[f"{kind}.l{il}.{k}"] = v
        out[f"{kind}.hp"] = np.array([hp[k] for k in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_ff", "n_ctx")], np.int32)
    np.savez_compressed(os.path.join(HERE, "qwen2_tiny.npz"), **out)
    print("wrote qwen2_tiny.npz")


if __name__ == "__main__":
    main()

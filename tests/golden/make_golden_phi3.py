"""Writes tests/golden/phi3_tiny.npz from the reference's own graph engine (oracle/_ref/libref_ne_qwen2.so with zero biases, which
is the op sequence of models/phi/phi3.cpp; needs the reference sources):

  {kind}.*   a tiny Phi-3 model, kind "mha64", "gqa64", "mha96" or "gqa96" (head size 64 or 96; layers l{il}.*), and the logits
             the reference computes for a 4-token prompt and three single-token steps (oracle.phi3.RefNePhi3)

Run: python tests/golden/make_golden_phi3.py"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

import oracle  # noqa: E402
from oracle.phi3 import RefNePhi3, ref_ne_phi3  # noqa: E402

STEPS = [[1, 40, 7, 91], [13], [55], [2]]
KINDS = (("mha64", 64, 2), ("gqa64", 64, 1), ("mha96", 96, 2), ("gqa96", 96, 1))  # (kind, head size, n_head_kv) with 2 heads


def tiny(rm, hd, n_head_kv):
    hp = dict(n_vocab=96, n_embd=2 * hd, n_head=2, n_head_kv=n_head_kv, n_layer=2, n_ff=128, n_ctx=16, norm_eps=1e-5,
              rope_theta=10000.0, rope_scale=1.0)
    E, FF, V = hp["n_embd"], hp["n_ff"], hp["n_vocab"]
    kvd = hd * n_head_kv
    qw = lambda n, k: oracle.quantize_q4_0(rm.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32), "ref")
    mdl = dict(tok=rm.normal(0, 1, (V, E)).astype(np.float32), out_norm=rm.uniform(0.5, 1.5, E).astype(np.float32), output=qw(V, E))
    layers = []
    for _ in range(hp["n_layer"]):
        layers.append(dict(attn_norm=rm.uniform(0.5, 1.5, E).astype(np.float32), ffn_norm=rm.uniform(0.5, 1.5, E).astype(np.float32),
                           wq=qw(E, E), wk=qw(kvd, E), wv=qw(kvd, E), wo=qw(E, E), w1=qw(FF, E), w2=qw(E, FF), w3=qw(FF, E)))
    return hp, mdl, layers


def main():
    assert ref_ne_phi3() is not None, "oracle/_ref/libref_ne_qwen2.so is not built"
    out = {}
    rm = np.random.default_rng(3131)
    for kind, hd, hk in KINDS:
        hp, mdl, layers = tiny(rm, hd, hk)
        ref = RefNePhi3(hp, mdl["tok"], mdl["out_norm"], mdl["output"], layers)
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
    np.savez_compressed(os.path.join(HERE, "phi3_tiny.npz"), **out)
    print("wrote phi3_tiny.npz")


if __name__ == "__main__":
    main()

"""oracle/phi3.py -- TEST INFRASTRUCTURE ONLY.  The graph of the reference's phi3 architecture (models/phi/phi3.cpp; Phi-3-mini /
medium at their native context), restated on top of oracle/qwen2.py, and the reference's own engine running it.

  OraclePhi3     OracleQwen2 without biases at any even head size: RMSNorm, q / k / v projections, NeoX RoPE with n_rot = head
                 size (phi3.cpp:187-188), the non-fused attention over an fp16 KV cache (:253), up * silu(gate) (:322-330)
  RefNePhi3      the reference's engine running that graph: the qwen2 harness (oracle/ref_ne_qwen2.c) with zero biases, whose
                 adds are exact (x + 0 == x), so the op sequence left is the one phi3.cpp builds on the ne_layers.c path

phi3.cpp runs the q / k / v projections as ONE mul_mat over the fused attn_qkv rows and the gate / up projections as one over the
fused ffn_up rows, then views the result.  Each output element of a mul_mat is an independent vec_dot of one weight row with the
(once-quantised) activation row, so the fused matmul and the split ones (OracleLlama's wq / wk / wv, w1 / w3) give the same bits.

Parity status: PINNED (tests/test_phi3_cpu.py): OraclePhi3 bit for bit against RefNePhi3, or against tests/golden/phi3_tiny.npz
where the reference is not built.
"""
from __future__ import annotations

import numpy as np

from oracle.llama_model import OracleLlama
from oracle.qwen2 import RefNeQwen2, ref_ne_qwen2, rope_neox_rows


def _zero_biases(hp, layers):
    E = hp["n_embd"]
    kvd = E // hp["n_head"] * hp["n_head_kv"]
    z = lambda n: np.zeros(n, np.float32)
    return [dict(L, bq=z(E), bk=z(kvd), bv=z(kvd)) for L in layers]


class OraclePhi3(OracleLlama):
    """OracleLlama's constructor arguments: its graph with q and k rotated NeoX-style (OracleQwen2's rotation, without its biases)"""

    def _rope(self, x, pos):
        return rope_neox_rows(x[None], [pos], self.hd, self.hp.get("rope_theta", 10000.0), self.hp.get("rope_scale", 1.0))[0]


def ref_ne_phi3():
    """the qwen2 harness library (oracle/_ref/libref_ne_qwen2.so) or None"""
    return ref_ne_qwen2()


class RefNePhi3(RefNeQwen2):
    """A Phi-3 model (OraclePhi3's constructor arguments, Q4_0 weights) evaluated by the reference's engine.  Only available where
    oracle/_ref/libref_ne_qwen2.so is built."""

    def __init__(self, hp, tok_embd, out_norm, output_rows, layers):
        super().__init__(hp, tok_embd, out_norm, output_rows, _zero_biases(hp, layers))

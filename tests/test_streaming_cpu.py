"""Generation past n_ctx: the StreamingLLM ring of the reference's shift-RoPE-K mode as oracle/streaming.py restates it
(shift_table, rope_shift_f16, OracleLlamaRing), bit for bit against the reference's own graph engine (oracle/ref_ne_ring.c:
core/ne_layers.c through its public API) -- or, where that cannot be built, against the digests of the engine's results in
tests/golden/streaming_digests.json."""
import numpy as np
import pytest

import oracle
from oracle import streaming as sm

N = sm.ref_ne_ring() is not None


def _ref_shift(kc, n_keep, table, base):
    return sm.ref_rope_shift(kc, n_keep, table, base)


@pytest.mark.parametrize("hd", [64, 128])
def test_shift_table(hd):
    """kv_self.cossin (model_utils.cpp:165-192): read out of the engine's own table by shifting rows (1, 0) -> (cos, sin)"""
    for base in (10000.0, 500000.0):
        one = np.zeros((1, 1, hd), np.float16)
        one[..., 0::2] = 1
        sm.check(f"shift_table[{hd}-{base:g}]", sm.shift_table(hd, base),
                     lambda: _ref_shift(one, 0, None, base).reshape(hd), N)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("n_keep", [0, 1, 4])
def test_rope_shift_f16(hd, n_keep):
    """three successive shifts of random fp16 caches, pairs of magnitude 1e-4 up to 6e4 (a rotation keeps them below the fp16
    maximum), with the caller's table and with the op's"""
    r = np.random.default_rng(hd + n_keep)
    base = 10000.0
    table = sm.shift_table(hd, base)
    mag = 10.0 ** r.uniform(-4, np.log10(6e4), (3, 37, hd // 2))
    phi = r.uniform(0, 2 * np.pi, mag.shape)
    kc = np.empty((3, 37, hd), np.float16)
    kc[..., 0::2], kc[..., 1::2] = mag * np.cos(phi), mag * np.sin(phi)
    ours, theirs = kc, kc
    for step in range(3):
        ours = sm.rope_shift_f16(ours, n_keep, table)
        assert np.isfinite(ours.astype(np.float32)).all()
        assert np.array_equal(ours[:, :n_keep].view(np.uint16), kc[:, :n_keep].view(np.uint16)), "sink rows moved"
        prev = theirs
        theirs = sm.check(f"rope_shift_f16[{hd}-{n_keep}-{step}]", ours, lambda: _ref_shift(prev, n_keep, table, base), N)
        if N:  # the op's own table (cossin NULL) gives the same bits
            assert np.array_equal(_ref_shift(prev, n_keep, None, base).view(np.uint16), theirs.view(np.uint16))


def _toy(seed, n_head, n_head_kv, n_ctx):
    r = np.random.default_rng(seed)
    hp = dict(n_vocab=160, n_embd=256, n_head=n_head, n_head_kv=n_head_kv, n_layer=2, n_ff=384, n_ctx=n_ctx, norm_eps=1e-5,
              rope_theta=10000.0, rope_scale=1.0)
    E, FF, V = hp["n_embd"], hp["n_ff"], hp["n_vocab"]
    kvd = E // n_head * n_head_kv
    w = lambda n, k: oracle.quantize_q4_0(r.normal(0, 1.0 / np.sqrt(k), (n, k)).astype(np.float32))
    tok = r.normal(0, 1, (V, E)).astype(np.float32)
    on = r.uniform(0.5, 1.5, E).astype(np.float32)
    layers = [dict(attn_norm=r.uniform(0.5, 1.5, E).astype(np.float32), ffn_norm=r.uniform(0.5, 1.5, E).astype(np.float32),
                   wq=w(E, E), wk=w(kvd, E), wv=w(kvd, E), wo=w(E, E), w1=w(FF, E), w2=w(E, FF), w3=w(FF, E)) for _ in range(2)]
    return hp, tok, on, w(V, E), layers


@pytest.mark.parametrize("n_head,n_head_kv,n_keep", [(4, 4, 4), (4, 2, 1), (8, 2, 0)])
def test_ring_run_end_to_end(n_head, n_head_kv, n_keep):
    """a 5-token prompt, then 3 n_ctx + 3 single-token steps (the ring wraps three times), n_ctx 24, teacher-forced tokens:
    OracleLlama in ring mode == the engine running the shift-RoPE-K graph of llama.cpp, logits at every step"""
    n_ctx = 24
    hp, tok, on, out, layers = _toy(70 + n_head + n_keep, n_head, n_head_kv, n_ctx)
    seq = np.random.default_rng(n_keep).integers(0, hp["n_vocab"], 5 + 3 * n_ctx + 3)
    steps = [(list(seq[:5]), 0)] + [([int(seq[t])], t) for t in range(5, seq.size)]
    orc = sm.OracleLlamaRing(hp, tok, on, out, layers, n_keep)
    ours = np.stack([orc.eval(toks, pos) for toks, pos in steps])

    def theirs():
        ref = sm.RefNeLlamaRing(hp, tok, on, out, layers, n_keep, orc.table)
        try:
            return np.stack([ref.eval(toks, pos) for toks, pos in steps])
        finally:
            ref.close()

    sm.check(f"ring_run[{n_head}-{n_head_kv}-{n_keep}]", ours, theirs, N)

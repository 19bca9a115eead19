"""ggml Q8_0 weights on the CPU: the arithmetic the device is held to, the file readers and the ring GEMV's plans.

* The CPU restatement of ne_vec_dot_q8_0_q8_0 / ne_compute_forward_mul_mat_q_f32 (tests/q8_0_model.py) is bit-identical to the
  reference's own build (oracle/_ref) on random and edge blocks: codes +-127, weight codes -128, all-zero blocks, d = 0 and
  subnormal fp16 d.  Where the reference sources are absent the golden fixture (tests/golden/ggml_q8_0.npz, written by
  tests/golden/make_golden_q8_0.py from that build) holds it instead.
* gguf_loader and ne_loader read Q8_0 tensors into the untouched rows and, for token_embd / 1-D tensors, fp32 tables with
  dequantize_row_q8_0's arithmetic.
* ns_gemv_ring_plan_q8_0 finds a ring plan for every node of Llama-2-7B in plain, QKV, gate/up and fused-norm launches.
"""
import ctypes as C
import hashlib
import os
import struct

import numpy as np
import pytest

import neural_speed_b200 as ns
import oracle
import q8_0_model as q8
from neural_speed_b200 import gguf_loader, ne_loader

HERE = os.path.dirname(os.path.abspath(__file__))
GOLDEN = os.path.join(HERE, "golden", "ggml_q8_0.npz")
# SHA-256 of each array of the fixture as written by tests/golden/make_golden_q8_0.py
DIGESTS = {
    "a": "089e5efbceb725dcf02b310e12809d577d95d43b9dbd273fbd15be406d330539",
    "aq": "c89a9b85eec70a724a99e11114ed3176febc11082ba6bed5cc9ea0c46e403ef9",
    "out": "68ea61b238c9afcd8515ee4944b809ca08cf1f86148649ebe33d583cfdd235f0",
    "w": "9425d8934cd538e5540544aa222c292a1c14304366f07f2965a1208319315b9f",
    "wdq": "d189cc8d2935b9a6ffa2625c9c8afeab6f3a23325860bcb6a4e13a0f8ecf1b6b",
    "wq": "1d8bbefb17ef86034ad5f292484e988fd076ff8c33af52cd0e7d842707f6a75f",
}


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def edge_rows(rng, n, k):
    """Q8_0 weight rows with the edge blocks a file may hold, next to random ones"""
    q = rng.integers(-128, 128, (n, k)).astype(np.int32)
    d = rng.uniform(1e-4, 2e-2, (n, k // 32)).astype(np.float16).astype(np.float32)
    q[0, :32] = 127
    q[0, 32:64] = -127
    q[1, :32] = -128                                   # maddubs sees |w| = 128: still exact
    q[1, 32:64] = np.where(np.arange(32) % 2, -128, 127)
    q[2, :32] = 0                                      # all-zero block
    d[2, 1] = 0.0                                      # d = 0
    d[3, 0] = np.float32(np.float16(6e-8))             # subnormal fp16 d
    d[3, 1] = np.float32(np.float16(2.0 ** -24))
    return q8.join(q, d)


def edge_acts(rng, m, k):
    a = rng.normal(0, 1, (m, k)).astype(np.float32)
    a[0, :32] = 0.0                                    # an all-zero activation block (d = 0)
    a[-1, 32:64] = np.where(np.arange(32) % 2, 1.0, -1.0)  # codes +-127
    return a


def test_golden_fixture_digests_and_cpu_model():
    g = np.load(GOLDEN)
    for name, want in DIGESTS.items():
        assert hashlib.sha256(np.ascontiguousarray(g[name]).tobytes()).hexdigest() == want, name
    k = g["w"].shape[1]
    assert np.array_equal(oracle.quantize_q8_0(g["a"]), g["aq"])                       # quantize_row_q8_0 (x86 body)
    assert np.array_equal(bits(q8.dequantize(g["wq"], k)), bits(g["wdq"]))
    assert np.array_equal(bits(gguf_loader.dequantize_q8_0(g["wq"], k)), bits(g["wdq"]))
    assert np.array_equal(bits(q8.mul_mat(g["wq"], g["a"])), bits(g["out"]))


needs_ref = pytest.mark.skipif(oracle.ref_ggml() is None, reason="oracle/_ref (the reference build) not available")


def ref_dot(wrow, arow, k):
    s = C.c_float()
    oracle.ref_ggml().ref_vec_dot_q8_0_q8_0(C.c_int(k), C.byref(s), np.ascontiguousarray(wrow).ctypes.data_as(C.c_void_p),
                                           np.ascontiguousarray(arow).ctypes.data_as(C.c_void_p))
    return np.float32(s.value)


@needs_ref
@pytest.mark.parametrize("k", [64, 512, 4096])
def test_vec_dot_bitwise_against_reference(k):
    rng = np.random.default_rng(k)
    rows = edge_rows(rng, 8, k)
    a = edge_acts(rng, 3, k)
    aq = oracle.quantize_q8_0(a)
    for n in range(rows.shape[0]):
        for m in range(a.shape[0]):
            assert bits(q8.vec_dot(rows[n], aq[m], k)) == bits(ref_dot(rows[n], aq[m], k)), (n, m)


@needs_ref
def test_mul_mat_bitwise_against_reference():
    rng = np.random.default_rng(11)
    n, k, m = 40, 1024, 4
    rows = np.concatenate([edge_rows(rng, 8, k), q8.quantize_weights(rng.normal(0, 0.02, (n - 8, k)).astype(np.float32))])
    a = edge_acts(rng, m, k)
    got = q8.mul_mat(rows, a)
    aq = oracle.quantize_q8_0(a, "ref", "runtime")
    want = np.array([[ref_dot(rows[j], aq[i], k) for j in range(n)] for i in range(m)], np.float32)
    assert np.array_equal(bits(got), bits(want))


@needs_ref
def test_weight_quantiser_and_dequantiser_against_reference():
    rng = np.random.default_rng(12)
    w = rng.normal(0, 0.05, (16, 512)).astype(np.float32)
    w[0, :32] = 0.0
    rows = q8.quantize_weights(w)
    assert np.array_equal(rows, oracle.quantize_q8_0(w, "ref", "reference"))   # ne_quantize_q8_0's rows
    assert np.array_equal(bits(q8.dequantize(rows, 512)), bits(oracle.dequantize_q8_0(rows, 512, "ref")))


# ------------------------------------------------------------------------------------------------------------- file readers
def test_gguf_reader_q8_0(tmp_path):
    pytest.importorskip("gguf")
    m, tok_rows = q8.toy(seed=3, n_head=4, n_head_kv=2)
    path = str(tmp_path / "q8.gguf")
    q8.write_gguf(path, m.hp, tok_rows, m.out_norm, m.out_rows, m.layers)
    p = gguf_loader.parse(path)
    for key in ("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_ff", "n_ctx"):
        assert p.hparams[key] == m.hp[key], key
    assert np.array_equal(bits(p.tok_embd), bits(m.tok))                   # dequantize_row_q8_0's values
    assert np.array_equal(p.out_norm, m.out_norm)
    assert p.output[0] == "q8_0" and np.array_equal(p.output[1], m.out_rows)
    for L, want in zip(p.layers, m.layers):
        assert np.array_equal(L["attn_norm"], want["attn_norm"]) and np.array_equal(L["ffn_norm"], want["ffn_norm"])
        for name in ("wq", "wk", "wv", "wo", "w1", "w2", "w3"):
            assert L[name][0] == "q8_0" and np.array_equal(L[name][1], want[name]), name


def test_gguf_q8_0_weight_with_wrong_shape_is_refused(tmp_path):
    pytest.importorskip("gguf")
    m, tok_rows = q8.toy(seed=4)
    m.layers[1]["w2"] = m.layers[1]["w1"]  # ffn_down written with ffn_gate's shape
    path = str(tmp_path / "bad.gguf")
    q8.write_gguf(path, m.hp, tok_rows, m.out_norm, m.out_rows, m.layers)
    with pytest.raises(ValueError, match="ffn_down"):
        gguf_loader.parse(path)


def _ne_header(f, shape, name, ftype):
    s = name.encode()
    f.write(struct.pack("iii", len(shape), len(s), ftype))
    f.write(struct.pack("i" * len(shape), *shape[::-1]))
    f.write(s)
    f.seek((f.tell() + 31) & -32)


def test_ne_reader_q8_0(tmp_path):
    rng = np.random.default_rng(21)
    V, E, H, HK, NL, FF = 48, 256, 4, 2, 2, 384
    kvd = E // H * HK
    path = str(tmp_path / "q8.bin")
    ref = {}
    with open(path, "wb") as f:
        f.write(b"ggjt"[::-1])
        f.write(struct.pack("i" * 9, 1, V, E, 256, H, HK, NL, E // H, 7))
        f.write(struct.pack("i", 0))
        f.write(struct.pack("ff", 0, 0))
        f.write(struct.pack("iii", 0, 0, 0))
        f.write(struct.pack("i", 0))
        f.write(struct.pack("i", FF))
        f.write(struct.pack("iiii", 0, 0, 0, 0))
        f.write(struct.pack("fff", 1e-5, 10000.0, 1.0))
        f.write(struct.pack("f", 0.0))
        f.write(struct.pack("ii", 0, 0))
        f.write(struct.pack("iiii", 1, 2, 0, 0))
        for i in range(V):
            t = f"t{i}".encode()
            f.write(struct.pack("i", len(t)))
            f.write(t)
            f.write(struct.pack("f", -float(i)))

        def q8w(name, n, k):
            rows = q8.quantize_weights(rng.normal(0, 0.05, (n, k)).astype(np.float32))
            ref[name] = rows
            _ne_header(f, [n, k], name, 8)
            rows.tofile(f)

        def fp32(name, arr):
            ref[name] = arr
            _ne_header(f, list(arr.shape), name, 0)
            arr.tofile(f)

        q8w("tok_embeddings.weight", V, E)
        fp32("norm.weight", rng.uniform(0.5, 1.5, E).astype(np.float32))
        q8w("output.weight", V, E)
        for il in range(NL):
            for nm, (n, k) in dict(wq=(E, E), wk=(kvd, E), wv=(kvd, E), wo=(E, E)).items():
                q8w(f"layers.{il}.attention.{nm}.weight", n, k)
            for nm, (n, k) in dict(w1=(FF, E), w2=(E, FF), w3=(FF, E)).items():
                q8w(f"layers.{il}.feed_forward.{nm}.weight", n, k)
            fp32(f"layers.{il}.attention_norm.weight", rng.uniform(0.5, 1.5, E).astype(np.float32))
            fp32(f"layers.{il}.ffn_norm.weight", rng.uniform(0.5, 1.5, E).astype(np.float32))
    m = ne_loader.parse(path)
    assert (m.hparams["n_vocab"], m.hparams["n_embd"], m.hparams["n_ff"], m.hparams["n_head_kv"]) == (V, E, FF, HK)
    assert np.array_equal(bits(m.tok_embd), bits(q8.dequantize(ref["tok_embeddings.weight"], E)))
    assert m.output[0] == "q8_0" and np.array_equal(m.output[1], ref["output.weight"])
    for il, L in enumerate(m.layers):
        for nm in ("wq", "wk", "wv", "wo"):
            assert L[nm][0] == "q8_0" and np.array_equal(L[nm][1], ref[f"layers.{il}.attention.{nm}.weight"])
        for nm in ("w1", "w2", "w3"):
            assert L[nm][0] == "q8_0" and np.array_equal(L[nm][1], ref[f"layers.{il}.feed_forward.{nm}.weight"])


# ------------------------------------------------------------------------------------------------------------- ring plans
# Llama-2-7B's nodes: (k, mode, rows per launch) -- q/k/v as one QKV launch, o, gate/up, down, and the lm_head
NODES_7B = {"qkv": (4096, 1), "o": (4096, 0), "gate_up": (4096, 2), "down": (11008, 0), "lm_head": (4096, 0)}


def plan(k, mode, m, fused, norm):
    out = (C.c_int * 5)()
    rc = ns.lib().ns_gemv_ring_plan_q8_0(k, mode, m, fused, norm, out)
    return rc, list(out)


@pytest.mark.parametrize("node", sorted(NODES_7B))
@pytest.mark.parametrize("m", [1, 2, 4])
@pytest.mark.parametrize("fused", [0, 1])
def test_ring_plan_every_7b_node(node, m, fused):
    k, mode = NODES_7B[node]
    rc, out = plan(k, mode, m, fused, 0)
    assert rc == 1, (node, m, fused, ns.last_error())
    wide, rows, stages, active, ctas = out
    assert rows in (1, 2) and stages >= active >= 1 and stages % active == 0 and ctas in (1, 2)
    assert wide == (1 if (m == 1 and fused) else 0)
    if mode == 2:
        assert rows == 2                                       # the gate/up epilogue needs both rows in one warp


@pytest.mark.parametrize("node", ["qkv", "gate_up", "lm_head", "o"])
@pytest.mark.parametrize("m", [1, 2])
def test_ring_plan_fused_norm_7b(node, m):
    k, mode = NODES_7B[node]
    rc, out = plan(k, mode, m, 1, 1)
    assert rc == 1, ns.last_error()
    assert out[2] >= 1


def test_ring_plan_7b_choices_recorded():
    """The planner's choice at 7B shapes (DESIGN.md section 4): a Q8_0 row of K = 11008 is 11,696 B (a Q4_0 row 6,192 B), so the
    down projection's 4-row tiles take single-row stages"""
    assert plan(4096, 0, 1, 1, 0) == (1, [1, 2, 14, 14, 1])    # wide kernel, row pairs
    assert plan(4096, 2, 1, 1, 1) == (1, [1, 2, 14, 14, 1])    # gate/up with the folded norm
    assert plan(11008, 0, 1, 1, 0) == (1, [1, 1, 14, 14, 1])   # down: single rows
    assert plan(11008, 0, 2, 1, 0) == (1, [0, 1, 7, 7, 2])
    assert plan(11008, 0, 4, 1, 0) == (1, [0, 1, 5, 5, 2])     # 4-row tiles: five stages per CTA


def test_ring_plan_refusals():
    out = (C.c_int * 5)()
    L = ns.lib()
    assert L.ns_gemv_ring_plan_q8_0(4100, 0, 1, 1, 0, out) < 0     # k % 32 != 0
    assert L.ns_gemv_ring_plan_q8_0(4096, 3, 1, 1, 0, out) < 0
    assert L.ns_gemv_ring_plan_q8_0(4096, 0, 3, 1, 1, out) < 0     # a folded norm takes <= 2 rows
    assert L.ns_gemv_ring_plan_q8_0(4096, 0, 1, 0, 1, out) < 0     # ... and the fused quantiser

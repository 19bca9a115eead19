"""Qwen2 on the CPU: the NeoX RoPE restatement, the interleave identity the eval step relies on, the Qwen2 CPU graph against the
reference's own engine (or its golden fixture where oracle/_ref is not built), and GGUF qwen2 files."""
import os

import numpy as np
import pytest

import oracle
from neural_speed_b200 import gguf_loader
from oracle.llama_model import OracleLlama, rope_mode0_rows
from oracle.qwen2 import OracleQwen2, RefNeQwen2, interleave_heads, interleave_perm, ref_ne_qwen2, ref_rope, rope_neox_rows

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qwen2_tiny.npz")
HAVE_REF = ref_ne_qwen2() is not None


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


# (n_past, n_tokens): a prompt over every position 0 .. 8191, and single tokens at the edges
GRID = [(0, 8192), (0, 1), (1, 1), (4095, 1), (8191, 1)]


def test_interleave_perm_pairs():
    for hd in (64, 128):
        p = interleave_perm(hd)
        assert sorted(p.tolist()) == list(range(hd))
        assert np.array_equal(p[0::2], np.arange(hd // 2)) and np.array_equal(p[1::2], np.arange(hd // 2) + hd // 2)


@pytest.mark.parametrize("hd", [64, 128])
@pytest.mark.parametrize("base", [10000.0, 1000000.0])
def test_rope_neox_and_interleave_identity(hd, base):
    """rope_neox_rows is bit-identical to ne_rope_inplace(mode 2), and rope_mode0(P x) == P rope_neox(x) bit for bit, in the
    oracle and through the reference's own two modes"""
    rng = np.random.default_rng(hd + int(base))
    for n_past, n in GRID:
        x = rng.standard_normal((n, 2, hd)).astype(np.float32)
        pos = np.arange(n_past, n_past + n)
        neox = rope_neox_rows(x, pos, hd, base)
        px = interleave_heads(x, hd)
        assert np.array_equal(_bits(rope_mode0_rows(px, pos, hd, base)), _bits(interleave_heads(neox, hd))), (n_past, n)
        if HAVE_REF:
            assert np.array_equal(_bits(neox), _bits(ref_rope(x, hd, n_past, base, True))), (n_past, n)
            assert np.array_equal(_bits(ref_rope(px, hd, n_past, base, False)),
                                  _bits(interleave_heads(ref_rope(x, hd, n_past, base, True), hd))), (n_past, n)


def test_rope_neox_golden():
    """the reference's mode-2 outputs stored in the fixture (positions 8180 .. 8191)"""
    g = np.load(GOLDEN)
    for hd in (64, 128):
        for base in (10000.0, 1000000.0):
            x, y = g[f"rope.{hd}.{int(base)}.x"], g[f"rope.{hd}.{int(base)}.y"]
            got = rope_neox_rows(x, np.arange(8180, 8180 + x.shape[0]), hd, base)
            assert np.array_equal(_bits(got), _bits(y)), (hd, base)


def _golden_model(g, kind):
    hp = dict(zip(("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_ff", "n_ctx"), (int(v) for v in g[f"{kind}.hp"])))
    hp.update(norm_eps=1e-6, rope_theta=1000000.0, rope_scale=1.0)
    names = ("attn_norm", "ffn_norm", "wq", "wk", "wv", "wo", "w1", "w2", "w3", "bq", "bk", "bv")
    layers = [{k: g[f"{kind}.l{il}.{k}"] for k in names} for il in range(hp["n_layer"])]
    return hp, g[f"{kind}.tok"], g[f"{kind}.out_norm"], g[f"{kind}.output"], layers


STEPS = [[1, 40, 7, 91], [13], [55], [2]]


@pytest.mark.parametrize("kind", ["mha", "gqa"])
def test_qwen2_graph_matches_reference(kind):
    """OracleQwen2 reproduces the reference engine's qwen2 graph bit for bit: a masked 4-token prompt, then single
    tokens; against RefNeQwen2 where oracle/_ref is built, and against the stored logits always"""
    g = np.load(GOLDEN)
    hp, tok, out_norm, output, layers = _golden_model(g, kind)
    orc = OracleQwen2(hp, tok, out_norm, output, layers)
    ref = RefNeQwen2(hp, tok, out_norm, output, layers) if HAVE_REF else None
    pos = 0
    for i, t in enumerate(STEPS):
        got = orc.eval(t, pos)
        assert np.array_equal(_bits(got), _bits(g[f"{kind}.logits{i}"])), i
        if ref is not None:
            assert np.array_equal(_bits(got), _bits(ref.eval(t, pos))), i
        pos += len(t)
    if ref is not None:
        ref.close()


@pytest.mark.skipif(not HAVE_REF, reason="oracle/_ref not built")
def test_qwen2_graph_fresh_model_matches_reference():
    """a model drawn here (not the fixture's), GQA with head size 128, a 9-token prompt and two steps"""
    import qwen2_models
    m = qwen2_models.toy(n_head=2, n_head_kv=1, seed=5, n_ctx=16)
    orc, ref = m.graph(), m.reference()
    pos = 0
    for t in ([5, 9, 300, 2, 17, 44, 8, 1, 0], [77], [3]):
        assert np.array_equal(_bits(orc.eval(t, pos)), _bits(ref.eval(t, pos)))
        pos += len(t)
    ref.close()


def test_qwen2_graph_differs_from_llama_by_its_biases_and_rope():
    """OracleQwen2 with zero biases on a model whose W_q / W_k rows are in P order is bit for bit the Llama graph on those rows
    (the identity the eval step relies on, through whole graphs); with the fixture's biases it is not"""
    g = np.load(GOLDEN)
    hp, tok, out_norm, output, layers = _golden_model(g, "gqa")
    hd = hp["n_embd"] // hp["n_head"]

    def rows_p(w):
        n = w.shape[0]
        return np.ascontiguousarray(w[np.arange(n) // hd * hd + interleave_perm(hd)[np.arange(n) % hd]])

    zero = [dict(L, bq=L["bq"] * 0, bk=L["bk"] * 0, bv=L["bv"] * 0) for L in layers]
    twin = [dict(L, wq=rows_p(L["wq"]), wk=rows_p(L["wk"])) for L in layers]
    a = OracleQwen2(hp, tok, out_norm, output, zero).eval(STEPS[0], 0)
    b = OracleLlama(hp, tok, out_norm, output, twin).eval(STEPS[0], 0)
    assert np.array_equal(_bits(a), _bits(b))
    assert not np.array_equal(a, OracleQwen2(hp, tok, out_norm, output, layers).eval(STEPS[0], 0))


# ---------------------------------------------------------------------------------------------------------------- GGUF
gguf = pytest.importorskip("gguf")


def _write(path, arch="qwen2", tie=False, n_head_kv=2):
    rng = np.random.default_rng(3)
    V, E, H, NL, FF = 64, 256, 4, 2, 512
    kvd = E // H * n_head_kv
    w = gguf.GGUFWriter(path, arch)
    w.add_context_length(256)
    w.add_embedding_length(E)
    w.add_block_count(NL)
    w.add_feed_forward_length(FF)
    w.add_head_count(H)
    w.add_head_count_kv(n_head_kv)
    w.add_layer_norm_rms_eps(1e-6)
    w.add_rope_freq_base(1000000.0)
    T = gguf.GGMLQuantizationType
    ref = {}

    def q4(name, n, k):
        rows = oracle.quantize_q4_0(rng.normal(0, 0.05, (n, k)).astype(np.float32))
        ref[name] = rows
        w.add_tensor(name, rows, raw_dtype=T.Q4_0)

    def f32(name, a):
        ref[name] = a
        w.add_tensor(name, a)

    q4("token_embd.weight", V, E)
    f32("output_norm.weight", rng.uniform(0.5, 1.5, E).astype(np.float32))
    if not tie:
        q4("output.weight", V, E)
    for il in range(NL):
        for nm in ("attn_norm", "ffn_norm"):
            f32(f"blk.{il}.{nm}.weight", rng.uniform(0.5, 1.5, E).astype(np.float32))
        for nm, (n, k) in dict(attn_q=(E, E), attn_k=(kvd, E), attn_v=(kvd, E), attn_output=(E, E), ffn_gate=(FF, E),
                               ffn_down=(E, FF), ffn_up=(FF, E)).items():
            q4(f"blk.{il}.{nm}.weight", n, k)
        if arch == "qwen2":
            for nm, n in (("attn_q", E), ("attn_k", kvd), ("attn_v", kvd)):
                f32(f"blk.{il}.{nm}.bias", rng.normal(0, 0.5, n).astype(np.float32))
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    return ref, dict(n_vocab=V, n_embd=E, n_head=H, n_head_kv=n_head_kv, n_layer=NL, n_ff=FF, n_ctx=256)


@pytest.mark.parametrize("tie", [False, True])
@pytest.mark.parametrize("n_head_kv", [4, 2])
def test_parse_qwen2_gguf(tmp_path, tie, n_head_kv):
    path = str(tmp_path / "qwen2.gguf")
    ref, hp = _write(path, tie=tie, n_head_kv=n_head_kv)
    m = gguf_loader.parse(path)
    assert m.arch == "qwen2"
    for k, v in hp.items():
        assert m.hparams[k] == v, k
    assert m.hparams["rope_theta"] == 1000000.0 and abs(m.hparams["norm_eps"] - 1e-6) < 1e-12 and m.hparams["rope_scale"] == 1.0
    out_name = "token_embd.weight" if tie else "output.weight"
    assert m.output[0] == "q4_0" and np.array_equal(m.output[1], ref[out_name])
    for il, L in enumerate(m.layers):
        assert np.array_equal(L["wq"][1], ref[f"blk.{il}.attn_q.weight"]) and np.array_equal(L["wk"][1], ref[f"blk.{il}.attn_k.weight"])
        for ours, theirs in (("bq", "attn_q"), ("bk", "attn_k"), ("bv", "attn_v")):
            assert L[ours].dtype == np.float32 and np.array_equal(L[ours], ref[f"blk.{il}.{theirs}.bias"]), (il, ours)
    # through the CPU graph: the parsed tensors are the model the graph runs (and the biases move its logits)
    layers = [{k: v[1] if isinstance(v, tuple) else v for k, v in L.items()} for L in m.layers]
    cpu = OracleQwen2(m.hparams, m.tok_embd, m.out_norm, m.output[1], layers)
    logits = cpu.eval([1, 2, 3], 0)
    assert logits.shape == (hp["n_vocab"],) and np.isfinite(logits).all()
    nob = [dict(L, bq=L["bq"] * 0, bk=L["bk"] * 0, bv=L["bv"] * 0) for L in layers]
    assert not np.array_equal(logits, OracleQwen2(m.hparams, m.tok_embd, m.out_norm, m.output[1], nob).eval([1, 2, 3], 0))


def test_parse_llama_gguf_still_llama(tmp_path):
    path = str(tmp_path / "llama.gguf")
    ref, hp = _write(path, arch="llama")
    m = gguf_loader.parse(path)
    assert m.arch == "llama"
    for k, v in hp.items():
        assert m.hparams[k] == v, k
    assert all(set(L) == {"attn_norm", "ffn_norm", "wq", "wk", "wv", "wo", "w1", "w2", "w3"} for L in m.layers)


def test_parse_rejects_other_architecture(tmp_path):
    path = str(tmp_path / "phi.gguf")
    w = gguf.GGUFWriter(path, "phi2")
    w.add_tensor("token_embd.weight", np.zeros((4, 32), np.float32))
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    with pytest.raises(ValueError, match="architecture"):
        gguf_loader.parse(path)

"""Phi-3 on the CPU: the interleave identity at head size 96, the Phi-3 CPU graph against the reference's own engine (or its golden
fixture where oracle/_ref is not built) at head sizes 64 and 96, and GGUF phi3 files."""
import os

import numpy as np
import pytest

import oracle
from neural_speed_b200 import gguf_loader
from oracle.llama_model import OracleLlama, rope_mode0_rows
from oracle.phi3 import OraclePhi3, RefNePhi3, ref_ne_phi3
from oracle.qwen2 import interleave_heads, interleave_perm, ref_rope, rope_neox_rows

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "phi3_tiny.npz")
HAVE_REF = ref_ne_phi3() is not None
KINDS = ["mha64", "gqa64", "mha96", "gqa96"]
STEPS = [[1, 40, 7, 91], [13], [55], [2]]


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def test_interleave_perm_at_head_size_96():
    """P at hd 96: i -> 2i and i + 48 -> 2i + 1"""
    p = interleave_perm(96)
    assert sorted(p.tolist()) == list(range(96))
    assert np.array_equal(p[0::2], np.arange(48)) and np.array_equal(p[1::2], np.arange(48) + 48)


@pytest.mark.parametrize("base", [10000.0, 500000.0])
def test_interleave_identity_at_head_size_96(base):
    """rope_mode0(P x) == P rope_neox(x) bit for bit at every position 0 .. 8191, and rope_neox_rows is the reference's mode 2"""
    rng = np.random.default_rng(96 + int(base))
    x = rng.standard_normal((8192, 2, 96)).astype(np.float32)
    pos = np.arange(8192)
    neox = rope_neox_rows(x, pos, 96, base)
    assert np.array_equal(_bits(rope_mode0_rows(interleave_heads(x, 96), pos, 96, base)), _bits(interleave_heads(neox, 96)))
    if HAVE_REF:
        assert np.array_equal(_bits(neox), _bits(ref_rope(x, 96, 0, base, True)))


def _golden_model(g, kind):
    hp = dict(zip(("n_vocab", "n_embd", "n_head", "n_head_kv", "n_layer", "n_ff", "n_ctx"), (int(v) for v in g[f"{kind}.hp"])))
    hp.update(norm_eps=1e-5, rope_theta=10000.0, rope_scale=1.0)
    names = ("attn_norm", "ffn_norm", "wq", "wk", "wv", "wo", "w1", "w2", "w3")
    layers = [{k: g[f"{kind}.l{il}.{k}"] for k in names} for il in range(hp["n_layer"])]
    return hp, g[f"{kind}.tok"], g[f"{kind}.out_norm"], g[f"{kind}.output"], layers


@pytest.mark.parametrize("kind", KINDS)
def test_phi3_graph_matches_reference(kind):
    """OraclePhi3 reproduces the reference engine's bias-free qwen2 graph (phi3.cpp's op sequence) bit for bit: a masked 4-token
    prompt, then single tokens; against RefNePhi3 where oracle/_ref is built, and against the stored logits always"""
    g = np.load(GOLDEN)
    hp, tok, out_norm, output, layers = _golden_model(g, kind)
    orc = OraclePhi3(hp, tok, out_norm, output, layers)
    ref = RefNePhi3(hp, tok, out_norm, output, layers) if HAVE_REF else None
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
def test_phi3_graph_fresh_model_matches_reference():
    """a model drawn here (not the fixture's), GQA with head size 96, a 9-token prompt and two steps"""
    import phi3_models
    m = phi3_models.toy(n_head=2, n_head_kv=1, seed=5, n_ctx=16)
    orc, ref = m.graph(), m.reference()
    pos = 0
    for t in ([5, 9, 300, 2, 17, 44, 8, 1, 0], [77], [3]):
        assert np.array_equal(_bits(orc.eval(t, pos)), _bits(ref.eval(t, pos)))
        pos += len(t)
    ref.close()


def test_phi3_graph_is_the_llama_graph_on_interleaved_rows():
    """OraclePhi3 is bit for bit the Llama graph on W_q / W_k rows in P order (the identity the eval step relies on), at hd 96"""
    g = np.load(GOLDEN)
    hp, tok, out_norm, output, layers = _golden_model(g, "gqa96")
    hd = hp["n_embd"] // hp["n_head"]

    def rows_p(w):
        n = w.shape[0]
        return np.ascontiguousarray(w[np.arange(n) // hd * hd + interleave_perm(hd)[np.arange(n) % hd]])

    twin = [dict(L, wq=rows_p(L["wq"]), wk=rows_p(L["wk"])) for L in layers]
    a = OraclePhi3(hp, tok, out_norm, output, layers).eval(STEPS[0], 0)
    assert np.array_equal(_bits(a), _bits(OracleLlama(hp, tok, out_norm, output, twin).eval(STEPS[0], 0)))
    assert not np.array_equal(a, OracleLlama(hp, tok, out_norm, output, layers).eval(STEPS[0], 0))


# ---------------------------------------------------------------------------------------------------------------- GGUF
gguf = pytest.importorskip("gguf")

V, H, NL, FF = 64, 4, 2, 256


def _write(path, fused=True, tie=False, n_head_kv=4, hd=96, n_rot=None, longrope=False, qkv_rows=None):
    """a synthetic phi3 file; returns the tensors written and the hyper-parameters"""
    rng = np.random.default_rng(3)
    E = hd * H
    kvd = hd * n_head_kv
    w = gguf.GGUFWriter(path, "phi3")
    w.add_context_length(256)
    w.add_embedding_length(E)
    w.add_block_count(NL)
    w.add_feed_forward_length(FF)
    w.add_head_count(H)
    w.add_head_count_kv(n_head_kv)
    w.add_layer_norm_rms_eps(1e-5)
    w.add_rope_freq_base(10000.0)
    w.add_rope_dimension_count(hd if n_rot is None else n_rot)
    T = gguf.GGMLQuantizationType
    ref = {}

    def q4(name, n, k, rows=None):
        rows = oracle.quantize_q4_0(rng.normal(0, 0.05, (n, k)).astype(np.float32)) if rows is None else rows
        ref[name] = rows
        w.add_tensor(name, rows, raw_dtype=T.Q4_0)

    def f32(name, a):
        ref[name] = a
        w.add_tensor(name, a)

    q4("token_embd.weight", V, E)
    f32("output_norm.weight", rng.uniform(0.5, 1.5, E).astype(np.float32))
    if not tie:
        q4("output.weight", V, E)
    if longrope:
        f32("rope_factors_long.weight", np.ones(hd // 2, np.float32))
        f32("rope_factors_short.weight", np.ones(hd // 2, np.float32))
    for il in range(NL):
        for nm in ("attn_norm", "ffn_norm"):
            f32(f"blk.{il}.{nm}.weight", rng.uniform(0.5, 1.5, E).astype(np.float32))
        qkv = oracle.quantize_q4_0(rng.normal(0, 0.05, (E + 2 * kvd if qkv_rows is None else qkv_rows, E)).astype(np.float32))
        if fused:
            q4(f"blk.{il}.attn_qkv.weight", 0, 0, qkv)
        else:  # the same rows as three tensors
            for nm, (a, b) in (("attn_q", (0, E)), ("attn_k", (E, E + kvd)), ("attn_v", (E + kvd, E + 2 * kvd))):
                q4(f"blk.{il}.{nm}.weight", 0, 0, np.ascontiguousarray(qkv[a:b]))
        for nm, (n, k) in dict(attn_output=(E, E), ffn_down=(E, FF), ffn_up=(2 * FF, E)).items():
            q4(f"blk.{il}.{nm}.weight", n, k)
    w.write_header_to_file()
    w.write_kv_data_to_file()
    w.write_tensors_to_file()
    w.close()
    return ref, dict(n_vocab=V, n_embd=E, n_head=H, n_head_kv=n_head_kv, n_layer=NL, n_ff=FF, n_ctx=256)


@pytest.mark.parametrize("tie", [False, True])
@pytest.mark.parametrize("n_head_kv", [4, 2])
def test_parse_phi3_gguf(tmp_path, tie, n_head_kv):
    """the fused q / k / v and gate / up rows split into the layer dict; tied and untied output"""
    path = str(tmp_path / "phi3.gguf")
    ref, hp = _write(path, tie=tie, n_head_kv=n_head_kv)
    m = gguf_loader.parse(path)
    assert m.arch == "phi3"
    for k, v in hp.items():
        assert m.hparams[k] == v, k
    assert m.hparams["rope_theta"] == 10000.0 and m.hparams["rope_scale"] == 1.0
    out_name = "token_embd.weight" if tie else "output.weight"
    assert m.output[0] == "q4_0" and np.array_equal(m.output[1], ref[out_name])
    E, kvd = hp["n_embd"], hp["n_embd"] // H * n_head_kv
    for il, L in enumerate(m.layers):
        assert set(L) == {"attn_norm", "ffn_norm", "wq", "wk", "wv", "wo", "w1", "w2", "w3"}
        qkv, up = ref[f"blk.{il}.attn_qkv.weight"], ref[f"blk.{il}.ffn_up.weight"]
        assert np.array_equal(L["wq"][1], qkv[:E]) and np.array_equal(L["wk"][1], qkv[E:E + kvd])
        assert np.array_equal(L["wv"][1], qkv[E + kvd:])
        assert np.array_equal(L["w1"][1], up[:FF]) and np.array_equal(L["w3"][1], up[FF:])  # gate first
        assert all(L[k][0] == "q4_0" and L[k][1].flags.c_contiguous for k in ("wq", "wk", "wv", "w1", "w3"))
    layers = [{k: v[1] if isinstance(v, tuple) else v for k, v in L.items()} for L in m.layers]
    logits = OraclePhi3(m.hparams, m.tok_embd, m.out_norm, m.output[1], layers).eval([1, 2, 3], 0)
    assert logits.shape == (V,) and np.isfinite(logits).all()


@pytest.mark.parametrize("n_head_kv", [4, 2])
def test_parse_phi3_separate_qkv_is_the_fused_split(tmp_path, n_head_kv):
    """a file with separate attn_q / k / v gives the same layer dicts as the file whose attn_qkv stacks their rows"""
    fused, sep = str(tmp_path / "fused.gguf"), str(tmp_path / "sep.gguf")
    _write(fused, n_head_kv=n_head_kv)
    _write(sep, fused=False, n_head_kv=n_head_kv)
    a, b = gguf_loader.parse(fused), gguf_loader.parse(sep)
    assert a.hparams == b.hparams
    for La, Lb in zip(a.layers, b.layers):
        assert set(La) == set(Lb)
        for k in La:
            x, y = (La[k][1], Lb[k][1]) if isinstance(La[k], tuple) else (La[k], Lb[k])
            assert np.array_equal(x, y), k


@pytest.mark.parametrize("case,match", [(dict(longrope=True), "LongRoPE"), (dict(n_rot=64), "partial rotary"),
                                        (dict(qkv_rows=96 * H * 3 - 32), "attn_qkv"), (dict(n_head_kv=2, qkv_rows=96 * H * 3),
                                                                                        "attn_qkv")])
def test_parse_phi3_refusals(tmp_path, case, match):
    path = str(tmp_path / "bad.gguf")
    _write(path, **case)
    with pytest.raises(ValueError, match=match):
        gguf_loader.parse(path)


def test_parse_llama_and_qwen2_unchanged(tmp_path):
    """llama and qwen2 files parse to the same layer dicts as before: the separate tensors, and the biases for qwen2 only"""
    import test_qwen2_cpu
    for arch in ("llama", "qwen2"):
        path = str(tmp_path / f"{arch}.gguf")
        ref, hp = test_qwen2_cpu._write(path, arch=arch)
        m = gguf_loader.parse(path)
        assert m.arch == arch
        keys = {"attn_norm", "ffn_norm", "wq", "wk", "wv", "wo", "w1", "w2", "w3"} | ({"bq", "bk", "bv"} if arch == "qwen2" else set())
        for il, L in enumerate(m.layers):
            assert set(L) == keys
            for ours, theirs in (("wq", "attn_q"), ("wk", "attn_k"), ("wv", "attn_v"), ("w1", "ffn_gate"), ("w3", "ffn_up")):
                assert np.array_equal(L[ours][1], ref[f"blk.{il}.{theirs}.weight"]), (arch, ours)

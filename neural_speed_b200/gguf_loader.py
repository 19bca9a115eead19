"""GGUF (llama, qwen2 and phi3 architectures) -> tensors for the device eval step (SURVEY §8 f.3, first slice).

The reference reads GGUF in C++ (`models/model_utils/gguf.h`, `model_files.h:246-860`: header, key/value metadata, tensor
infos, aligned data) and maps llama tensors to `model.others[0..2]` / `layers[il].norm/attn/ffn` (`models/llama/llama_utils.cpp`).
Here the container is parsed with the `gguf` Python package (the format's own reader) and the tensors are handed over in the
types the eval step consumes:

  token_embd.weight   F32/F16/Q4_0/Q8_0 -> fp32 table (the reference's ne_get_rows dequantises the looked-up rows; same values)
  *_norm.weight       F32
  attn_q/k/v.bias     F32 (qwen2 only: Qwen1.5 / Qwen2 / Qwen2.5 files, models/qwen/qwen_utils.cpp:130-143)
  attn_q/k/v/output, ffn_gate/down/up, output.weight   Q4_0 rows (18-byte blocks), Q8_0 rows (34-byte blocks) or Q6_K rows
                      (210-byte blocks), untouched
  phi3 files          attn_qkv.weight: the fused q / k / v rows, split by rows into wq [0, E), wk [E, E + kvd), wv [E + kvd,
                      E + 2 kvd) (separate attn_q / k / v are accepted too); ffn_up.weight: 2 n_ff rows, gate first (phi3.cpp:327-329),
                      split into w1 (gate) and w3 (up).  Rows of every supported type are self-contained, so a split is a row
                      slice.  LongRoPE files (rope_factors_long / _short, the 128k variants) and partial rotary
                      (rope.dimension_count != head size) are refused.

Host logic only (numpy); `parse()` is covered on CPU (tests/test_gguf_cpu.py).  `load_into_engine()` composes already-tested
device entry points (Weight.from_q4_0_host / from_q6_K_host, Llama.set_*) but has not itself been run on a GPU in round 1.
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

Q4_0_BLOCK, Q8_0_BLOCK, Q6_K_BLOCK = 18, 34, 210


def dequantize_q4_0(rows: np.ndarray, k: int) -> np.ndarray:
    """block_q4_0 rows uint8 [N, K/32*18] -> fp32 [N, K]: d * (nibble - 8), element j in the low nibble of byte j and element
    j + 16 in the high nibble (dequantize_row_q4_0, vectors/cpu/quantize.h:281-300)."""
    n = rows.shape[0]
    b = np.ascontiguousarray(rows, np.uint8).reshape(n, k // 32, Q4_0_BLOCK)
    d = b[:, :, :2].copy().view(np.float16).astype(np.float32)            # [n, nb, 1]
    q = b[:, :, 2:]
    lo = (q & 0x0F).astype(np.int8) - 8
    hi = (q >> 4).astype(np.int8) - 8
    vals = np.concatenate([lo, hi], axis=2).astype(np.float32) * d        # [n, nb, 32]
    return vals.reshape(n, k)


def dequantize_q8_0(rows: np.ndarray, k: int) -> np.ndarray:
    """block_q8_0 rows uint8 [N, K/32*34] -> fp32 [N, K]: fp32(d) * q, one fp32 product per element, element j in byte j of the
    block's codes (dequantize_row_q8_0, vectors/cpu/quantize.h:780)."""
    n = rows.shape[0]
    b = np.ascontiguousarray(rows, np.uint8).reshape(n, k // 32, Q8_0_BLOCK)
    d = b[:, :, :2].copy().view(np.float16).astype(np.float32)            # [n, nb, 1]
    q = b[:, :, 2:].copy().view(np.int8).astype(np.float32)
    return (q * d).reshape(n, k)


@dataclass
class GGUFLlama:
    hparams: dict
    tok_embd: np.ndarray                      # fp32 [n_vocab, n_embd]
    out_norm: np.ndarray                      # fp32 [n_embd]
    output: tuple                             # (type, rows uint8)
    layers: list = field(default_factory=list)  # dicts: attn_norm, ffn_norm (fp32) and wq, wk, wv, wo, w1, w2, w3 = (type, rows)
    arch: str = "llama"                       # "qwen2": the layer dicts also hold bq, bk, bv (fp32); or "phi3"


_LAYER_TENSORS = {"attn_q": "wq", "attn_k": "wk", "attn_v": "wv", "attn_output": "wo", "ffn_gate": "w1", "ffn_down": "w2", "ffn_up": "w3"}


def _field(reader, key, default=None):
    f = reader.get_field(key)
    if f is None:
        return default
    v = f.parts[f.data[0]]
    return v[0].item() if hasattr(v[0], "item") else v[0]


def parse(path: str) -> GGUFLlama:
    import gguf
    r = gguf.GGUFReader(path)
    arch = bytes(r.get_field("general.architecture").parts[-1]).decode()
    if arch not in ("llama", "qwen2", "phi3"):
        raise ValueError(f"only the llama, qwen2 and phi3 architectures are supported, file says {arch!r}")
    hp = dict(n_embd=int(_field(r, f"{arch}.embedding_length")), n_layer=int(_field(r, f"{arch}.block_count")),
              n_ff=int(_field(r, f"{arch}.feed_forward_length")), n_head=int(_field(r, f"{arch}.attention.head_count")),
              n_ctx=int(_field(r, f"{arch}.context_length", 2048)),
              norm_eps=float(_field(r, f"{arch}.attention.layer_norm_rms_epsilon", 1e-6)),  # reference default (model_types.h)
              rope_theta=float(_field(r, f"{arch}.rope.freq_base", 10000.0)), rope_scale=1.0)
    hp["n_head_kv"] = int(_field(r, f"{arch}.attention.head_count_kv", hp["n_head"]))
    tensors = {t.name: t for t in r.tensors}
    if arch == "phi3":
        hd = hp["n_embd"] // hp["n_head"]
        n_rot = int(_field(r, "phi3.rope.dimension_count", hd))
        if n_rot != hd:
            raise ValueError(f"phi3: rope.dimension_count {n_rot} != head size {hd} (partial rotary is not supported)")
        if any(n.startswith(("rope_factors_long", "rope_factors_short")) for n in tensors):
            raise ValueError("phi3: rope_factors_long / rope_factors_short tensors (LongRoPE, the 128k models) are not supported")

    def f32(name):
        t = tensors[name]
        if t.tensor_type == gguf.GGMLQuantizationType.F32:
            return np.array(t.data, np.float32).reshape([int(d) for d in reversed(t.shape)])
        if t.tensor_type == gguf.GGMLQuantizationType.F16:
            return np.array(t.data).astype(np.float32).reshape([int(d) for d in reversed(t.shape)])
        if t.tensor_type == gguf.GGMLQuantizationType.Q4_0:
            k, n = int(t.shape[0]), int(t.shape[1])
            return dequantize_q4_0(np.array(t.data, np.uint8).reshape(n, k // 32 * Q4_0_BLOCK), k)
        if t.tensor_type == gguf.GGMLQuantizationType.Q8_0:
            k, n = int(t.shape[0]), int(t.shape[1])
            return dequantize_q8_0(np.array(t.data, np.uint8).reshape(n, k // 32 * Q8_0_BLOCK), k)
        raise ValueError(f"{name}: unsupported type {t.tensor_type.name} for an fp32 tensor")

    def quant(name, n_expect, k_expect):
        t = tensors[name]
        k, n = int(t.shape[0]), int(t.shape[1])
        if (n, k) != (n_expect, k_expect):
            raise ValueError(f"{name}: shape {n}x{k}, expected {n_expect}x{k_expect}")
        if t.tensor_type == gguf.GGMLQuantizationType.Q4_0:
            return ("q4_0", np.array(t.data, np.uint8).reshape(n, k // 32 * Q4_0_BLOCK))
        if t.tensor_type == gguf.GGMLQuantizationType.Q8_0:
            return ("q8_0", np.array(t.data, np.uint8).reshape(n, k // 32 * Q8_0_BLOCK))
        if t.tensor_type == gguf.GGMLQuantizationType.Q6_K:
            return ("q6_K", np.array(t.data, np.uint8).reshape(n, k // 256 * Q6_K_BLOCK))
        raise ValueError(f"{name}: weight type {t.tensor_type.name} not supported (Q4_0 / Q8_0 / Q6_K)")

    def split(name, parts, k):
        """the fused rows of `name` sliced into consecutive row ranges of parts[i] rows each"""
        typ, rows = quant(name, sum(parts), k)
        bounds = np.cumsum([0] + list(parts))
        return [(typ, np.ascontiguousarray(rows[a:b])) for a, b in zip(bounds[:-1], bounds[1:])]

    tok = f32("token_embd.weight")
    hp["n_vocab"] = int(tok.shape[0])
    E, FF = hp["n_embd"], hp["n_ff"]
    kvd = E // hp["n_head"] * hp["n_head_kv"]
    shapes = dict(wq=(E, E), wk=(kvd, E), wv=(kvd, E), wo=(E, E), w1=(FF, E), w2=(E, FF), w3=(FF, E))
    out_name = "output.weight" if "output.weight" in tensors else "token_embd.weight"  # tied embeddings
    model = GGUFLlama(hp, tok, f32("output_norm.weight"), quant(out_name, hp["n_vocab"], E), arch=arch)
    for il in range(hp["n_layer"]):
        L = dict(attn_norm=f32(f"blk.{il}.attn_norm.weight"), ffn_norm=f32(f"blk.{il}.ffn_norm.weight"))
        pre = f"blk.{il}."
        if arch == "phi3" and pre + "attn_qkv.weight" in tensors:
            L["wq"], L["wk"], L["wv"] = split(pre + "attn_qkv.weight", (E, kvd, kvd), E)
        if arch == "phi3":
            L["w1"], L["w3"] = split(pre + "ffn_up.weight", (FF, FF), E)
        for gname, ours in _LAYER_TENSORS.items():
            if ours not in L:
                L[ours] = quant(f"{pre}{gname}.weight", *shapes[ours])
        if arch == "qwen2":
            for gname, ours, n in (("attn_q", "bq", E), ("attn_k", "bk", kvd), ("attn_v", "bv", kvd)):
                b = f32(f"blk.{il}.{gname}.bias").reshape(-1)
                if b.size != n:
                    raise ValueError(f"blk.{il}.{gname}.bias: {b.size} values, expected {n}")
                L[ours] = b
        model.layers.append(L)
    return model


def load_into_engine(model: GGUFLlama, n_ctx: int | None = None, queue=None):
    """-> neural_speed_b200.Llama with every tensor set (weights repacked on the device)."""
    from . import Llama, Weight
    hp = dict(model.hparams)
    if n_ctx:
        hp["n_ctx"] = n_ctx
    elif hp["n_ctx"] > 32768:
        # files advertise their training length (131072 ...): the KV cache is allocated for n_ctx up front and the attention
        # kernel keeps one score per position in shared memory (~54k positions at head size 128); ask explicitly for more
        hp["n_ctx"] = 32768
    eng = Llama(hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["n_ff"], hp["n_ctx"],
                hp["norm_eps"], hp["rope_theta"], hp["rope_scale"], queue, arch=model.arch)

    def weight(tr, n, k):
        typ, rows = tr
        if typ == "btla":  # a serialized BesTLA blob (NE files, neural_speed_b200/ne_loader.py)
            return Weight.from_blob(rows, queue)
        if typ == "q6_K":
            return Weight.from_q6_K_host(rows, n, k, queue)
        if typ == "q8_0":
            return Weight.from_q8_0_host(rows, n, k, queue)
        return Weight.from_q4_0_host(rows, n, k, queue)

    E, FF = hp["n_embd"], hp["n_ff"]
    kvd = E // hp["n_head"] * hp["n_head_kv"]
    eng.set_f32(Llama.TOK_EMBD, 0, model.tok_embd)
    eng.set_f32(Llama.OUT_NORM, 0, model.out_norm)
    eng.set_weight(Llama.OUTPUT, 0, weight(model.output, hp["n_vocab"], E))
    ids = dict(wq=(Llama.WQ, E, E), wk=(Llama.WK, kvd, E), wv=(Llama.WV, kvd, E), wo=(Llama.WO, E, E), w1=(Llama.W1, FF, E),
               w2=(Llama.W2, E, FF), w3=(Llama.W3, FF, E))
    for il, L in enumerate(model.layers):
        eng.set_f32(Llama.ATTN_NORM, il, L["attn_norm"])
        eng.set_f32(Llama.FFN_NORM, il, L["ffn_norm"])
        for name, (tid, n, k) in ids.items():
            eng.set_weight(tid, il, weight(L[name], n, k))
        if model.arch == "qwen2":
            for name, tid in (("bq", Llama.BQ), ("bk", Llama.BK), ("bv", Llama.BV)):
                eng.set_f32(tid, il, L[name])
    return eng

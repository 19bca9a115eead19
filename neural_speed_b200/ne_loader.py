"""neural-speed's native `.bin` ("NE") model file -> tensors for the device eval step (SURVEY §8 f.3, second slice).

Format as read by the reference (`models/model_utils/model_files.h:1025-1230`) and written by its converters
(`convert/convert_quantized_llama.py:131-198`, `convert/common.py:467-472`), little-endian:

  u32 magic 'ggjt' (0x67676a74), u32 version (1..3)
  hparams (26 fields, model_files.h:1080-1143): n_vocab n_embd n_mult n_head n_head_kv n_layer n_rot ftype max_seq_len
      f32 alibi_bias_max f32 clip_qkv par_res word_embed_proj_dim do_layer_norm_before multi_query_group_num ffn_hidden_size
      inner_hidden_size n_experts n_experts_used n_embd_head_k f32 norm_eps f32 freq_base f32 freq_scale
      f32 rope_scaling_factor original_max_position_embeddings use_yarn
  vocab: i32 bos eos pad sep, then n_vocab x { u32 len, bytes, f32 score }
  tensors until EOF: u32 n_dims, u32 name_len, u32 type, u32 ne[n_dims] (fastest dimension first), name,
      pad to a 32-byte file offset, data.  type 0 = F32, 1 = F16, 2 = Q4_0 (18-byte blocks), 8 = Q8_0 (34-byte blocks), 19 = BTLA:
      a serialized BesTLA blob whose own leading size_t gives its length (model_files.h:1208-1213).

Llama tensor names (model_files.h:146-186): tok_embeddings.weight, norm.weight, output.weight,
layers.N.{attention_norm, ffn_norm}.weight, layers.N.attention.{wq,wk,wv,wo}.weight, layers.N.feed_forward.{w1,w2,w3}.weight.

Host logic only (numpy), CPU-tested (tests/test_ne_loader_cpu.py); the hand-off to the device (`gguf_loader.load_into_engine`)
composes already-tested entry points but was not itself run on a GPU in round 1.
"""
from __future__ import annotations

import struct

import numpy as np

from .gguf_loader import GGUFLlama, dequantize_q4_0, dequantize_q8_0

MAGIC_GGJT = 0x67676A74
NE_F32, NE_F16, NE_Q4_0, NE_Q8_0, NE_BTLA = 0, 1, 2, 8, 19

_HPARAMS = [("n_vocab", "I"), ("n_embd", "I"), ("n_mult", "I"), ("n_head", "I"), ("n_head_kv", "I"), ("n_layer", "I"), ("n_rot", "I"),
            ("ftype", "I"), ("max_seq_len", "I"), ("alibi_bias_max", "f"), ("clip_qkv", "f"), ("par_res", "I"),
            ("word_embed_proj_dim", "I"), ("do_layer_norm_before", "I"), ("multi_query_group_num", "I"), ("ffn_hidden_size", "I"),
            ("inner_hidden_size", "I"), ("n_experts", "I"), ("n_experts_used", "I"), ("n_embd_head_k", "I"), ("norm_eps", "f"),
            ("freq_base", "f"), ("freq_scale", "f"), ("rope_scaling_factor", "f"), ("original_max_position_embeddings", "I"),
            ("use_yarn", "I")]


def read_file(path: str):
    """-> (hparams dict, vocab list of (bytes, score), special ids dict, tensors dict name -> (type, shape (rows, cols) or (n,), data))"""
    buf = np.fromfile(path, np.uint8)
    mv = memoryview(buf)
    pos = 0

    def take(fmt):
        nonlocal pos
        v = struct.unpack_from("<" + fmt, mv, pos)
        pos += struct.calcsize("<" + fmt)
        return v if len(v) > 1 else v[0]

    magic, version = take("I"), take("I")
    if magic != MAGIC_GGJT or version not in (1, 2, 3):
        raise ValueError(f"not an NE/ggjt model file (magic {magic:#x}, version {version})")
    hp = {name: take(fmt) for name, fmt in _HPARAMS}
    special = dict(zip(("bos", "eos", "pad", "sep"), take("iiii")))
    vocab = []
    for _ in range(hp["n_vocab"]):
        ln = take("I")
        word = bytes(mv[pos:pos + ln])
        pos += ln
        vocab.append((word, take("f")))
    tensors = {}
    size = buf.size
    while pos < size:
        n_dims, name_len, typ = take("III")
        if n_dims < 1 or n_dims > 2:
            raise ValueError(f"tensor with {n_dims} dimensions at offset {pos}")
        ne = [take("I") for _ in range(n_dims)]
        name = bytes(mv[pos:pos + name_len]).decode()
        pos += name_len
        pos = (pos + 31) & ~31
        k = ne[0]
        n = ne[1] if n_dims == 2 else 1
        if typ == NE_BTLA:
            nbytes = struct.unpack_from("<Q", mv, pos)[0]
        elif typ == NE_F32:
            nbytes = 4 * n * k
        elif typ == NE_F16:
            nbytes = 2 * n * k
        elif typ == NE_Q4_0:
            nbytes = n * (k // 32) * 18
        elif typ == NE_Q8_0:
            nbytes = n * (k // 32) * 34
        else:
            raise ValueError(f"{name}: tensor type {typ} not supported")
        if pos + nbytes > size:
            raise ValueError(f"{name}: data runs past the end of the file")
        raw = buf[pos:pos + nbytes]
        pos += nbytes
        shape = (n, k) if n_dims == 2 else (k,)
        if typ == NE_F32:
            data = raw.view(np.float32).reshape(shape).copy()
        elif typ == NE_F16:
            data = raw.view(np.float16).reshape(shape).astype(np.float32)
        elif typ == NE_Q4_0:
            data = raw.reshape(n, (k // 32) * 18).copy()
        elif typ == NE_Q8_0:
            data = raw.reshape(n, (k // 32) * 34).copy()
        else:
            data = raw.copy()
        tensors[name] = (typ, shape, data)
    return hp, vocab, special, tensors


def parse(path: str) -> GGUFLlama:
    """NE llama file -> the same structure gguf_loader.parse returns (weights as ("q4_0", rows), ("q8_0", rows) or ("btla", blob))."""
    hp_raw, _vocab, _special, tensors = read_file(path)
    n_head_kv = hp_raw["n_head_kv"] or hp_raw["n_head"]
    n_ff = hp_raw["ffn_hidden_size"]
    if not n_ff:  # older converters store n_mult only (llama.cpp's rounding of 8/3 * n_embd)
        n_ff = ((2 * (4 * hp_raw["n_embd"]) // 3 + hp_raw["n_mult"] - 1) // hp_raw["n_mult"]) * hp_raw["n_mult"]
    hp = dict(n_vocab=hp_raw["n_vocab"], n_embd=hp_raw["n_embd"], n_head=hp_raw["n_head"], n_head_kv=n_head_kv, n_layer=hp_raw["n_layer"],
              n_ff=n_ff, n_ctx=hp_raw["max_seq_len"] or 2048, norm_eps=hp_raw["norm_eps"] or 1e-6,
              rope_theta=hp_raw["freq_base"] or 10000.0, rope_scale=hp_raw["freq_scale"] or 1.0)
    E = hp["n_embd"]
    kvd = E // hp["n_head"] * n_head_kv

    def f32(name):
        typ, shape, data = tensors[name]
        if typ in (NE_F32, NE_F16):
            return data
        if typ == NE_Q4_0:
            return dequantize_q4_0(data, shape[-1])   # 1-D tensors: the row length is the only dimension
        if typ == NE_Q8_0:
            return dequantize_q8_0(data, shape[-1])
        raise ValueError(f"{name}: type {typ} cannot be used as an fp32 tensor")

    def weight(name, n, k):
        typ, shape, data = tensors[name]
        if tuple(shape) != (n, k):
            raise ValueError(f"{name}: shape {shape}, expected {(n, k)}")
        if typ == NE_Q4_0:
            return ("q4_0", data)
        if typ == NE_Q8_0:
            return ("q8_0", data)
        if typ == NE_BTLA:
            return ("btla", data)
        raise ValueError(f"{name}: weight type {typ} not supported (Q4_0 / Q8_0 / BTLA)")

    model = GGUFLlama(hp, f32("tok_embeddings.weight"), f32("norm.weight"), weight("output.weight", hp["n_vocab"], E))
    shapes = dict(wq=(E, E), wk=(kvd, E), wv=(kvd, E), wo=(E, E), w1=(n_ff, E), w2=(E, n_ff), w3=(n_ff, E))
    for il in range(hp["n_layer"]):
        L = dict(attn_norm=f32(f"layers.{il}.attention_norm.weight"), ffn_norm=f32(f"layers.{il}.ffn_norm.weight"))
        for nm in ("wq", "wk", "wv", "wo"):
            L[nm] = weight(f"layers.{il}.attention.{nm}.weight", *shapes[nm])
        for nm in ("w1", "w2", "w3"):
            L[nm] = weight(f"layers.{il}.feed_forward.{nm}.weight", *shapes[nm])
        model.layers.append(L)
    return model

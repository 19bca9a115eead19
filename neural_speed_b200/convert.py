"""GPTQ / AWQ / AutoRound checkpoint tensors -> BesTLA blobs or device weights (host side, numpy).

Mirrors the tensor-level part of the reference converter, neural_speed/convert/common.py:
  unpack_gptq_weight_4bits :396-417, unpack_gptq_weight_8bits :341-393, unpack_awq_weight :448-464,
  the desc_act regrouping of convert_q4_bestla_tensor :667-683, the "-8" recentring :687-690 and the
  np_bestla_qpack call :703-712.  Everything here is integer/byte work and is bit-exact with the reference
  (tests/golden/gptq_awq.npz is produced by importing the reference's own functions).

HF layouts (in_features = K, out_features = N):
  GPTQ : qweight int32 [K*bits/32, N]  (values packed LSB-first along K)
         qzeros  int32 [K/g, N*bits/32] (packed LSB-first along N, stored minus one)
         scales  f16   [K/g, N]          g_idx int32 [K]
  AWQ  : qweight int32 [K, N/8], qzeros int32 [K/g, N/8] (nibble order 0,4,1,5,2,6,3,7 along N), scales f16 [K/g, N]
"""
from __future__ import annotations

import numpy as np

AWQ_ORDER = (0, 4, 1, 5, 2, 6, 3, 7)  # common.py:451


def _as_u32(x) -> np.ndarray:
    a = np.asarray(x)
    if a.dtype != np.int32 and a.dtype != np.uint32:
        raise TypeError(f"packed tensors must be int32, got {a.dtype}")
    return np.ascontiguousarray(a).view(np.uint32)


def unpack_gptq(qweight, scales, qzeros, bits: int = 4, sym: bool = False):
    """-> (int_weight [K,N], scales [K/g,N] f32, zeros [K/g,N]) exactly as unpack_gptq_weight_{4,8}bits return them:
    4 bit: weight in 0..15, zeros = nibble + 1 (int8);  8 bit: already recentred to int8 (common.py:341-393)."""
    if bits not in (4, 8):
        raise ValueError(f"unsupported bits {bits} (int3 layouts are not on the GPU path)")
    per = 32 // bits
    mask = (1 << bits) - 1
    qw, qz = _as_u32(qweight), _as_u32(qzeros)
    sc = np.asarray(scales, np.float32)
    shifts = (np.arange(per, dtype=np.uint32) * bits)
    w = (qw[:, None, :] >> shifts[None, :, None]) & mask             # [K/per, per, N]
    w = w.reshape(-1, qw.shape[1]).astype(np.int16)
    z = ((qz[:, :, None] >> shifts[None, None, :]) & mask).astype(np.int16)  # [K/g, N/per, per]
    if bits == 4:
        z = (z + 1).reshape(sc.shape).astype(np.int8)
        return w.astype(np.int8), sc, z
    # 8 bit (common.py:352-392)
    if sym:
        z = z.astype(np.uint8).view(np.int8).astype(np.int16)
    z = z + 1
    if z.size != sc.size:
        z = z[z != 1]
    z = z.reshape(sc.shape)
    if sym:
        w = (w - 128).astype(np.int8)
        z = z.astype(np.int8)
    else:
        w = (w.astype(np.int32) - 128).astype(np.int8)
        z = ((z.astype(np.int32) & 0xff) - 128).astype(np.int8)
    return w, sc, z


def unpack_awq(qweight, scales, qzeros, bits: int = 4):
    """-> (weight [K,N] in 0..15, scales, zeros [K/g,N] in 0..15); common.py:448-464 (returns float there; ints here)."""
    if bits != 4:
        raise ValueError("AWQ checkpoints are 4 bit")
    qw, qz = _as_u32(qweight), _as_u32(qzeros)
    shifts = np.array([4 * o for o in AWQ_ORDER], np.uint32)
    w = ((qw[:, :, None] >> shifts[None, None, :]) & 15).reshape(qw.shape[0], -1).astype(np.int8)
    z = ((qz[:, :, None] >> shifts[None, None, :]) & 15).reshape(qz.shape[0], -1).astype(np.int8)
    return w, np.asarray(scales, np.float32), z


def regroup_by_g_idx(int_weight: np.ndarray, g_idx, group: int) -> np.ndarray:
    """desc_act: move row i to slot g_idx[i]*group + (rank of i among the rows of its group) (common.py:667-683)."""
    gi = np.asarray(g_idx, np.int64)
    order = np.argsort(gi, kind="stable")                   # rows of group 0 in ascending i, then group 1, ...
    counts = np.bincount(gi, minlength=(int_weight.shape[0] + group - 1) // group)
    if np.any(counts > group):
        raise ValueError("g_idx assigns more than group_size rows to one group")
    starts = np.arange(counts.size, dtype=np.int64) * group
    rank = np.arange(gi.size) - np.repeat(np.cumsum(counts) - counts, counts)
    target = np.repeat(starts, counts) + rank
    out = int_weight.copy()                                  # the reference starts from a clone; untouched slots keep it
    out[target] = int_weight[order]
    return out


def permute_llama(w: np.ndarray, n_head: int, n_head_kv: int = 0) -> np.ndarray:
    """HF rotary layout -> ggml/NE layout for q/k projections, on an [N, ...] tensor (convert_quantized_llama.py:24-28, convert_llama.py:341-345)."""
    if n_head_kv and n_head != n_head_kv:
        n_head = n_head_kv
    n = w.shape[0]
    return w.reshape(n_head, 2, n // n_head // 2, *w.shape[1:]).swapaxes(1, 2).reshape(w.shape)


def to_canonical(qweight, scales, qzeros, g_idx=None, *, quant_method="gptq", bits=4, group_size=128, sym=False, desc_act=False,
                 permute_heads=None):
    """-> dict(q int8 [K,N] centred, scales f32 [K/g,N], zp int8 [K/g,N] or None, g_idx int32 [K] or None): the arguments
    convert_q4_bestla_tensor hands to np_bestla_qpack (common.py:685-712)."""
    method = quant_method.lower()
    if method in ("gptq", "autoround", "rtn"):
        w, sc, z = unpack_gptq(qweight, scales, qzeros, bits, sym)
    elif method == "awq":
        w, sc, z = unpack_awq(qweight, scales, qzeros, bits)
    else:
        raise ValueError(f"unsupported quant_method {quant_method}")
    if permute_heads:
        nh, nkv = permute_heads
        w = np.ascontiguousarray(permute_llama(w.T, nh, nkv).T)
        sc = np.ascontiguousarray(permute_llama(sc.T, nh, nkv).T)
        z = np.ascontiguousarray(permute_llama(z.T, nh, nkv).T)
    gi = None
    if desc_act:
        if g_idx is None:
            raise ValueError("desc_act needs g_idx")
        gi = np.ascontiguousarray(g_idx, np.int32)
        w = regroup_by_g_idx(w, gi, group_size)
    if bits == 4:
        w = (w.astype(np.int16) - 8).astype(np.int8)
        z = (z.astype(np.int16) - 8).astype(np.int8)
    return dict(q=np.ascontiguousarray(w, np.int8), scales=np.ascontiguousarray(sc, np.float32),
                zp=None if sym else np.ascontiguousarray(z, np.int8), g_idx=gi)


def to_blob(qweight, scales, qzeros, g_idx=None, *, compute_dtype="int8", scale_dtype="fp32", **q_config) -> np.ndarray:
    """HF quantised linear -> serialized BesTLA blob (what convert_q4_bestla_tensor writes after the tensor header)."""
    from . import np_bestla_qpack
    c = to_canonical(qweight, scales, qzeros, g_idx, **q_config)
    bits, g = q_config.get("bits", 4), q_config.get("group_size", 128)
    return np_bestla_qpack(c["q"], c["scales"], c["zp"], c["g_idx"], "int4" if bits == 4 else "int8", g,
                           "sym" if c["zp"] is None else "asym", scale_dtype, compute_dtype)


def to_weight(qweight, scales, qzeros, g_idx=None, *, comp=None, queue=None, **q_config):
    """HF quantised linear -> device-resident weight (no intermediate blob)."""
    from . import Weight, W_S4, W_S8, S_F32, COMP_INT8
    c = to_canonical(qweight, scales, qzeros, g_idx, **q_config)
    bits, g = q_config.get("bits", 4), q_config.get("group_size", 128)
    shuffle = None
    if c["g_idx"] is not None:
        shuffle = np.argsort(c["g_idx"], kind="stable").astype(np.int32)   # setShuffleIndices, bestla_prologue_b.h:337-356
    return Weight.from_unpacked(c["q"], c["scales"], c["zp"], g, W_S4 if bits == 4 else W_S8, S_F32,
                                COMP_INT8 if comp is None else comp, shuffle=shuffle)

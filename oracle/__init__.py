"""CPU oracle for the weight-only matmul hot path -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference``
legs may import this package.  It wraps

* ``oracle/liboracle.so``   -- our plain-C restatement (oracle_ggml.c, oracle_btla.c), and
* ``oracle/_ref/*.so``      -- the reference's own sources compiled in place (ref_ggml.c, ref_btla.cpp),
  present when built in a container that has ``/root/reference`` (the built .so travels to the GPU box).

Parity status: PINNED (tests/test_oracle_vs_ref.py + tests/golden/).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
_i8p = np.ctypeslib.ndpointer(np.int8, flags="C_CONTIGUOUS")
_u8p = np.ctypeslib.ndpointer(np.uint8, flags="C_CONTIGUOUS")
_i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")

Q4_0_BLOCK_BYTES = 18
Q8_0_BLOCK_BYTES = 34
BTLA_S4_CLIP = 4 | (1 << 8)
BTLA_S8 = 8 | (1 << 8)
BTLA_F32 = 32
BTLA_BF16 = 16 | (1 << 16)


def build(force: bool = False) -> None:
    """Compile liboracle.so and (when /root/reference exists) oracle/_ref/."""
    need = force or not os.path.exists(os.path.join(_HERE, "liboracle.so"))
    if os.path.isdir("/root/reference/neural_speed") and not all(
            os.path.exists(os.path.join(_HERE, "_ref", f)) for f in ("libref_ggml.so", "libref_btla.so", "libref_ne.so")):
        need = True
    if need:
        subprocess.run(["make", "-C", _HERE, "-s"] + (["-B"] if force else []), check=True)


_lib = None
_ref_ggml = None
_ref_btla = None
_ref_ne = None


def ref_ne():
    """The reference's graph engine (core/ne_layers.c through its public API; oracle/_ref/libref_ne.so) or None."""
    global _ref_ne
    if _ref_ne is None:
        p = os.path.join(_HERE, "_ref", "libref_ne.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        L.ref_ne_rope.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float]
        L.ref_ne_soft_max.argtypes = [C.c_void_p, C.c_int, C.c_int]
        L.ref_ne_rms_norm.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_float]
        L.ref_ne_attn_1tok.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float]
        for f in (L.ref_ne_rope, L.ref_ne_soft_max, L.ref_ne_rms_norm, L.ref_ne_attn_1tok):
            f.restype = None
        _bind_llama(L)
        _ref_ne = L
    return _ref_ne


def _bind_llama(L):
    L.ref_ne_mul_mat_id.restype = None
    L.ref_ne_mul_mat_id.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p,
                                    C.c_int, C.c_void_p, C.c_int]
    L.ref_ne_llama_create.restype = C.c_void_p
    L.ref_ne_llama_create.argtypes = [C.c_int] * 7 + [C.c_float] * 3
    L.ref_ne_llama_create_ex.restype = C.c_void_p
    L.ref_ne_llama_create_ex.argtypes = [C.c_int] * 7 + [C.c_float] * 3 + [C.c_int, C.c_void_p, C.c_int, C.c_int]
    L.ref_ne_llama_set.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    L.ref_ne_llama_eval.restype = None
    L.ref_ne_llama_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.ref_ne_llama_free.restype = None
    L.ref_ne_llama_free.argtypes = [C.c_void_p]



def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(os.path.join(_HERE, "liboracle.so"))
        L.orc_fp16_to_fp32.restype = C.c_float
        L.orc_fp16_to_fp32.argtypes = [C.c_uint16]
        L.orc_fp32_to_fp16.restype = C.c_uint16
        L.orc_fp32_to_fp16.argtypes = [C.c_float]
        L.orc_f32_to_bf16.restype = C.c_uint16
        L.orc_f32_to_bf16.argtypes = [C.c_float]
        L.orc_bf16_to_f32.restype = C.c_float
        L.orc_bf16_to_f32.argtypes = [C.c_uint16]
        L.orc_nf4_unpack.restype = C.c_float
        L.orc_nf4_unpack.argtypes = [C.c_int]
        L.orc_nf4_quantize.restype = C.c_int
        L.orc_nf4_quantize.argtypes = [C.c_float]
        L.orc_silu.restype = C.c_float
        L.orc_silu.argtypes = [C.c_float]
        for n, r in (("orc_cast_f32_s8", C.c_int8), ("orc_cast_f32_u8", C.c_uint8), ("orc_cast_f32_s32", C.c_int)):
            getattr(L, n).restype = r
            getattr(L, n).argtypes = [C.c_float]
        _lib = L
    return _lib


def ref_ggml():
    """The reference's own ggml Q4_0/Q8_0 code (oracle/_ref/libref_ggml.so) or None."""
    global _ref_ggml
    if _ref_ggml is None:
        p = os.path.join(_HERE, "_ref", "libref_ggml.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        L.ref_ggml_init()
        L.ref_fp16_to_fp32.restype = C.c_float
        L.ref_fp16_to_fp32.argtypes = [C.c_uint16]
        L.ref_fp32_to_fp16.restype = C.c_uint16
        L.ref_fp32_to_fp16.argtypes = [C.c_float]
        _ref_ggml = L
    return _ref_ggml


def ref_btla():
    """The reference's kernel_ref.h (oracle/_ref/libref_btla.so) or None."""
    global _ref_btla
    if _ref_btla is None:
        p = os.path.join(_HERE, "_ref", "libref_btla.so")
        if not os.path.exists(p):
            try:
                build()
            except Exception:
                pass
        if not os.path.exists(p):
            return None
        L = C.CDLL(p)
        L.ref_btla_nf4_unpack.restype = C.c_float
        L.ref_btla_nf4_unpack.argtypes = [C.c_int8]
        L.ref_btla_nf4_quantize.restype = C.c_int8
        L.ref_btla_nf4_quantize.argtypes = [C.c_float]
        L.ref_btla_f32_to_bf16.restype = C.c_uint16
        L.ref_btla_f32_to_bf16.argtypes = [C.c_float]
        L.ref_btla_bf16_to_f32.restype = C.c_float
        L.ref_btla_bf16_to_f32.argtypes = [C.c_uint16]
        L.ref_btla_cast_f32_s8.restype = C.c_int8
        L.ref_btla_cast_f32_s8.argtypes = [C.c_float]
        L.ref_btla_cast_f32_u8.restype = C.c_uint8
        L.ref_btla_cast_f32_u8.argtypes = [C.c_float]
        L.ref_btla_cast_f32_s32.restype = C.c_int
        L.ref_btla_cast_f32_s32.argtypes = [C.c_float]
        _ref_btla = L
    return _ref_btla


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _c(a, dt):
    return np.ascontiguousarray(a, dtype=dt)


# ----------------------------------------------------------------------------- ggml Q4_0 / Q8_0
def _rowwise(fn, x, out_bytes_per_block):
    x = _c(x, np.float32)
    rows, k = x.reshape(-1, x.shape[-1]).shape
    assert k % 32 == 0
    out = np.empty((rows, k // 32 * out_bytes_per_block), np.uint8)
    x2 = x.reshape(rows, k)
    for r in range(rows):
        fn(_p(x2[r]), _p(out[r]), C.c_int(k))
    return out


def quantize_q4_0(w, impl="oracle"):
    """w [N,K] f32 -> uint8 [N, K/32*18] (block_q4_0 rows)."""
    L = lib() if impl == "oracle" else ref_ggml()
    fn = L.orc_quantize_row_q4_0 if impl == "oracle" else L.ref_quantize_row_q4_0
    return _rowwise(fn, w, Q4_0_BLOCK_BYTES)


def quantize_q8_0(x, impl="oracle", variant="runtime"):
    """x [M,K] f32 -> uint8 [M, K/32*34] (block_q8_0 rows). variant: 'runtime' (x86 body) | 'reference'."""
    if impl == "oracle":
        fn = lib().orc_quantize_row_q8_0 if variant == "runtime" else lib().orc_quantize_row_q8_0_reference
    else:
        fn = ref_ggml().ref_quantize_row_q8_0 if variant == "runtime" else ref_ggml().ref_quantize_row_q8_0_reference
    return _rowwise(fn, x, Q8_0_BLOCK_BYTES)


def dequantize_q4_0(wq, k, impl="oracle"):
    wq = _c(wq, np.uint8)
    out = np.empty((wq.shape[0], k), np.float32)
    fn = lib().orc_dequantize_row_q4_0 if impl == "oracle" else ref_ggml().ref_dequantize_row_q4_0
    for r in range(wq.shape[0]):
        fn(_p(wq[r]), _p(out[r]), C.c_int(k))
    return out


def dequantize_q8_0(xq, k, impl="oracle"):
    xq = _c(xq, np.uint8)
    out = np.empty((xq.shape[0], k), np.float32)
    fn = lib().orc_dequantize_row_q8_0 if impl == "oracle" else ref_ggml().ref_dequantize_row_q8_0
    for r in range(xq.shape[0]):
        fn(_p(xq[r]), _p(out[r]), C.c_int(k))
    return out


def vec_dot_q4_0_q8_0(wrow, arow, k, impl="oracle", scalar=False):
    s = C.c_float()
    if impl == "oracle":
        fn = lib().orc_vec_dot_q4_0_q8_0_scalar if scalar else lib().orc_vec_dot_q4_0_q8_0
    else:
        fn = ref_ggml().ref_vec_dot_q4_0_q8_0
    fn(C.c_int(k), C.byref(s), _p(_c(wrow, np.uint8)), _p(_c(arow, np.uint8)))
    return np.float32(s.value)


def block_isum_q4_0_q8_0(wrow, arow, k):
    out = np.empty(k // 32, np.int32)
    lib().orc_block_isum_q4_0_q8_0(C.c_int(k), _p(out), _p(_c(wrow, np.uint8)), _p(_c(arow, np.uint8)))
    return out


def mul_mat_q4_0_f32(wq, a, impl="oracle", nth=0):
    """wq uint8 [N, K/32*18], a f32 [M,K] -> f32 [M,N] (ne_compute_forward_mul_mat_q_f32 semantics)."""
    wq = _c(wq, np.uint8)
    a = _c(a, np.float32)
    m, k = a.shape
    n = wq.shape[0]
    assert wq.shape[1] == k // 32 * Q4_0_BLOCK_BYTES
    dst = np.empty((m, n), np.float32)
    wdata = np.empty(m * (k // 32) * Q8_0_BLOCK_BYTES + 64, np.uint8)
    fn = lib().orc_mul_mat_q4_0_f32 if impl == "oracle" else ref_ggml().ref_mul_mat_q4_0_f32
    fn.restype = C.c_int
    used = fn(_p(wq), _p(a), _p(dst), C.c_int(n), C.c_int(k), C.c_int(m), _p(wdata), C.c_int(nth))
    mul_mat_q4_0_f32.threads_used = used
    return dst


# ----------------------------------------------------------------------------- ggml Q6_K / Q8_K
Q6_K_BLOCK_BYTES = 210   # block_q6_K, data_types.h:133-138
Q8_K_BLOCK_BYTES = 292   # block_q8_K, data_types.h:140-144


def _rowwise_k(fn, x, out_bytes_per_block):
    x = _c(x, np.float32)
    rows, k = x.reshape(-1, x.shape[-1]).shape
    assert k % 256 == 0
    out = np.zeros((rows, k // 256 * out_bytes_per_block), np.uint8)
    x2 = x.reshape(rows, k)
    for r in range(rows):
        fn(_p(x2[r]), _p(out[r]), C.c_int(k))
    return out


def quantize_q6_K(w, impl="oracle"):
    """w [N,K] f32 -> uint8 [N, K/256*210] (block_q6_K rows)."""
    fn = lib().orc_quantize_row_q6_K if impl == "oracle" else ref_ggml().ref_quantize_row_q6_K
    return _rowwise_k(fn, w, Q6_K_BLOCK_BYTES)


def quantize_q8_K(x, impl="oracle"):
    """x [M,K] f32 -> uint8 [M, K/256*292] (block_q8_K rows)."""
    fn = lib().orc_quantize_row_q8_K if impl == "oracle" else ref_ggml().ref_quantize_row_q8_K
    return _rowwise_k(fn, x, Q8_K_BLOCK_BYTES)


def dequantize_q6_K(wq, k, impl="oracle"):
    wq = _c(wq, np.uint8)
    out = np.empty((wq.shape[0], k), np.float32)
    fn = lib().orc_dequantize_row_q6_K if impl == "oracle" else ref_ggml().ref_dequantize_row_q6_K
    for r in range(wq.shape[0]):
        fn(_p(wq[r]), _p(out[r]), C.c_int(k))
    return out


def vec_dot_q6_K_q8_K(wrow, arow, k, impl="oracle"):
    s = C.c_float()
    fn = lib().orc_vec_dot_q6_K_q8_K if impl == "oracle" else ref_ggml().ref_vec_dot_q6_K_q8_K
    fn(C.c_int(k), C.byref(s), _p(_c(wrow, np.uint8)), _p(_c(arow, np.uint8)))
    return np.float32(s.value)


def mul_mat_q6_K_f32(wq, a, impl="oracle", nth=0):
    """wq uint8 [N, K/256*210], a f32 [M,K] -> f32 [M,N]."""
    wq = _c(wq, np.uint8)
    a = _c(a, np.float32)
    m, k = a.shape
    n = wq.shape[0]
    assert wq.shape[1] == k // 256 * Q6_K_BLOCK_BYTES
    dst = np.empty((m, n), np.float32)
    wdata = np.zeros(m * (k // 256) * Q8_K_BLOCK_BYTES + 64, np.uint8)
    fn = lib().orc_mul_mat_q6_K_f32 if impl == "oracle" else ref_ggml().ref_mul_mat_q6_K_f32
    fn.restype = C.c_int
    fn(_p(wq), _p(a), _p(dst), C.c_int(n), C.c_int(k), C.c_int(m), _p(wdata), C.c_int(nth))
    return dst


NE_TYPE_Q4_0, NE_TYPE_BTLA = 2, 19  # enum ne_type (core/data_types.h:32-55)


def _blob_table(blobs):
    blobs = [np.ascontiguousarray(b) for b in blobs]
    ptrs = (C.c_void_p * len(blobs))(*[b.ctypes.data for b in blobs])
    sizes = (C.c_size_t * len(blobs))(*[b.nbytes for b in blobs])
    return blobs, ptrs, sizes


def ref_mul_mat_id(L, experts, wtype, n, k, ids, id, b, n_threads=1):
    """ne_mul_mat_id through the REFERENCE's engine L (ref_ne()): NE_TYPE_Q4_0 experts.
    experts: list of Q4_0 row arrays / BesTLA blobs; ids int32 [n_tok][n_used]; b fp32 [n_tok][k] -> [n_tok][n]."""
    keep, ptrs, sizes = _blob_table(experts)
    ids = np.ascontiguousarray(ids, np.int32)
    b = np.ascontiguousarray(b, np.float32)
    out = np.zeros((b.shape[0], n), np.float32)
    L.ref_ne_mul_mat_id(ptrs, sizes, wtype, len(keep), n, k, _p(ids), ids.shape[1], id, _p(b), b.shape[0], _p(out), n_threads)
    return out


def mul_mat_id_q4_0_f32(expert_rows, ids, id, a):
    """Restatement of ne_compute_forward_mul_mat_id_q_f32 (core/ne_layers.c:7345-7498) for Q4_0 experts: token t takes expert
    ids[t][id]; its row is quantised to Q8_0 (NE_TASK_INIT, :7418-7431) and dotted with every weight row of that expert."""
    ids = np.asarray(ids, np.int32)
    a = np.ascontiguousarray(a, np.float32)
    n = expert_rows[0].shape[0]
    out = np.zeros((a.shape[0], n), np.float32)
    for t in range(a.shape[0]):
        e = int(ids[t, id])
        assert 0 <= e < len(expert_rows)  # NE_ASSERT(row_id >= 0 && row_id < n_as), :7445
        out[t] = mul_mat_q4_0_f32(expert_rows[e], a[t:t + 1])[0]
    return out


def argmax(x):
    x = _c(x, np.float32).ravel()
    lib().orc_argmax_f32.restype = C.c_int
    return int(lib().orc_argmax_f32(_p(x), C.c_int(x.size)))


# ----------------------------------------------------------------------------- BesTLA
def btla_quantize(w_kn, g, nbits=4, asym=False, impl="oracle"):
    """RTN quantise W [K,N] f32 -> (q int8 [K,N], scales f32 [ceil(K/g),N], zps int8 [..] | None)."""
    w = _c(w_kn, np.float32)
    k, n = w.shape
    nb = (k + g - 1) // g
    q = np.zeros((k, n), np.int8)
    sc = np.zeros((nb, n), np.float32)
    zp = np.zeros((nb, n), np.int8) if asym else None
    if impl == "oracle":
        lib().orc_btla_quantize_rowblock(_p(w), _p(q), C.c_int(k), C.c_int(n), C.c_int(n), C.c_int(n), _p(sc),
                                         _p(zp) if asym else None, C.c_int(g), C.c_int(nbits))
    else:
        qt = nbits | (1 << 8)  # S{n}_CLIP / S8 = EleBits | TypeInt (bestla.h:38-87)
        ref_btla().ref_btla_quantize_f32_sign_int_rowblock(_p(w), _p(q), C.c_int(k), C.c_int(n), C.c_int(n), C.c_int(n),
                                                           _p(sc), _p(zp) if asym else None, C.c_int(g), C.c_uint32(qt))
    return q, sc, zp


def btla_quantize_nf4(w_kn, g, impl="oracle"):
    w = _c(w_kn, np.float32)
    k, n = w.shape
    nb = (k + g - 1) // g
    q = np.zeros((k, n), np.int8)
    sc = np.zeros((nb, n), np.float32)
    if impl == "oracle":
        lib().orc_btla_quantize_nf4_rowblock(_p(w), _p(q), C.c_int(k), C.c_int(n), C.c_int(n), C.c_int(n), _p(sc), C.c_int(g))
    else:
        ref_btla().ref_btla_quantize_f32_nf4_rowblock(_p(w), _p(q), C.c_int(k), C.c_int(n), C.c_int(n), C.c_int(n), _p(sc),
                                                      C.c_int(g))
    return q, sc


def btla_dequant(q, sc, zp, g, nf4=False):
    q = _c(q, np.int8)
    k, n = q.shape
    w = np.empty((k, n), np.float32)
    lib().orc_btla_dequant(_p(q), _p(_c(sc, np.float32)), _p(_c(zp, np.int8)) if zp is not None else None, _p(w),
                           C.c_int(k), C.c_int(n), C.c_int(g), C.c_int(1 if nf4 else 0))
    return w


def btla_quantize_act_u8(a, g, impl="oracle", want_reduce=False):
    a = _c(a, np.float32)
    m, k = a.shape
    nb = (k + g - 1) // g
    q = np.zeros((m, k), np.uint8)
    sc = np.zeros((m, nb), np.float32)
    zp = np.zeros((m, nb), np.uint8)
    red = np.zeros((m, nb), np.float32) if want_reduce else None
    if impl == "oracle":
        lib().orc_btla_quantize_act_u8(C.c_int(m), C.c_int(k), _p(a), C.c_int(k), _p(q), C.c_int(k), _p(sc), C.c_int(nb),
                                       _p(zp), C.c_int(g), _p(red) if want_reduce else None)
    else:
        ref_btla().ref_btla_quantize_fp_u8_colblock(C.c_int(m), C.c_int(k), _p(a), C.c_int(k), _p(q), C.c_int(k), _p(sc),
                                                    C.c_int(nb), _p(zp), C.c_int(g), _p(red) if want_reduce else None)
    return (q, sc, zp, red) if want_reduce else (q, sc, zp)


def btla_quantize_act_s8(a, g, impl="oracle"):
    a = _c(a, np.float32)
    m, k = a.shape
    nb = (k + g - 1) // g
    q = np.zeros((m, k), np.int8)
    sc = np.zeros((m, nb), np.float32)
    if impl == "oracle":
        lib().orc_btla_quantize_act_s8(C.c_int(m), C.c_int(k), _p(a), C.c_int(k), _p(q), C.c_int(k), _p(sc), C.c_int(nb),
                                       C.c_int(g), None)
    else:
        ref_btla().ref_btla_quantize_fp_s8_colblock(C.c_int(m), C.c_int(k), _p(a), C.c_int(k), _p(q), C.c_int(k), _p(sc),
                                                    C.c_int(nb), C.c_int(g), None)
    return q, sc


def btla_gemv_fp32(a, q, sc, zp, g):
    a = _c(a, np.float32)
    m, k = a.shape
    n = q.shape[1]
    c = np.empty((m, n), np.float32)
    lib().orc_btla_gemv_fp32(_p(a), C.c_int(k), _p(_c(q, np.int8)), _p(_c(sc, np.float32)),
                             _p(_c(zp, np.int8)) if zp is not None else None, _p(c), C.c_int(n), C.c_int(m), C.c_int(n),
                             C.c_int(k), C.c_int(g))
    return c


def btla_gemv_u8s8(a8, asc, azp, q, sc, zp, g, blocksum=False):
    a8 = _c(a8, np.uint8)
    m, k = a8.shape
    n = q.shape[1]
    nb = asc.shape[1]
    c = np.empty((m, n), np.float32)
    fn = lib().orc_btla_gemv_u8s8_blocksum if blocksum else lib().orc_btla_gemv_u8s8
    fn(_p(a8), _p(_c(asc, np.float32)), _p(_c(azp, np.uint8)), C.c_int(k), C.c_int(nb), _p(_c(q, np.int8)),
       _p(_c(sc, np.float32)), _p(_c(zp, np.int8)) if zp is not None else None, _p(c), C.c_int(n), C.c_int(m), C.c_int(n),
       C.c_int(k), C.c_int(g))
    return c


def btla_gemv_s8s8(a8, asc, q, sc, zp, g):
    a8 = _c(a8, np.int8)
    m, k = a8.shape
    n = q.shape[1]
    nb = asc.shape[1]
    c = np.empty((m, n), np.float32)
    lib().orc_btla_gemv_s8s8(_p(a8), _p(_c(asc, np.float32)), C.c_int(k), C.c_int(nb), _p(_c(q, np.int8)),
                             _p(_c(sc, np.float32)), _p(_c(zp, np.int8)) if zp is not None else None, _p(c), C.c_int(n),
                             C.c_int(m), C.c_int(n), C.c_int(k), C.c_int(g))
    return c


def gemm_f64acc(a, w_kn):
    a = _c(a, np.float32)
    w = _c(w_kn, np.float32)
    m, k = a.shape
    n = w.shape[1]
    c = np.empty((m, n), np.float32)
    lib().orc_gemm_f64acc(_p(a), C.c_int(k), _p(w), _p(c), C.c_int(n), C.c_int(m), C.c_int(n), C.c_int(k))
    return c


def f32_to_bf16_bits(x):
    """RNE fp32 -> bf16 bit pattern (bestla_utils.h:146-153), vectorised."""
    u = _c(x, np.float32).view(np.uint32).astype(np.uint64)
    u = u + 0x7FFF + ((u >> 16) & 1)
    return ((u >> 16) & 0xFFFF).astype(np.uint16)


def bf16_bits_to_f32(b):
    return (np.asarray(b, np.uint16).astype(np.uint32) << 16).view(np.float32)


class RefNeLlama:
    """A Llama model evaluated by the REFERENCE's own graph engine (oracle/ref_ne.c: core/ne_layers.c through the public ne_*
    API, graph of models/llama/llama.cpp).  Same constructor arguments as oracle.llama_model.OracleLlama (Q4_0 weights; GQA
    through ne_mul_mat's head broadcast).  Only available where oracle/_ref was built (needs /root/reference)."""

    NAMES = ["attn_norm", "wq", "wk", "wv", "wo", "ffn_norm", "w1", "w2", "w3"]
    NE_TYPE_Q4_0 = 2  # core/data_types.h:32-55

    def __init__(self, hp, tok_embd, out_norm, output_rows, layers, fused=True, n_threads=1):
        """fused: ne_mul_qkv / ne_ffn_silu nodes where the *_support probes agree."""
        L = ref_ne()
        if L is None:
            raise RuntimeError("oracle/_ref/libref_ne.so not built")
        self.L, self.n_vocab = L, hp["n_vocab"]
        self.h = C.c_void_p(L.ref_ne_llama_create_ex(hp["n_vocab"], hp["n_embd"], hp["n_head"], hp["n_head_kv"], hp["n_layer"], hp["n_ff"],
                                                     hp["n_ctx"], hp.get("norm_eps", 1e-6), hp.get("rope_theta", 10000.0),
                                                     hp.get("rope_scale", 1.0), self.NE_TYPE_Q4_0, None, 1 if fused else 0, n_threads))

        def put(layer, which, arr, dt):
            a = _c(arr, dt)
            assert L.ref_ne_llama_set(self.h, layer, which, _p(a), a.nbytes) == 0, (layer, which, a.nbytes)

        put(0, -1, tok_embd, np.float32)
        put(0, -2, out_norm, np.float32)
        put(0, -3, output_rows, np.uint8)
        for il, lay in enumerate(layers):
            for j, name in enumerate(self.NAMES):
                put(il, j, lay[name], np.float32 if "norm" in name else np.uint8)

    def eval(self, tokens, n_past):
        t = _c(tokens, np.int32)
        logits = np.zeros(self.n_vocab, np.float32)
        self.L.ref_ne_llama_eval(self.h, _p(t), t.size, n_past, _p(logits))
        return logits

    def close(self):
        if self.h:
            self.L.ref_ne_llama_free(self.h)
            self.h = None

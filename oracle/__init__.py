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


# Float-compute GEMV bar: |got - model| <= GEMV_F32_C * sqrt(K) * 2^-24 * sum_k |a_eff w_eff| per output, model = the fp64 sum.
# Measured on an H100 80GB HBM3 (700 W limit; tests/test_gpu_gemv.py, uniform(-0.5, 0.5) data, K = 1000 .. 51200): at most 0.0116
# of the unit bar.  Dropping the bf16 rounding of the activations moves a bf16-compute output by 4 (K = 28672) to 30 (K = 4128).
GEMV_F32_C = 0.05


def gemv_stated(a_eff, w_eff):
    """fp64 model of a GEMV in fp32 arithmetic on its effective operands (bf16-rounded activations for bf16 compute, dequantised
    fp32 weights [K,N]): (sum_k a_eff w_eff, sum_k |a_eff w_eff|), each [M,N] float64."""
    a = np.asarray(a_eff, np.float64)
    w = np.asarray(w_eff, np.float64)
    return a @ w, np.abs(a) @ np.abs(w)


def gemv_bound_ratio(got, a_eff, w_eff):
    """max over outputs of |got - model| / (sqrt(K) * 2^-24 * sum_k |a_eff w_eff|); a float-compute GEMV stays below GEMV_F32_C"""
    want, mag = gemv_stated(a_eff, w_eff)
    unit = np.sqrt(np.asarray(a_eff).shape[1]) * 2.0 ** -24 * np.maximum(mag, np.finfo(np.float32).tiny)
    return float((np.abs(np.asarray(got, np.float64) - want) / unit).max())


# 4-bit float codebooks by code (sign in bit 3 for the FP4 ones): FP4 "BNB" and FP4 E2M1 (kernel_ref.h:1209-1230, :1300-1321);
# NF4 comes from liboracle (orc_nf4_unpack)
_F4_BNB = [0.0, 5.208333333e-03, 0.66666667, 1.0, 0.33333333, 0.5, 0.16666667, 0.25]
_F4_E2M1 = [0.0, 0.010416666666666666, 0.16666666666666666, 0.25, 0.3333333333333333, 0.5, 0.6666666666666666, 1.0]


def f4_levels(kind):
    """the 16 fp32 levels of codebook 'nf4', 'f4_bnb' or 'f4_e2m1', indexed by code"""
    if kind == "nf4":
        return np.array([lib().orc_nf4_unpack(c) for c in range(16)], np.float32)
    half = np.array(_F4_BNB if kind == "f4_bnb" else _F4_E2M1, np.float32)
    return np.concatenate([half, -half])


def _bf16(x):
    return bf16_bits_to_f32(f32_to_bf16_bits(np.asarray(x, np.float32)))


def tc_operands(a, fmt, q=None, scales=None, zp=None, group=32, stype="f32", shuffle=None):
    """The operands of the wgmma GEMM (gemm_w4_tc_kernel, DESIGN.md section 4): (a_eff [M,K], w_eff [K,N]), bf16 values in fp32.
      a        fp32 [M,K] (None: a_eff is None); with an act-order shuffle (int [K]) image column k is a[:, shuffle[k]]
      fmt      's4' / 's8': q = signed integer codes, zp [ceil(K/g),N] or None;  'nf4' / 'f4_bnb' / 'f4_e2m1': q = codebook
               codes 0..15;  'q4_0': q = nibble - 8;  'q8_0': q = int8 codes (both: group 32, fp16 d)
      scales   [ceil(K/g),N] as handed to the weight loader, stored as stype 'f32' / 'bf16' / 'f16' (round to nearest even)
    a_eff = bf16_rn(a).  With s = bf16_rn(stored scale, widened to fp32):
      integer codes  w_eff = bf16_rn(bf16(q - zp) * s)          (q - zp is exact in bf16: |q - zp| <= 255)
      codebooks      w_eff = bf16_rn(bf16_rn(level[q]) * s)
    Products of two bf16 values are exact in fp32, so each bf16_rn above is the kernel's single rounding of an HMUL2."""
    a_eff = None
    if a is not None:
        a = np.asarray(a, np.float32)
        a_eff = _bf16(a[:, np.asarray(shuffle)] if shuffle is not None else a)
    qi = np.asarray(q, np.int32)
    k = qi.shape[0]
    if fmt in ("q4_0", "q8_0"):
        group, stype, zp = 32, "f16", None
    sc = np.asarray(scales, np.float32)
    if stype == "bf16":
        sc = _bf16(sc)
    elif stype == "f16":
        sc = sc.astype(np.float16).astype(np.float32)
    s = _bf16(sc)[np.arange(k) // group]
    if fmt in ("nf4", "f4_bnb", "f4_e2m1"):
        base = _bf16(f4_levels(fmt)[qi])
    else:
        d = qi - (np.asarray(zp, np.int32)[np.arange(k) // group] if zp is not None else 0)
        assert np.abs(d).max(initial=0) <= 255
        base = d.astype(np.float32)
    return a_eff, _bf16(base * s)


def tc_grid(a_eff, w_eff):
    """log2 of the finest product grid of two bf16 operand sets: min lsb(a) + min lsb(w), lsb(v) = floor(log2|v|) - 7 (the weight of
    the last of a bf16 value's 8 significand bits).  Every product a * w is an integer multiple of 2^grid."""
    def lsb(x):
        x = np.abs(np.asarray(x, np.float64))
        return int(np.floor(np.log2(x[x > 0].min()))) - 7
    return lsb(a_eff) + lsb(w_eff)


def tc_exact_budget(a_eff, w_eff, mag=None, extra=None):
    """max over outputs of (sum_k |a_eff w_eff| [+ extra]) in units of 2^tc_grid.  Below 2^24 every partial sum of the products
    (and of extra, when its terms lie on the grid), in any order and any split, is an integer multiple of the grid below 2^24
    of it: an exact fp32 value, so an fp32 accumulation gives the fp64 sum bit for bit.  mag: gemv_stated's second output, if
    already computed; extra: [M,N] magnitudes of the epilogue's addends (|bias| + |residual|)."""
    if mag is None:
        mag = gemv_stated(a_eff, w_eff)[1]
    if extra is not None:
        mag = mag + np.asarray(extra, np.float64)
    return float(np.max(mag)) / 2.0 ** tc_grid(a_eff, w_eff)


def imma_act(a, comp, g):
    """The activations of an integer block-sum matmul as the quantisers give them: (codes - zero point) int64 [M,K], scales fp32
    [M, K/ab] and the activation block ab.  comp: 'q8_0' (quantize_row_q8_0: blocks of 32, fp16 d), 'int8' (u8 with zero points
    per weight group) or 'int8_s8' (s8 per weight group)."""
    a = _c(a, np.float32)
    m, k = a.shape
    if comp == "q8_0":
        blk = quantize_q8_0(a).reshape(m, k // 32, 34)
        codes = blk[:, :, 2:].copy().view(np.int8).reshape(m, k).astype(np.int64)
        return codes, blk[:, :, :2].copy().view(np.float16).reshape(m, k // 32).astype(np.float32), 32
    if comp == "int8":
        q, sc, zp = btla_quantize_act_u8(a, g)
        return q.astype(np.int64) - np.repeat(zp.astype(np.int64), g, axis=1)[:, :k], sc, g
    q, sc = btla_quantize_act_s8(a, g)
    return q.astype(np.int64), sc, g


def imma_stated(a_codes, a_scale, ab, q, w_scale, w_zp, g):
    """fp64 model of the integer block-sum matmul (gemm_imma_kernel, DESIGN.md section 4).  a_codes / a_scale / ab as imma_act;
    q int [K,N] signed weight codes, w_scale fp32 [K/g, N] as stored, w_zp [K/g, N] or None.  Per activation block b:
    isum_b = sum (a - za)(q - zp), an exact integer; c_b = fp32(a_scale_b * w_scale_b); t_b = isum_b * c_b (exact in fp64).
    Returns (sum_b t_b, sum_b |t_b|, number of blocks), [M,N] float64."""
    a = np.asarray(a_codes, np.float64)
    w = np.asarray(q, np.float64)
    k, n = w.shape
    if w_zp is not None:
        w = w - np.repeat(np.asarray(w_zp, np.float64), g, axis=0)[:k]
    asc, wsc = np.asarray(a_scale, np.float32), np.asarray(w_scale, np.float32)
    tot = np.zeros((a.shape[0], n))
    mag = np.zeros((a.shape[0], n))
    nb = k // ab
    for b in range(nb):
        isum = a[:, b * ab:(b + 1) * ab] @ w[b * ab:(b + 1) * ab]  # integers below 2^53: exact
        c = np.multiply(asc[:, b, None], wsc[b * ab // g][None, :], dtype=np.float32)
        t = isum * c.astype(np.float64)
        tot += t
        mag += np.abs(t)
    return tot, mag, nb


def imma_bound_ratio(got, tot, mag, nb, splits=16):
    """max over outputs of |got - sum t_b| / (gamma_n sum |t_b|), n = nb + splits: one fp32 fma per block and at most `splits`
    partial sums, each one rounding (gamma_n = n u / (1 - n u), u = 2^-24).  A correct kernel stays at or below 1."""
    n = nb + splits
    gam = n * 2.0 ** -24 / (1 - n * 2.0 ** -24)
    err = np.abs(np.asarray(got, np.float64) - tot)
    return float((err / np.maximum(gam * mag, np.finfo(np.float64).tiny)).max())


_F32_NORMAL = 2.0 ** -126


def _assert_normal(*arrs):
    for a in arrs:
        a = np.abs(np.asarray(a, np.float64))
        assert np.isfinite(a).all() and not ((a > 0) & (a < _F32_NORMAL)).any(), "subnormal or non-finite fp32 value"


def fma32(x, y, z):
    """fmaf(x, y, z) for arrays: the exact x * y + z rounded once to fp32 (nearest, ties to even).  x: fp32 values or integers
    below 2^29, y and z fp32, so x * y is exact in fp64; the fp64 sum is split into s + e exactly (TwoSum), and s rounds to the
    right fp32 unless it is an fp32 midpoint, where the sign of e decides.  Operands and results must be normal fp32 (asserted)."""
    x = np.asarray(x)
    if np.issubdtype(x.dtype, np.integer):
        assert np.abs(x).max(initial=0) < 2 ** 29
    else:
        assert x.dtype == np.float32, x.dtype
    y, z = np.asarray(y, np.float32), np.asarray(z, np.float32)
    _assert_normal(x, y, z)
    p, zd = x.astype(np.float64) * y.astype(np.float64), z.astype(np.float64)
    s = p + zd
    bb = s - zd
    e = (zd - (s - bb)) + (p - bb)  # s + e == p + z exactly
    r = s.astype(np.float32)
    d = s - r.astype(np.float64)   # exact
    nb = np.nextafter(r, np.where(d > 0, np.float32(np.inf), np.float32(-np.inf)))
    mid = (d != 0) & (2 * d == nb.astype(np.float64) - r.astype(np.float64))
    out = np.where(mid & (np.sign(e) == np.sign(d)), nb, r)
    _assert_normal(out)
    return out


def warp_butterfly(v):
    """lane 0 of warp_sum (nsb.cuh): v [32, ...] fp32 per lane, v_L += v_{L xor o} for o = 16, 8, 4, 2, 1, in fp32"""
    v = np.asarray(v, np.float32)
    assert v.shape[0] == 32
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        v = v + v[lanes ^ o]
    return v[0]


def ring_stated(a_codes, a_scale, ab, q, w_scale, w_zp, g, lanes=False):
    """The ring GEMV's exact fp32 result before its epilogue (gemv_ring_kernel, DESIGN.md section 4).  a_codes / a_scale / ab as
    imma_act (codes minus zero point [M, K], one scale per activation block of ab); q int [K, N] signed weight codes, w_scale
    [ceil(K/g), N] as stored, w_zp the same shape or None.  Per 32-element chunk c: isum_c = sum (a - za)(q - zp), an exact
    integer (the chunk's elements past K are zero), t_c = fp32(a_scale_c * w_scale_gi), gi = c // ceil(g / 32).  Lane L runs
    acc = fmaf(isum_c, t_c, acc) over c = L, L + 32, ... from +0; lane 0 of the xor butterfly is the output.
    Returns fp32 [M, N] (and with lanes=True the per-lane accumulators [32, M, N] too)."""
    a = np.asarray(a_codes, np.int64)
    m, k = a.shape
    w = np.asarray(q, np.int64)
    n = w.shape[1]
    cpg = -(-g // 32)
    nch = -(-k // 32)
    gi = np.arange(nch) // cpg
    if w_zp is not None:
        w = w - np.asarray(w_zp, np.int64)[gi].repeat(32, axis=0)[:k]
    ap = np.zeros((m, nch * 32), np.float64)
    ap[:, :k] = a
    wp = np.zeros((nch * 32, n), np.float64)
    wp[:k] = w
    # integers below 2^17 per chunk: exact in fp64 whatever the summation order
    isum = np.matmul(ap.reshape(m, nch, 32).transpose(1, 0, 2), wp.reshape(nch, 32, n))  # [nch, M, N]
    assert np.abs(isum).max(initial=0) < 2 ** 17
    asc = np.asarray(a_scale, np.float32)[:, (np.arange(nch) * 32) // ab]                 # [M, nch]
    wsc = np.asarray(w_scale, np.float32)[gi]                                             # [nch, N]
    t = asc.T[:, :, None] * wsc[:, None, :]                                                # fp32 products [nch, M, N]
    nst = -(-nch // 32)
    acc = np.zeros((32, m, n), np.float32)
    for j in range(nst):
        c0, c1 = 32 * j, min(32 * j + 32, nch)
        live = c1 - c0
        acc[:live] = fma32(isum[c0:c1].astype(np.int64), t[c0:c1], acc[:live])
    out = warp_butterfly(acc)
    return (out, acc) if lanes else out


def ring_norm_row(x, w, eps, nt):
    """The fp32 row the ring GEMV's fused RMSNorm prologue hands to its quantiser (quantise_to_smem, csrc/gemv_ring_impl.cuh) for a
    CTA of nt consumer threads (224: the two-CTA kernel, 448: the wide one).  Thread i owns the 8-groups i, i + nt, ... and runs
    ss = fmaf(v, v, ss) over them in that order (single-pass and multi-pass rows visit them alike); each warp's lane 0 of the
    xor butterfly, summed in warp order from 0; inv = 1 / sqrtf(tot / k + eps); row = (x * inv) * w, all fp32."""
    x = np.asarray(x, np.float32).ravel()
    wn = np.asarray(w, np.float32).ravel()
    k = x.size
    ng8 = -(-k // 32) * 4
    npass = -(-ng8 // nt)
    v = np.zeros(npass * nt * 8, np.float32)
    v[:k] = x
    v = v.reshape(npass, nt, 8)
    ss = np.zeros(nt, np.float32)
    for j in range(npass):
        for i in range(8):
            ss = fma32(v[j, :, i], v[j, :, i], ss)
    tot = np.float32(0)
    for wp in range(nt // 32):
        tot = np.float32(tot + warp_butterfly(ss[32 * wp:32 * wp + 32]))
    inv = np.float32(1) / np.sqrt(np.float32(tot / np.float32(k)) + np.float32(eps))
    return (x * np.float32(inv)) * wn


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

"""Generate tests/golden/ggml_q8_0.npz from the REFERENCE's own ggml code (oracle/_ref/libref_ggml.so = /root/reference compiled in
place): ne_quantize_q8_0's weight rows (quantize_row_q8_0_reference), quantize_row_q8_0 activations, dequantize_row_q8_0, and
the reference's ne_vec_dot_q8_0_q8_0 looped over every (activation row, weight row) pair on the quantised activations -- the two
phases ne_compute_forward_mul_mat_q_f32 runs for NE_TYPE_Q8_0 (INIT: quantize_row_q8_0 per row, COMPUTE: that vec_dot per pair),
composed here from the exported functions rather than called as one.

Run where the reference sources are present:  python tests/golden/make_golden_q8_0.py
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
import oracle  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))


def ref_mul_mat_q8_0(wq, a):
    R = oracle.ref_ggml()
    m, k = a.shape
    aq = oracle.quantize_q8_0(a, "ref", "runtime")
    out = np.empty((m, wq.shape[0]), np.float32)
    s = C.c_float()
    for i in range(m):
        for n in range(wq.shape[0]):
            R.ref_vec_dot_q8_0_q8_0(C.c_int(k), C.byref(s), wq[n].ctypes.data_as(C.c_void_p), aq[i].ctypes.data_as(C.c_void_p))
            out[i, n] = s.value
    return aq, out


def main():
    assert oracle.ref_ggml() is not None, "needs oracle/_ref (build with the reference sources)"
    rng = np.random.default_rng(1234)
    N, K, M = 64, 512, 5
    w = rng.normal(0, 0.02, (N, K)).astype(np.float32)
    w[3, :32] = 0.0                       # an all-zero block: d = 0
    a = rng.normal(0, 1.0, (M, K)).astype(np.float32)
    a[1, :32] = 0.0
    wq = oracle.quantize_q8_0(w, "ref", "reference")
    wq = np.ascontiguousarray(wq)
    b = wq.reshape(N, K // 32, 34)
    b[5, 2, 2:] = np.uint8(0x80)         # codes -128 (a file may hold them; the quantisers never write them)
    b[6, 1, 2:] = np.uint8(127)
    b[4, 1, :2] = np.array([0x0003], np.uint16).view(np.uint8)  # a subnormal fp16 d
    aq, out = ref_mul_mat_q8_0(wq, a)
    np.savez_compressed(os.path.join(HERE, "ggml_q8_0.npz"), w=w, a=a, wq=wq, aq=aq, out=out, wdq=oracle.dequantize_q8_0(wq, K, "ref"))


if __name__ == "__main__":
    main()

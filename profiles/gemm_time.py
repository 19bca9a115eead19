"""Time single wgmma GEMMs (CUDA events) -- tuning aid.  usage: python profiles/gemm_time.py [M]"""
import ctypes as C
import sys

import torch

import neural_speed_b200 as ns

M = int(sys.argv[1]) if len(sys.argv) > 1 else 2048
L = ns.lib()
L.bestla_init()


def mk(n, k):
    w = torch.randn(n, k, device="cuda") * 0.02
    rows = torch.empty(n * (k // 32) * 18, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    assert L.ns_device_quantize_q4_0(C.c_void_p(w.data_ptr()), C.c_void_p(rows.data_ptr()), n, k, None) == 0
    L.bestla_device_sync(None)
    return ns.Weight.from_q4_0_device(rows.data_ptr(), n, k, (k // 32) * 18)


for n, k in ((4096, 4096), (11008, 4096), (4096, 11008)):
    w = mk(n, k)
    x = torch.randn(M, k, device="cuda")
    o = torch.zeros(M, n, device="cuda")
    st = torch.cuda.Stream()  # NOT the legacy default stream: handle 0 would select the library's own stream
    q = C.c_void_p(st.cuda_stream)
    for _ in range(3):
        ns.mul_mat(w, x.data_ptr(), k, o.data_ptr(), n, M, queue=q)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record(st)
    for _ in range(20):
        ns.mul_mat(w, x.data_ptr(), k, o.data_ptr(), n, M, queue=q)
    e1.record(st)
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / 20
    print(f"M={M} N={n} K={k}: {ms * 1e3:.1f} us  {2.0 * M * n * k / ms / 1e9:.0f} TFLOP/s (incl. fp32->bf16 conversion)")

"""Decode speed of ggml Q8_0 weights: the ring GEMV per Llama-2-7B node and the whole decode step, against Q4_0.

Per node (q / k / v / o 4096 x 4096, gate / up 11008 x 4096, down 4096 x 11008, lm_head 32000 x 4096), one activation row,
ns_mul_mat as the eval step calls it (the kernel quantises its own activations), three weights of the same geometry called in
turn: Q8_0 (the ring GEMV on 8-bit codes), the register GEMV on the same kind of codes (NS_W_S8, group 32, fp16 scales,
NS_COMP_Q8_0) and Q4_0 (the ring GEMV on nibbles).  Weights are random codes generated on the device (the decode path is
bandwidth bound; its speed does not depend on the values).  Each format cycles through enough copies of the node's weight to
span more than 3x the 50 MB L2, so every call reads its weight from HBM, as in a decode step.  Time per call from CUDA events
around ITERS calls, median of REPEATS windows; achieved bandwidth = algorithmic bytes (ns_weight_algorithmic_bytes) / time.

Whole step: Llama-2-7B shapes, 32 layers, vocab 32000, Q8_0 and Q4_0 engines alternating, generate() of NEW tokens after a
16-token prompt, host clock around calls that end in a device synchronise; tok/s and bytes per token / time.

  python profiles/q8_0_time.py [--iters N] [--new NEW] [--seconds S]
"""
import argparse
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import neural_speed_b200 as ns  # noqa: E402

NODES = [("q/k/v/o", 4096, 4096), ("gate/up", 11008, 4096), ("down", 4096, 11008), ("lm_head", 32000, 4096)]
N_VOCAB, N_EMBD, N_HEAD, N_LAYER, N_FF, N_CTX = 32000, 4096, 32, 32, 11008, 512


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


L2_SPAN = 160 << 20  # bytes of distinct weights each format cycles through (H100: 50 MB of L2)


def weights(n, k, seed):
    fmts = {"q8_0 ring": ns.W_Q8_0, "s8 register": ns.W_S8, "q4_0 ring": ns.W_S4}
    out = {}
    for i, (key, wf) in enumerate(fmts.items()):
        first = ns.Weight.random(n, k, 32, wf, ns.S_F16, ns.COMP_Q8_0, seed=seed + 100 * i)
        copies = max(2, -(-L2_SPAN // first.algorithmic_bytes))
        out[key] = [first] + [ns.Weight.random(n, k, 32, wf, ns.S_F16, ns.COMP_Q8_0, seed=seed + 100 * i + j) for j in range(1, copies)]
    return out


def time_nodes(iters, repeats):
    print(f"{'node':>9} {'N x K':>13} " + " ".join(f"{k:>24}" for k in ("q8_0 ring", "s8 register", "q4_0 ring")))
    ws_bytes = int(ns.lib().ns_device_workspace_bytes(4, 11008))
    wsb = torch.zeros(ws_bytes // 4 + 64, device="cuda")
    stream = torch.cuda.Stream()  # the calls and the events on one explicit stream (a NULL queue is the library's own stream)
    q = stream.cuda_stream
    for name, n, k in NODES:
        ws = weights(n, k, 7)
        x = torch.randn(1, k, device="cuda")
        out = torch.empty(1, n, device="cuda")
        times = {key: [] for key in ws}
        for key, wl in ws.items():  # warm-up: module load, attribute set-up
            for w in wl:
                ns.mul_mat(w, x.data_ptr(), k, out.data_ptr(), n, 1, ws_ptr=wsb.data_ptr(), queue=q)
        torch.cuda.synchronize()
        for _ in range(repeats):
            for key, wl in ws.items():  # alternating
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for i in range(iters):
                    ns.mul_mat(wl[i % len(wl)], x.data_ptr(), k, out.data_ptr(), n, 1, ws_ptr=wsb.data_ptr(), queue=q)
                e1.record(stream)
                e1.synchronize()
                times[key].append(e0.elapsed_time(e1) * 1e-3 / iters)
        cells = []
        for key, wl in ws.items():
            t = float(np.median(times[key]))
            cells.append(f"{t * 1e6:8.2f} us {wl[0].algorithmic_bytes / t / 1e12:5.2f} TB/s")
        print(f"{name:>9} {f'{n}x{k}':>13} " + " ".join(f"{c:>24}" for c in cells))
        for wl in ws.values():
            for w in wl:
                w.free()


def engine(fmt, seed):
    E, FF = N_EMBD, N_FF
    rng = np.random.default_rng(seed)
    eng = ns.Llama(N_VOCAB, E, N_HEAD, N_HEAD, N_LAYER, FF, N_CTX, 1e-5)
    wf, sf = (ns.W_Q8_0, ns.S_F16) if fmt == "q8_0" else (ns.W_S4, ns.S_F16)
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    keep = []
    nbytes = 0
    for il in range(N_LAYER):
        eng.set_f32(ns.Llama.ATTN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        eng.set_f32(ns.Llama.FFN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        for t, (n, k) in shapes.items():
            w = ns.Weight.random(n, k, 32, wf, sf, ns.COMP_Q8_0, seed=il * 8 + t)
            eng.set_weight(t, il, w)
            keep.append(w)
            nbytes += w.algorithmic_bytes
    out = ns.Weight.random(N_VOCAB, E, 32, wf, sf, ns.COMP_Q8_0, seed=999)
    keep.append(out)
    nbytes += out.algorithmic_bytes
    eng.set_weight(ns.Llama.OUTPUT, 0, out)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32))
    eng.set_f32(ns.Llama.OUT_NORM, 0, rng.uniform(0.5, 1.5, E).astype(np.float32))
    return eng, keep, nbytes


def time_steps(new, seconds):
    engs = {fmt: engine(fmt, 3) for fmt in ("q8_0", "q4_0")}
    prompt = list(range(1, 17))
    for fmt, (eng, _, _) in engs.items():
        eng.eval(prompt, 0, want_logits=False)
        eng.generate(5, 16, 4)
    ts = {fmt: [] for fmt in engs}
    t_end = time.perf_counter() + seconds
    while time.perf_counter() < t_end or len(ts["q8_0"]) < 3:
        for fmt, (eng, _, _) in engs.items():
            t0 = time.perf_counter()
            eng.generate(5, 16, new)
            ts[fmt].append(time.perf_counter() - t0)
    print(f"decode step, 7B shapes, {N_LAYER} layers, vocab {N_VOCAB}, generate({new}) from position 16, {len(ts['q8_0'])} calls each:")
    for fmt, (eng, _, nbytes) in engs.items():
        t = float(np.median(ts[fmt])) / new
        print(f"  {fmt}: {1 / t:8.1f} tok/s  {t * 1e3:.3f} ms/token  weights {nbytes:,} B/token  {nbytes / t / 1e12:.2f} TB/s")
    for eng, _, _ in engs.values():
        eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--repeats", type=int, default=9)
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=6.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    ns.lib().bestla_init()
    print(f"card: {card()}")
    time_nodes(args.iters, args.repeats)
    time_steps(args.new, args.seconds)


if __name__ == "__main__":
    main()

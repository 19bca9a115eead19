"""Decode speed of a Qwen2 context against a Llama context of the same shapes and weights.

Qwen2-7B shapes: n_embd 3584, 28 heads over 4 KV heads of 128, n_ff 18944, vocab 151936, all 28 layers, Q4_0-type weights
(int4 codes, group 32, fp16 scales, the ring GEMV's Q8_0 activations), random codes generated on the device (the decode path is
bandwidth bound).  Both contexts borrow the same weight handles; the Qwen2 one runs its own P-order copies of W_q / W_k and adds
the q / k / v biases in the matmul epilogues.  The two alternate in one process: generate() of NEW tokens after a 16-token prompt,
host clock around calls that end in a device synchronise; ms/token, median over the calls.

  python profiles/qwen2_time.py [--new NEW] [--seconds S]
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

N_VOCAB, N_EMBD, N_HEAD, N_HEAD_KV, N_LAYER, N_FF, N_CTX = 151936, 3584, 28, 4, 28, 18944, 512


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


def tensors(seed):
    E, FF, kvd = N_EMBD, N_FF, N_EMBD // N_HEAD * N_HEAD_KV
    rng = np.random.default_rng(seed)
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (kvd, E), ns.Llama.WV: (kvd, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    layers = []
    for il in range(N_LAYER):
        L = {"attn_norm": rng.uniform(0.5, 1.5, E).astype(np.float32), "ffn_norm": rng.uniform(0.5, 1.5, E).astype(np.float32),
             "bias": [rng.normal(0, 0.5, n).astype(np.float32) for n in (E, kvd, kvd)]}
        L["w"] = {t: ns.Weight.random(n, k, 32, ns.W_S4, ns.S_F16, ns.COMP_Q8_0, seed=il * 8 + t) for t, (n, k) in shapes.items()}
        layers.append(L)
    out = ns.Weight.random(N_VOCAB, E, 32, ns.W_S4, ns.S_F16, ns.COMP_Q8_0, seed=999)
    tok = (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32)
    return layers, out, tok, rng.uniform(0.5, 1.5, E).astype(np.float32)


def engine(arch, t):
    layers, out, tok, out_norm = t
    eng = ns.Llama(N_VOCAB, N_EMBD, N_HEAD, N_HEAD_KV, N_LAYER, N_FF, N_CTX, 1e-6, 1000000.0, arch=arch)
    for il, L in enumerate(layers):
        eng.set_f32(ns.Llama.ATTN_NORM, il, L["attn_norm"])
        eng.set_f32(ns.Llama.FFN_NORM, il, L["ffn_norm"])
        for tid, w in L["w"].items():
            eng.set_weight(tid, il, w)
        if arch == "qwen2":
            for tid, b in zip((ns.Llama.BQ, ns.Llama.BK, ns.Llama.BV), L["bias"]):
                eng.set_f32(tid, il, b)
    eng.set_weight(ns.Llama.OUTPUT, 0, out)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, tok)
    eng.set_f32(ns.Llama.OUT_NORM, 0, out_norm)
    return eng


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=10.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    ns.lib().bestla_init()
    print(f"card: {card()}")
    t = tensors(3)
    engs = {arch: engine(arch, t) for arch in ("llama", "qwen2")}
    prompt = list(range(1, 17))
    for eng in engs.values():
        eng.eval(prompt, 0, want_logits=False)
        eng.generate(5, 16, 4)
    L = ns.lib()
    launches = {}
    for arch, eng in engs.items():  # kernels of one decode pass: the first step of a fresh graph enqueues it twice
        before = L.ns_launch_count()
        eng.set_streaming(-1)  # drops the decode graph
        eng.eval([5], 16, want_logits=False)
        launches[arch] = (L.ns_launch_count() - before) // 2
    ts = {arch: [] for arch in engs}
    t_end = time.perf_counter() + args.seconds
    while time.perf_counter() < t_end or len(ts["qwen2"]) < 3:
        for arch, eng in engs.items():
            t0 = time.perf_counter()
            eng.generate(5, 16, args.new)
            ts[arch].append(time.perf_counter() - t0)
    print(f"decode step, Qwen2-7B shapes, {N_LAYER} layers, vocab {N_VOCAB}, generate({args.new}) from position 16, "
          f"{len(ts['qwen2'])} calls each (alternating):")
    for arch in engs:
        v = np.array(ts[arch]) / args.new * 1e3
        print(f"  {arch:>6}: {np.median(v):.3f} ms/token (min {v.min():.3f}, max {v.max():.3f})  kernels per step {launches[arch]}")
    for eng in engs.values():
        eng.close()


if __name__ == "__main__":
    main()

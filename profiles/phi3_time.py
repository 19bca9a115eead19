"""Decode speed of a Phi-3 context at Phi-3-mini's shapes, and the head size 96 attention kernels on their own.

Phi-3-mini shapes: n_embd 3072, 32 heads of 96 (MHA), n_ff 8192, vocab 32064, all 32 layers, Q4_0-type weights (int4 codes, group
32, fp16 scales, the ring GEMV's Q8_0 activations), random codes generated on the device (the decode path is bandwidth bound).
Measured in one process, host clock around calls that end in a device synchronise, medians over the calls:
  * generate(NEW) from position 16 and from 2048 cached positions (ms/token);
  * generate_batch at n = 8 and 32 sequences (ms per step of n tokens);
  * one layer's attention alone at n_ctx 4096, one new token at position 4095: NS_ATTN_SPLIT_DECODE against NS_ATTN_GENERIC
    through ns_llama_attention, rounds of 200 calls alternating between the two (q is rotated in place by the generic path's
    rope_kv_kernel each call; the time does not depend on its values), and the kernel time per call from torch.profiler.

  python profiles/phi3_time.py [--new NEW] [--seconds S]
"""
import argparse
import os
import re
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import neural_speed_b200 as ns  # noqa: E402

N_VOCAB, N_EMBD, N_HEAD, N_HEAD_KV, N_LAYER, N_FF, N_CTX = 32064, 3072, 32, 32, 32, 8192, 4096
HD = N_EMBD // N_HEAD


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


def engine():
    E, FF = N_EMBD, N_FF
    rng = np.random.default_rng(3)
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    eng = ns.Llama(N_VOCAB, N_EMBD, N_HEAD, N_HEAD_KV, N_LAYER, N_FF, N_CTX, 1e-5, 10000.0, arch="phi3")
    for il in range(N_LAYER):
        eng.set_f32(ns.Llama.ATTN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        eng.set_f32(ns.Llama.FFN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        for t, (n, k) in shapes.items():
            eng.set_weight(t, il, ns.Weight.random(n, k, 32, ns.W_S4, ns.S_F16, ns.COMP_Q8_0, seed=il * 8 + t))
    eng.set_weight(ns.Llama.OUTPUT, 0, ns.Weight.random(N_VOCAB, E, 32, ns.W_S4, ns.S_F16, ns.COMP_Q8_0, seed=999))
    eng.set_f32(ns.Llama.TOK_EMBD, 0, (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32))
    eng.set_f32(ns.Llama.OUT_NORM, 0, rng.uniform(0.5, 1.5, E).astype(np.float32))
    return eng


def timed(fn, seconds, min_calls=3):
    ts, t_end = [], time.perf_counter() + seconds
    while time.perf_counter() < t_end or len(ts) < min_calls:
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return np.array(ts)


def attention_alone(seconds):
    """one layer's attention at n_ctx 4096, position 4095: split decode against the generic kernel (us per call)"""
    L = ns.lib()
    r = np.random.default_rng(1)
    q = torch.from_numpy(r.normal(0, 1, (1, N_HEAD * HD)).astype(np.float32)).cuda()
    k = torch.from_numpy(r.normal(0, 1, (1, N_HEAD_KV * HD)).astype(np.float32)).cuda()
    v = torch.from_numpy(r.normal(0, 1, (1, N_HEAD_KV * HD)).astype(np.float32)).cuda()
    kc = torch.randn((N_HEAD_KV, N_CTX, HD), device="cuda").half()
    vc = torch.randn_like(kc)
    out = torch.zeros((1, N_HEAD * HD), device="cuda")
    ws = torch.zeros(L.ns_llama_attention_workspace_bytes(N_HEAD, HD, N_CTX), dtype=torch.uint8, device="cuda")
    kinds = {"split decode": ns.ATTN_SPLIT_DECODE, "generic": ns.ATTN_GENERIC}
    res = {name: [] for name in kinds}

    def calls(kind, n):
        """n calls back to back, host clock around them and a device synchronise (us per call, launch and state upload included)"""
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(n):
            rc = L.ns_llama_attention(kind, q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), N_HEAD, N_HEAD_KV,
                                      HD, N_CTX, N_CTX - 1, 1, 10000.0, 1.0, out.data_ptr(), ws.data_ptr(), None)
            assert rc == 0, ns.last_error()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / n * 1e6

    for kind in kinds.values():  # warm-up: module load, shared-memory grants
        calls(kind, 20)
    t_end = time.perf_counter() + seconds
    while time.perf_counter() < t_end or len(res["generic"]) < 5:
        for name, kind in kinds.items():
            res[name].append(calls(kind, 200))
    print(f"one layer's attention, {N_HEAD} heads of {HD}, n_ctx {N_CTX}, one token at position {N_CTX - 1} "
          f"({len(res['generic'])} rounds of 200 calls each, alternating):")
    for name, t in res.items():
        t = np.array(t)
        print(f"  {name:>12}: {np.median(t):.1f} us per call (min {t.min():.1f}, max {t.max():.1f})")
    # kernel time alone: torch.profiler over 50 calls of each, in a pass of its own after the timed rounds (the entry's per-call
    # host work -- state upload, shared-memory grant -- is not in it)
    from torch.profiler import ProfilerActivity, profile
    for name, kind in kinds.items():
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            calls(kind, 50)
        us = sum(e.device_time_total for e in prof.key_averages() if "attn" in e.key or "rope_kv" in e.key) / 50
        kern = sorted({m for e in prof.key_averages() for m in re.findall(r"\w+_kernel", e.key) if "attn" in m or "rope_kv" in m})
        print(f"  {name:>12}: {us:.1f} us of kernel time per call ({', '.join(kern)})")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=64)
    ap.add_argument("--seconds", type=float, default=6.0)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    ns.lib().bestla_init()
    print(f"card: {card()}")
    eng = engine()
    eng.eval(list(range(1, 17)), 0, want_logits=False)
    eng.eval([7] * 2048, 0, want_logits=False)  # 2048 cached positions (the first 16 are rewritten below, as before)
    eng.eval(list(range(1, 17)), 0, want_logits=False)
    for start in (16, 2048):
        eng.generate(5, start, 4)
        v = timed(lambda: eng.generate(5, start, args.new), args.seconds) / args.new * 1e3
        print(f"Phi-3-mini shapes, {N_LAYER} layers, int4: generate({args.new}) from position {start}: {np.median(v):.3f} ms/token "
              f"(min {v.min():.3f}, max {v.max():.3f}, {v.size} calls)")
    for n in (8, 32):
        eng.set_sequences(n)
        seqs = list(range(n))
        eng.generate_batch(seqs, [5] * n, [16] * n, 2)
        steps = 16
        v = timed(lambda: eng.generate_batch(seqs, [5] * n, [16] * n, steps), args.seconds) / steps * 1e3
        print(f"Phi-3-mini shapes, {N_LAYER} layers, int4: generate_batch n = {n}: {np.median(v):.3f} ms per step of {n} tokens "
              f"({n / np.median(v) * 1e3:.0f} tok/s; min {v.min():.3f}, max {v.max():.3f}, {v.size} calls)")
    eng.close()
    attention_alone(args.seconds)


if __name__ == "__main__":
    main()

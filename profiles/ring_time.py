"""Cost of a streaming ring step (ns_llama_set_streaming) against a plain decode step at the same length.

Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000; BesTLA int4 weights generated on
the device), n_ctx 2048, n_keep 4.  Two contexts share the weights: a plain one, whose steps run at 2047 cached positions (the
last slot), and a streaming one past its wrap, whose steps attend all 2048 slots and shift 2044 cached keys per layer.  Both go
through ns_llama_generate, one token per call, timed with a host clock around the call (which ends in a device synchronise),
alternated in one process.  Prints the card and its power limit, the byte model per token and the two step times.

  python profiles/ring_time.py [--steps N] [--warmup W]
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

N_VOCAB, N_EMBD, N_HEAD, N_LAYER, N_FF, N_CTX, N_KEEP = 32000, 4096, 32, 32, 11008, 2048, 4


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name from torch alone, the limit unknown
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    L = ns.lib()
    L.bestla_init()
    rng = np.random.default_rng(0)
    hp = dict(n_vocab=N_VOCAB, n_embd=N_EMBD, n_head=N_HEAD, n_head_kv=N_HEAD, n_layer=N_LAYER, n_ff=N_FF, n_ctx=N_CTX, norm_eps=1e-5)
    E, FF = N_EMBD, N_FF
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    weights = {(il, t): ns.Weight.random(n, k, seed=il * 8 + t) for il in range(N_LAYER) for t, (n, k) in shapes.items()}
    out_w = ns.Weight.random(N_VOCAB, E, seed=999)
    tok = (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32)
    norms = [rng.uniform(0.5, 1.5, E).astype(np.float32) for _ in range(2 * N_LAYER + 1)]
    weight_bytes = sum(w.algorithmic_bytes for w in weights.values()) + out_w.algorithmic_bytes

    def make(n_keep):
        eng = ns.Llama(**hp)
        eng.set_f32(ns.Llama.TOK_EMBD, 0, tok)
        eng.set_f32(ns.Llama.OUT_NORM, 0, norms[-1])
        eng.set_weight(ns.Llama.OUTPUT, 0, out_w)
        for il in range(N_LAYER):
            eng.set_f32(ns.Llama.ATTN_NORM, il, norms[2 * il])
            eng.set_f32(ns.Llama.FFN_NORM, il, norms[2 * il + 1])
            for t in shapes:
                eng.set_weight(t, il, weights[(il, t)])
        if n_keep is not None:
            eng.set_streaming(n_keep)
        return eng

    prompt = [int(t) for t in rng.integers(3, N_VOCAB, N_CTX - 1)]
    plain, ring = make(None), make(N_KEEP)
    plain.eval(prompt, 0, want_logits=False)
    ring.eval(prompt, 0, want_logits=False)
    n_total = N_CTX - 1
    ring.generate(5, n_total, 1)  # fills the last slot
    n_total += 1
    tp, tr = [], []
    for i in range(args.warmup + args.steps):
        t0 = time.perf_counter()
        plain.generate(7, N_CTX - 1, 1)
        t1 = time.perf_counter()
        ring.generate(7, n_total, 1)
        t2 = time.perf_counter()
        n_total += 1
        if i >= args.warmup:
            tp.append(t1 - t0)
            tr.append(t2 - t1)
    hd = E // N_HEAD
    kv_read = 2 * N_LAYER * N_HEAD * N_CTX * hd * 2
    k_write = N_LAYER * N_HEAD * (N_CTX - N_KEEP) * hd * 2
    mp, mr = float(np.median(tp)) * 1e3, float(np.median(tr)) * 1e3
    print(f"card: {card()}")
    print(f"7B shapes, {N_LAYER} layers, int4 weights, n_ctx {N_CTX}, n_keep {N_KEEP}, {args.steps} steps after {args.warmup} warm-up, "
          f"ring steps at n_total {N_CTX + args.warmup}..{n_total - 1}")
    print(f"bytes per token: weights {weight_bytes / 1e9:.2f} GB + K/V read {kv_read / 1e9:.2f} GB; the ring adds the K write-back "
          f"{k_write / 1e9:.2f} GB ({k_write / (weight_bytes + kv_read):.1%} more)")
    print(f"plain step (2047 cached): median {mp:.3f} ms (p10 {np.percentile(tp, 10) * 1e3:.3f}, p90 {np.percentile(tp, 90) * 1e3:.3f})")
    print(f"ring step  (2048 slots):  median {mr:.3f} ms (p10 {np.percentile(tr, 10) * 1e3:.3f}, p90 {np.percentile(tr, 90) * 1e3:.3f})")
    print(f"ring / plain: {mr / mp:.3f}")
    plain.close()
    ring.close()


if __name__ == "__main__":
    main()

"""Admitting prompts into a running batch: one mixed pass (ns_llama_eval_batch) against the decode step plus one prompt call each.

Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000; BesTLA int4 weights, group 128, int8
compute, generated on the device), n_ctx 1024.  16 sequences decode at 512 cached positions; k in {1, 4, 8} new prompts of P in
{16, 128} tokens arrive on free blocks.  For each (k, P):
  (a) one eval_batch carrying the 16 decode tokens and the k prompts (T = 16 + k P rows);
  (b) decode_batch of the 16 sequences, then k eval_seq calls of P tokens.
Every call restarts at the same positions (it rewrites the same K/V rows), so all repetitions do the same work.  (a) and (b) are
alternated in one process, after a warm-up of every shape, and timed with a host clock around each call (every call ends in a
device synchronise); the medians over at least --seconds per point are printed with the card's name and power limit.

  python profiles/mixed_time.py [--seconds S]
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

N_VOCAB, N_EMBD, N_HEAD, N_LAYER, N_FF, N_CTX, N_DEC, N_PAST = 32000, 4096, 32, 32, 11008, 1024, 16, 512
KS, PS = (1, 4, 8), (16, 128)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name from torch alone, the limit unknown
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=1.5, help="timed window per point (both variants together)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    L = ns.lib()
    L.bestla_init()
    rng = np.random.default_rng(0)
    hp = dict(n_vocab=N_VOCAB, n_embd=N_EMBD, n_head=N_HEAD, n_head_kv=N_HEAD, n_layer=N_LAYER, n_ff=N_FF, n_ctx=N_CTX, norm_eps=1e-5)
    E, FF = N_EMBD, N_FF
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    weights = {(il, t): ns.Weight.random(n, k, group=128, seed=il * 8 + t) for il in range(N_LAYER) for t, (n, k) in shapes.items()}
    out_w = ns.Weight.random(N_VOCAB, E, group=128, seed=999)
    tok = (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32)
    weight_bytes = sum(w.algorithmic_bytes for w in weights.values()) + out_w.algorithmic_bytes
    eng = ns.Llama(**hp)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, tok)
    eng.set_f32(ns.Llama.OUT_NORM, 0, rng.uniform(0.5, 1.5, E).astype(np.float32))
    eng.set_weight(ns.Llama.OUTPUT, 0, out_w)
    for il in range(N_LAYER):
        eng.set_f32(ns.Llama.ATTN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        eng.set_f32(ns.Llama.FFN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        for t in shapes:
            eng.set_weight(t, il, weights[(il, t)])
    eng.set_sequences(N_DEC + max(KS))
    for s in range(N_DEC):
        eng.eval_seq(s, [int(t) for t in rng.integers(3, N_VOCAB, N_PAST)], 0, want_logits=False)
    dec_seqs = np.arange(N_DEC, dtype=np.int32)
    dec_toks = rng.integers(3, N_VOCAB, N_DEC).astype(np.int32)
    dec_past = np.full(N_DEC, N_PAST, np.int32)
    prompts = [[int(t) for t in rng.integers(3, N_VOCAB, max(PS))] for _ in range(max(KS))]

    print(f"card: {card()}")
    print(f"7B shapes, {N_LAYER} layers, int4 g128 weights (int8 compute), n_ctx {N_CTX}; {N_DEC} sequences decode at {N_PAST} cached "
          f"positions; weights {weight_bytes / 1e9:.2f} GB per pass; >= {args.seconds} s per point")
    print(f"{'k':>2} {'P':>4} {'T':>5} {'(a) ms':>8} {'(b) ms':>8} {'(b)/(a)':>7} {'passes (b)':>10} calls")
    for P in PS:
        for k in KS:
            seqs = np.concatenate([dec_seqs, np.arange(N_DEC, N_DEC + k, dtype=np.int32)])
            segs = [[int(t)] for t in dec_toks] + [prompts[j][:P] for j in range(k)]
            past = np.concatenate([dec_past, np.zeros(k, np.int32)])

            def mixed():
                eng.eval_batch(seqs, segs, past, want_logits=False)

            def separate():
                eng.decode_batch(dec_seqs, dec_toks, dec_past, want_logits=False)
                for j in range(k):
                    eng.eval_seq(N_DEC + j, prompts[j][:P], 0, want_logits=False)

            for _ in range(2):  # warm-up: buffers, graphs, routing of every shape
                mixed()
                separate()
            ta, tb = [], []
            t_end = time.perf_counter() + args.seconds
            while time.perf_counter() < t_end or len(ta) < 5:
                t0 = time.perf_counter()
                mixed()
                t1 = time.perf_counter()
                separate()
                ta.append(t1 - t0)
                tb.append(time.perf_counter() - t1)
            a, b = float(np.median(ta)), float(np.median(tb))
            print(f"{k:>2} {P:>4} {N_DEC + k * P:>5} {a * 1e3:>8.2f} {b * 1e3:>8.2f} {b / a:>7.2f} {k + 1:>10} {len(ta)}")
    eng.close()


if __name__ == "__main__":
    main()

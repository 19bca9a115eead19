"""Decode speed of the Q8_0 KV cache (ns_llama_set_kv_type) against the fp16 cache.

Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000; BesTLA int4 weights, group 128, int8
compute, generated on the device), n_ctx 2112, 32 KV blocks.  Two engines share the weights, one per cache format, each with the
same prompts: 512 tokens in blocks 1 .. 31 and 2048 in block 0.  Points, each alternating the two engines call by call in this
process, median of a host clock around calls that end in a device synchronise:
  generate_batch at n = 1 / 4 / 8 / 16 / 32 sequences from position 512 (NEW tokens per sequence and call)
  generate on block 0 from position 2048 (NEW tokens)
Prints the card and its power limit, ms per step for both formats, the ratio, and the byte model of a step (weights once + the K/V
bytes every sequence reads).  Also the logit distance, max |a - b| / max(1, max|b|), of the Q8_0 engine to the fp16 engine over a
12-token prompt and 16 greedy steps (the fp16 engine's picks fed to both), measured, not a bar.

  python profiles/kv_q8_time.py [--new NEW] [--seconds S]
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

N_VOCAB, N_EMBD, N_HEAD, N_LAYER, N_FF, N_CTX, N_SEQ, N_PAST, N_LONG = 32000, 4096, 32, 32, 11008, 2112, 32, 512, 2048


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:
        return f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"


def alternated(fa, fb, seconds):
    """median seconds per call of fa and fb, called in turn for at least `seconds` after one warm-up call each"""
    fa(), fb()
    ta, tb = [], []
    t_end = time.perf_counter() + seconds
    while time.perf_counter() < t_end or len(ta) < 3:
        t0 = time.perf_counter()
        fa()
        t1 = time.perf_counter()
        fb()
        ta.append(t1 - t0)
        tb.append(time.perf_counter() - t1)
    return float(np.median(ta)), float(np.median(tb)), len(ta)


def distance(a, b):
    return float(np.abs(a - b).max()) / max(1.0, float(np.abs(b).max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=32, help="tokens generated per sequence and call")
    ap.add_argument("--seconds", type=float, default=3.0, help="timed window per point (both formats)")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    ns.lib().bestla_init()
    rng = np.random.default_rng(0)
    E, FF, hd = N_EMBD, N_FF, N_EMBD // N_HEAD
    hp = dict(n_vocab=N_VOCAB, n_embd=E, n_head=N_HEAD, n_head_kv=N_HEAD, n_layer=N_LAYER, n_ff=FF, n_ctx=N_CTX, norm_eps=1e-5)
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    weights = {(il, t): ns.Weight.random(n, k, group=128, seed=il * 8 + t) for il in range(N_LAYER) for t, (n, k) in shapes.items()}
    out_w = ns.Weight.random(N_VOCAB, E, group=128, seed=999)
    tok = (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32)
    out_norm = rng.uniform(0.5, 1.5, E).astype(np.float32)
    norms = [(rng.uniform(0.5, 1.5, E).astype(np.float32), rng.uniform(0.5, 1.5, E).astype(np.float32)) for _ in range(N_LAYER)]
    weight_bytes = sum(w.algorithmic_bytes for w in weights.values()) + out_w.algorithmic_bytes
    prompts = [[int(t) for t in rng.integers(3, N_VOCAB, N_LONG if s == 0 else N_PAST)] for s in range(N_SEQ)]
    engines = {}
    for kind in ("f16", "q8_0"):
        eng = ns.Llama(**hp)
        eng.set_f32(ns.Llama.TOK_EMBD, 0, tok)
        eng.set_f32(ns.Llama.OUT_NORM, 0, out_norm)
        eng.set_weight(ns.Llama.OUTPUT, 0, out_w)
        for il in range(N_LAYER):
            eng.set_f32(ns.Llama.ATTN_NORM, il, norms[il][0])
            eng.set_f32(ns.Llama.FFN_NORM, il, norms[il][1])
            for t in shapes:
                eng.set_weight(t, il, weights[(il, t)])
        eng.set_sequences(N_SEQ)
        eng.set_kv_type(kind)
        engines[kind] = eng
    f16, q8 = engines["f16"], engines["q8_0"]
    print(f"card: {card()}")
    print(f"7B shapes, {N_LAYER} layers, int4 g128 weights (int8 compute), n_ctx {N_CTX}, {N_SEQ} KV blocks: fp16 "
          f"{f16.kv_bytes() / 1e9:.1f} GB, Q8_0 {q8.kv_bytes() / 1e9:.1f} GB")
    # logit distance of the Q8_0 engine to the fp16 engine, on a sequence of its own (block N_SEQ - 1, restarted afterwards)
    p = [1] + [int(t) for t in rng.integers(3, N_VOCAB, 11)]
    a, _ = q8.eval_seq(N_SEQ - 1, p, 0)
    b, pick = f16.eval_seq(N_SEQ - 1, p, 0)
    dist = distance(a, b)
    for i in range(16):
        a, _ = q8.eval_seq(N_SEQ - 1, [pick], 12 + i)
        b, pick = f16.eval_seq(N_SEQ - 1, [pick], 12 + i)
        dist = max(dist, distance(a, b))
    print(f"logit distance Q8_0 vs fp16 engine, 12-token prompt + 16 greedy steps: {dist:.3e} (max |d| / max(1, max|fp16|))")
    for eng in (f16, q8):
        for s in range(N_SEQ):
            eng.eval_seq(s, prompts[s], 0, want_logits=False)
    print(f"{'point':>24} {'fp16 ms/step':>13} {'Q8_0 ms/step':>13} {'speed-up':>9} {'model':>6} calls")
    firsts = rng.integers(3, N_VOCAB, N_SEQ).astype(np.int32)

    def row(label, past, n, ta, tb, calls):
        kv16 = 2 * N_LAYER * N_HEAD * (past + (args.new + 1) / 2) * hd * 2  # K and V one sequence reads per step, fp16
        model = (weight_bytes + n * kv16) / (weight_bytes + n * kv16 * 136 / 256)
        print(f"{label:>24} {ta / args.new * 1e3:>13.3f} {tb / args.new * 1e3:>13.3f} {ta / tb:>9.3f} {model:>6.2f} {calls}")

    for n in (1, 4, 8, 16, 32):
        seqs = np.arange(n, dtype=np.int32)
        past = np.full(n, N_PAST, np.int32)
        ta, tb, calls = alternated(lambda: f16.generate_batch(seqs, firsts[:n], past, args.new),
                                   lambda: q8.generate_batch(seqs, firsts[:n], past, args.new), args.seconds)
        row(f"generate_batch n={n} @{N_PAST}", N_PAST, n, ta, tb, calls)
    ta, tb, calls = alternated(lambda: f16.generate(int(firsts[0]), N_LONG, args.new), lambda: q8.generate(int(firsts[0]), N_LONG, args.new),
                               args.seconds)
    row(f"generate @{N_LONG}", N_LONG, 1, ta, tb, calls)
    print("model: the byte model's speed-up (weights once + K/V rows, Q8_0 at 136 / 256 of fp16's bytes)")
    for eng in (f16, q8):
        eng.close()


if __name__ == "__main__":
    main()

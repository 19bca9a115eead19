"""Cost of per-sequence sampling in the eval step: 7B-shaped batched generation in four pick modes, and the host cost of a config
change.

Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000; BesTLA int4 g128 weights, int8
compute, generated on the device), n_ctx 1024, 32 KV blocks, every sequence at 512 cached positions.

1. ns_llama_generate_batch step time for n = 1, 8 and 32 rows, N_NEW tokens per call, in four modes alternated call by call in
   one process: greedy; context-wide sampling (ns_llama_set_sampling, top_k 40 and the reference's other defaults); per-sequence
   sampling with the same parameters on every block and distinct seeds; per-sequence sampling on a mix of greedy, top_k 40 and
   top_k 1024 / top_p 1 blocks.  Each timed call follows an untimed call in the same mode, so no graph capture is timed.  Host
   clock around each call (which ends in a device synchronise), medians.
2. A config change between two steps of a running batch (n = 32, one token per call): ns_llama_set_sequence_sampling on one
   block, against ns_llama_set_sampling, which drops the captured graphs so that the next step pays an eager pass and a capture.
   Host clock around the config call and around the step after it, medians.
Prints the card and its power limit first.

  python profiles/sample_seq_time.py [--new N_NEW] [--seconds S]
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

N_VOCAB, N_EMBD, N_HEAD, N_LAYER, N_FF, N_CTX, N_SEQ, N_PAST = 32000, 4096, 32, 32, 11008, 1024, 32, 512
A = dict(top_k=40, top_p=0.95, temperature=0.8, repeat_penalty=1.1, repeat_last_n=64)


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name from torch alone, the limit unknown
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def engine():
    rng = np.random.default_rng(0)
    hp = dict(n_vocab=N_VOCAB, n_embd=N_EMBD, n_head=N_HEAD, n_head_kv=N_HEAD, n_layer=N_LAYER, n_ff=N_FF, n_ctx=N_CTX, norm_eps=1e-5)
    E, FF = N_EMBD, N_FF
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    eng = ns.Llama(**hp)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32))
    eng.set_f32(ns.Llama.OUT_NORM, 0, rng.uniform(0.5, 1.5, E).astype(np.float32))
    eng.set_weight(ns.Llama.OUTPUT, 0, ns.Weight.random(N_VOCAB, E, group=128, seed=999))
    for il in range(N_LAYER):
        eng.set_f32(ns.Llama.ATTN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        eng.set_f32(ns.Llama.FFN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        for t, (n, k) in shapes.items():
            eng.set_weight(t, il, ns.Weight.random(n, k, group=128, seed=il * 8 + t))
    eng.set_sequences(N_SEQ)
    for sq in range(N_SEQ):
        eng.eval_seq(sq, [int(t) for t in rng.integers(3, N_VOCAB, N_PAST)], 0, want_logits=False)
    return eng, rng.integers(3, N_VOCAB, N_SEQ).astype(np.int32)


def mix(b):
    """block b of the mixed batch: greedy, top_k 40, or top_k 1024 with top_p 1"""
    return [dict(top_k=None), dict(A, seed=b), dict(A, top_k=1024, top_p=1.0, seed=b)][b % 3]


def modes(eng):
    def per_seq(cfg):
        def set_all():
            for b in range(N_SEQ):
                eng.set_sequence_sampling(b, **cfg(b))
        return set_all

    return {
        "greedy": lambda: eng.set_sampling(None),
        "context top_k 40": lambda: eng.set_sampling(seed=1, **A),
        "per-seq top_k 40": per_seq(lambda b: dict(A, seed=b)),
        "per-seq mixed": per_seq(mix),
    }


def step_times(eng, firsts, args):
    print(f"\n1. generate_batch, {args.new} new tokens per sequence and call, ms per step (median), modes alternated")
    ms = modes(eng)
    print(f"{'n':>3} " + " ".join(f"{m:>17}" for m in ms) + "   calls")
    for n in (1, 8, 32):
        seqs, past, first = np.arange(n, dtype=np.int32), np.full(n, N_PAST, np.int32), firsts[:n]
        t = {m: [] for m in ms}
        t_end = time.perf_counter() + len(ms) * args.seconds
        while time.perf_counter() < t_end or len(t["greedy"]) < 3:
            for m, enter in ms.items():
                enter()
                eng.generate_batch(seqs, first, past, args.new)  # a switch between modes may recapture: untimed
                t0 = time.perf_counter()
                eng.generate_batch(seqs, first, past, args.new)
                t[m].append(time.perf_counter() - t0)
        med = {m: float(np.median(v)) / args.new * 1e3 for m, v in t.items()}
        print(f"{n:>3} " + " ".join(f"{med[m]:>17.3f}" for m in ms) + f"   {len(t['greedy'])} each")


def change_cost(eng, firsts, args):
    print("\n2. one config change between two steps of n = 32 rows (one token per step), ms (median)")
    seqs, past = np.arange(N_SEQ, dtype=np.int32), np.full(N_SEQ, N_PAST, np.int32)
    kinds = {
        "set_sequence_sampling(block 5)": lambda i: eng.set_sequence_sampling(5, **dict(A, seed=i)),
        "set_sampling (drops the graphs)": lambda i: eng.set_sampling(seed=i, **A),
    }
    t = {k: ([], []) for k in kinds}
    t_end = time.perf_counter() + 2 * args.seconds
    i = 0
    while time.perf_counter() < t_end or len(t[next(iter(kinds))][0]) < 3:
        for k, change in kinds.items():
            change(i)  # enters the call's mode: untimed
            eng.generate_batch(seqs, firsts, past, 1)
            eng.generate_batch(seqs, firsts, past, 1)
            t0 = time.perf_counter()
            change(i + 1)
            t1 = time.perf_counter()
            eng.generate_batch(seqs, firsts, past, 1)
            t2 = time.perf_counter()
            t[k][0].append(t1 - t0)
            t[k][1].append(t2 - t1)
            i += 2
    plain = []
    for _ in range(20):
        t0 = time.perf_counter()
        eng.generate_batch(seqs, firsts, past, 1)
        plain.append(time.perf_counter() - t0)
    print(f"{'':>32} {'config call':>12} {'next step':>10}   calls")
    for k, (c, s) in t.items():
        print(f"{k:>32} {np.median(c) * 1e3:>12.3f} {np.median(s) * 1e3:>10.3f}   {len(c)}")
    print(f"{'a step with no change':>32} {'':>12} {np.median(plain) * 1e3:>10.3f}   {len(plain)}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=32, help="tokens generated per sequence and call")
    ap.add_argument("--seconds", type=float, default=2.0, help="timed window per mode and row count")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    ns.lib().bestla_init()
    print(f"card: {card()}")
    eng, firsts = engine()
    print(f"7B shapes, {N_LAYER} layers, int4 g128 weights (int8 compute), n_ctx {N_CTX}, {N_SEQ} KV blocks, every sequence at "
          f"{N_PAST} cached positions; sampled modes: top_p 0.95, temperature 0.8, repeat_penalty 1.1, last 64")
    step_times(eng, firsts, args)
    change_cost(eng, firsts, args)
    eng.close()


if __name__ == "__main__":
    main()

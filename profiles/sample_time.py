"""Cost of sampling in the eval step: the sampler kernel on its own, and 7B-shaped generation greedy against sampled.

1. ns_llama_sample (one launch: penalty, top-k, top-p, temperature, draw) on random logits, for n = 1, 8, 32 rows, n_vocab 32000
   and 128256, top_k 40 and 1024 (top_p 0.95, temperature 0.8, repeat_penalty 1.1, a 64-token window): CUDA events around 200
   launches on one stream after 20 warm-up launches, microseconds per launch.
2. Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000; BesTLA int4 g128 weights,
   int8 compute, generated on the device), n_ctx 1024, every sequence at 512 cached positions: ns_llama_generate and
   ns_llama_generate_batch (n = 32) producing N_NEW tokens per call, greedy and sampled (the reference's defaults) alternated
   call by call in one process, host clock around each call (which ends in a device synchronise), medians.
Prints the card and its power limit first.

  python profiles/sample_time.py [--new N_NEW] [--seconds S]
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


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name from torch alone, the limit unknown
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def kernel_times():
    rng = np.random.default_rng(0)
    stream = torch.cuda.current_stream()
    print(f"{'n':>3} {'n_vocab':>8} {'top_k':>6} {'us/launch':>10}")
    for nv in (32000, 128256):
        for k in (40, 1024):
            for n in (1, 8, 32):
                lg = torch.from_numpy((rng.standard_normal((n, nv)) * 3).astype(np.float32)).cuda()
                win = torch.from_numpy(rng.integers(0, nv, (n, 64)).astype(np.int32)).cuda()
                mt = torch.from_numpy(ns.sample_seed_host(1).view(np.int32)).cuda()
                picks = torch.zeros(n, dtype=torch.int32, device="cuda")
                ws = torch.zeros(ns.lib().ns_llama_sample_workspace_bytes(n, k), dtype=torch.uint8, device="cuda")
                s = ns.sampling(k, 0.95, 0.8, 1.1, 64, 1)

                def launch():
                    rc = ns.sample(lg.data_ptr(), n, nv, win.data_ptr(), 64, s, mt.data_ptr(), picks.data_ptr(), None, None, None,
                                   ws.data_ptr(), stream.cuda_stream)
                    assert rc == 0, ns.last_error()

                for _ in range(20):
                    launch()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(200):
                    launch()
                e1.record(stream)
                e1.synchronize()
                torch.cuda.synchronize()
                print(f"{n:>3} {nv:>8} {k:>6} {e0.elapsed_time(e1) / 200 * 1e3:>10.1f}")


def generation(args):
    rng = np.random.default_rng(0)
    hp = dict(n_vocab=N_VOCAB, n_embd=N_EMBD, n_head=N_HEAD, n_head_kv=N_HEAD, n_layer=N_LAYER, n_ff=N_FF, n_ctx=N_CTX, norm_eps=1e-5)
    E, FF = N_EMBD, N_FF
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    weights = {(il, t): ns.Weight.random(n, k, group=128, seed=il * 8 + t) for il in range(N_LAYER) for t, (n, k) in shapes.items()}
    out_w = ns.Weight.random(N_VOCAB, E, group=128, seed=999)
    eng = ns.Llama(**hp)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32))
    eng.set_f32(ns.Llama.OUT_NORM, 0, rng.uniform(0.5, 1.5, E).astype(np.float32))
    eng.set_weight(ns.Llama.OUTPUT, 0, out_w)
    for il in range(N_LAYER):
        eng.set_f32(ns.Llama.ATTN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        eng.set_f32(ns.Llama.FFN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        for t in shapes:
            eng.set_weight(t, il, weights[(il, t)])
    eng.set_sequences(N_SEQ)
    for sq in range(N_SEQ):
        eng.eval_seq(sq, [int(t) for t in rng.integers(3, N_VOCAB, N_PAST)], 0, want_logits=False)
    firsts = rng.integers(3, N_VOCAB, N_SEQ).astype(np.int32)
    seqs, past = np.arange(N_SEQ, dtype=np.int32), np.full(N_SEQ, N_PAST, np.int32)
    print(f"7B shapes, {N_LAYER} layers, int4 g128 weights (int8 compute), n_ctx {N_CTX}, every sequence at {N_PAST} cached "
          f"positions, {args.new} new tokens per call; greedy and sampled (top_k 40, top_p 0.95, temperature 0.8, "
          f"repeat_penalty 1.1, last 64) alternated")
    calls = {
        "generate": (lambda: eng.generate(int(firsts[0]), N_PAST, args.new), args.new),
        f"generate_batch n={N_SEQ}": (lambda: eng.generate_batch(seqs, firsts, past, args.new), N_SEQ * args.new),
    }
    for name, (fn, toks) in calls.items():
        t = {"greedy": [], "sampled": []}
        # every switch drops the graphs: warm both modes outside the timed calls, then switch between them (graph re-capture
        # included in neither median: each timed call follows one untimed call in the same mode)
        t_end = time.perf_counter() + 2 * args.seconds
        while time.perf_counter() < t_end or len(t["greedy"]) < 3:
            for mode in ("greedy", "sampled"):
                eng.set_sampling(None) if mode == "greedy" else eng.set_sampling(seed=len(t[mode]))
                fn()
                t0 = time.perf_counter()
                fn()
                t[mode].append(time.perf_counter() - t0)
        g, s = float(np.median(t["greedy"])), float(np.median(t["sampled"]))
        print(f"{name}: greedy {g / args.new * 1e3:.3f} ms/step {toks / g:.0f} tok/s | sampled {s / args.new * 1e3:.3f} ms/step "
              f"{toks / s:.0f} tok/s | sampled - greedy {(s - g) / args.new * 1e6:+.1f} us/step ({len(t['greedy'])} calls each)")
    eng.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=32, help="tokens generated per sequence and call")
    ap.add_argument("--seconds", type=float, default=2.0, help="timed window per comparison")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    ns.lib().bestla_init()
    print(f"card: {card()}")
    kernel_times()
    generation(args)


if __name__ == "__main__":
    main()

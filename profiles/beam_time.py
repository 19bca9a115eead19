"""Cost of a beam-search step (ns_llama_beam_search) against a batched greedy step (ns_llama_generate_batch) of as many rows.

Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000; BesTLA int4 weights, group 128, int8
compute, generated on the device), n_ctx 1024, 32 KV blocks; num_beams B = 4 over R = 1 / 4 / 8 requests of 128-token prompts.
A step's time is (search with 64 new tokens - search with 1) / 63 -- the difference removes the prompt pass -- against
generate_batch on R B rows at position 128, 64 tokens per call / 64; the two are alternated in one process, medians of --rounds
rounds, host clock around calls that end in a device synchronise.  Also the candidates kernel alone on R B rows: CUDA events
around 200 launches issued one by one from Python -- launch-bound, an upper bound set by the host's issue rate, not the kernel's
time -- and the KV bytes a step can copy: at most B - 1 beams per request, each receiving every
generated position of every layer's K and V.  Prints the card and its power limit beside the numbers.

  python profiles/beam_time.py [--rounds N]
"""
import argparse
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

import neural_speed_b200 as ns  # noqa: E402
from profiles.batch_time import card  # noqa: E402

N_VOCAB, N_EMBD, N_HEAD, N_LAYER, N_FF, N_CTX, N_SEQ, N_PROMPT, N_NEW, B = 32000, 4096, 32, 32, 11008, 1024, 32, 128, 64, 4


def clock(fn):
    t0 = time.perf_counter()
    fn()
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    L = ns.lib()
    L.bestla_init()
    rng = np.random.default_rng(0)
    E, FF = N_EMBD, N_FF
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    eng = ns.Llama(n_vocab=N_VOCAB, n_embd=E, n_head=N_HEAD, n_head_kv=N_HEAD, n_layer=N_LAYER, n_ff=FF, n_ctx=N_CTX, norm_eps=1e-5)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, (rng.standard_normal((N_VOCAB, E), dtype=np.float32) * 0.05).astype(np.float32))
    eng.set_f32(ns.Llama.OUT_NORM, 0, rng.uniform(0.5, 1.5, E).astype(np.float32))
    eng.set_weight(ns.Llama.OUTPUT, 0, ns.Weight.random(N_VOCAB, E, group=128, seed=999))
    for il in range(N_LAYER):
        eng.set_f32(ns.Llama.ATTN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        eng.set_f32(ns.Llama.FFN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        for t, (n, k) in shapes.items():
            eng.set_weight(t, il, ns.Weight.random(n, k, group=128, seed=il * 8 + t))
    eng.set_sequences(N_SEQ)
    print(f"card: {card()}")
    print(f"7B shapes, 32 layers, int4 g128 int8 compute; {N_PROMPT}-token prompts, {N_NEW} new tokens, num_beams {B}")
    hd = E // N_HEAD
    for R in (1, 4, 8):
        prompts = [rng.integers(3, N_VOCAB, N_PROMPT).tolist() for _ in range(R)]
        rows = R * B
        eng.beam_search(prompts, B, N_NEW, eos_token_id=N_VOCAB - 1)  # captures every graph
        eng.generate_batch(list(range(rows)), [5] * rows, [N_PROMPT] * rows, N_NEW)
        full, one, greedy = [], [], []
        for _ in range(args.rounds):
            full.append(clock(lambda: eng.beam_search(prompts, B, N_NEW, eos_token_id=N_VOCAB - 1)))
            one.append(clock(lambda: eng.beam_search(prompts, B, 1, eos_token_id=N_VOCAB - 1)))
            greedy.append(clock(lambda: eng.generate_batch(list(range(rows)), [5] * rows, [N_PROMPT] * rows, N_NEW)))
        step = (np.median(full) - np.median(one)) / (N_NEW - 1) * 1e3
        g = np.median(greedy) / N_NEW * 1e3
        # the candidates kernel alone on R B rows of logits
        x = torch.randn(rows, N_VOCAB, device="cuda")
        ws = torch.zeros(L.ns_llama_beam_candidates_workspace_bytes(rows, 2 * B), dtype=torch.uint8, device="cuda")
        out = torch.zeros(rows, 2 * B, 2, dtype=torch.int32, device="cuda")
        prev, mask = np.zeros(rows, np.float32), np.zeros(rows, np.int32)
        for _ in range(10):
            ns.beam_candidates(x.data_ptr(), rows, N_VOCAB, 2 * B, prev, mask, 2, out.data_ptr(), ws.data_ptr())
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(200):
            ns.beam_candidates(x.data_ptr(), rows, N_VOCAB, 2 * B, prev, mask, 2, out.data_ptr(), ws.data_ptr())
        e1.record()
        torch.cuda.synchronize()
        kern_us = e0.elapsed_time(e1) / 200 * 1e3  # launch-bound: each launch is issued from Python through ctypes
        per_pos = N_LAYER * 2 * N_HEAD * hd * 2  # bytes of one position of one block
        copy_mb = R * (B - 1) * per_pos * (N_NEW // 2) / 2 ** 20
        print(f"R {R} ({rows} rows): beam step {step:.3f} ms, generate_batch step {g:.3f} ms ({step / g:.2f}x); candidates kernel "
              f"{kern_us:.1f} us per launch (launch-bound); candidates copied to the host {rows * 2 * B * 8} B per step; KV copy at most {copy_mb:.1f} MB per "
              f"step at position {N_NEW // 2} ({per_pos / 2 ** 20:.2f} MB per position per copied beam)")


if __name__ == "__main__":
    main()

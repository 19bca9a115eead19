"""Throughput of continuous batching (ns_llama_generate_batch) against one sequence through ns_llama_generate.

Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008, vocab 32000; BesTLA int4 weights, group 128
(the GPTQ / AWQ layout), int8 compute, generated on the device), n_ctx 1024, 32 KV blocks, every sequence holding a 512-token prompt.  For n = 1, 2, 4, 8, 16,
32 sequences, generate_batch produces N_NEW tokens per sequence from position 512 on (each call restarts there, so every step
attends 512 .. 512 + N_NEW - 1 cached positions); calls are repeated for at least --seconds, timed with a host clock around
each call (which ends in a device synchronise).  ns_llama_generate on sequence 0 with the same N_NEW is alternated with the n = 1
batched call in the same process.  Prints the card and its power limit, tokens/s (n x N_NEW / time) and the byte model of a step
(the weights once + the K/V rows every sequence reads).  Last, the batched decode attention of one layer on its own
(ns_llama_attention_batch, n = 32 rows at position 512 of their blocks): host clock around 200 calls and a device synchronise,
each call including its 640-byte upload of the rows' positions -- an upper bound of the kernel's time, times 32 layers.

  python profiles/batch_time.py [--new N_NEW] [--seconds S]
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


def timed(fn, seconds):
    """median seconds per call over calls repeated for at least `seconds` (after one warm-up call)"""
    fn()
    ts, t_end = [], time.perf_counter() + seconds
    while time.perf_counter() < t_end or len(ts) < 3:
        t0 = time.perf_counter()
        fn()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), len(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--new", type=int, default=32, help="tokens generated per sequence and call")
    ap.add_argument("--seconds", type=float, default=1.5, help="timed window per point")
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
    eng.set_sequences(N_SEQ)
    for s in range(N_SEQ):
        eng.eval_seq(s, [int(t) for t in rng.integers(3, N_VOCAB, N_PAST)], 0, want_logits=False)
    hd = E // N_HEAD
    mean_len = N_PAST + (args.new + 1) / 2  # positions a step attends, averaged over the call
    kv_row = 2 * N_LAYER * N_HEAD * mean_len * hd * 2  # K and V read by one sequence's step
    print(f"card: {card()}")
    print(f"7B shapes, {N_LAYER} layers, int4 g128 weights (int8 compute), n_ctx {N_CTX}, {N_SEQ} KV blocks ({eng.kv_bytes() / 1e9:.1f} GB), "
          f"every sequence at {N_PAST} cached positions, {args.new} new tokens per sequence and call, >= {args.seconds} s per point")
    print(f"byte model per step: weights {weight_bytes / 1e9:.3f} GB once + K/V {kv_row / 1e6:.1f} MB per sequence")
    print(f"{'n':>3} {'ms/step':>8} {'tok/s':>8} {'GB/step':>8} {'GB/s':>7} calls")
    firsts = rng.integers(3, N_VOCAB, N_SEQ).astype(np.int32)
    base = None
    for n in (1, 2, 4, 8, 16, 32):
        seqs = np.arange(n, dtype=np.int32)
        call = lambda: eng.generate_batch(seqs, firsts[:n], np.full(n, N_PAST, np.int32), args.new)  # noqa: E731
        if n == 1:  # alternated with the single-sequence graph on the same block and positions
            single = lambda: eng.generate(int(firsts[0]), N_PAST, args.new)  # noqa: E731
            call(), single()
            tb, ts = [], []
            t_end = time.perf_counter() + 2 * args.seconds
            while time.perf_counter() < t_end or len(tb) < 3:
                t0 = time.perf_counter()
                call()
                t1 = time.perf_counter()
                single()
                tb.append(t1 - t0)
                ts.append(time.perf_counter() - t1)
            t, calls = float(np.median(tb)), len(tb)
            base = float(np.median(ts))
        else:
            t, calls = timed(call, args.seconds)
        step = t / args.new
        gb = (weight_bytes + n * kv_row) / 1e9
        print(f"{n:>3} {step * 1e3:>8.3f} {n * args.new / t:>8.0f} {gb:>8.3f} {gb / step:>7.0f} {calls}")
    print(f"ns_llama_generate, one sequence, same positions: {base / args.new * 1e3:.3f} ms/step, {args.new / base:.0f} tok/s "
          f"(batched n = 1 alternated with it above)")
    eng.close()
    del eng
    n, H = N_SEQ, N_HEAD
    q = torch.randn((n, H * hd), device="cuda")
    k, v = torch.randn_like(q), torch.randn_like(q)
    kc = torch.randn((n, H, N_CTX, hd), device="cuda").half()
    vc = torch.randn_like(kc)
    out = torch.empty_like(q)
    ws = torch.zeros(L.ns_llama_attention_batch_workspace_bytes(n, H, hd, N_CTX), dtype=torch.uint8, device="cuda")
    seqs, past = np.arange(n, dtype=np.int32), np.full(n, N_PAST, np.int32)

    def attn():
        rc = ns.attention_batch(q.data_ptr(), k.data_ptr(), v.data_ptr(), kc.data_ptr(), vc.data_ptr(), n, seqs, past, H, H, hd, N_CTX,
                                out.data_ptr(), ws.data_ptr())
        assert rc == 0, ns.last_error()

    for _ in range(20):
        attn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(200):
        attn()
    torch.cuda.synchronize()
    ta = (time.perf_counter() - t0) / 200
    kv_read = n * 2 * H * (N_PAST + 1) * hd * 2
    print(f"batched decode attention, one layer, {n} rows at {N_PAST} cached positions: {ta * 1e6:.1f} us per call "
          f"({kv_read / ta / 1e9:.0f} GB/s of K/V), x {N_LAYER} layers = {ta * N_LAYER * 1e3:.2f} ms of a step")


if __name__ == "__main__":
    main()

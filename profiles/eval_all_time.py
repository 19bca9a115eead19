"""Scoring every token in one pass (ns_llama_eval_all) against the ways the eval step could score before it.

Llama-2-7B shapes with all 32 layers (n_embd 4096, 32 heads of 128, n_ff 11008; BesTLA int4 weights, group 128, int8 compute,
generated on the device), with an int4 g128 int8-compute lm_head and, separately, a Q6_K lm_head (random blocks with a fixed
scale: the kernels' speed does not depend on the values), at vocab 32000 and 128256.
  (a) one 2048-token segment: eval_all with targets only, eval_all with logits_host too, and eval_batch (last row only);
  (b) an lm-eval-shaped load, 32 requests of 128 tokens: one eval_all over all of them, 32 single-segment eval_all calls, and one
      ns_llama_eval per token with a host log-softmax of its logits -- that last arm is timed over one request's 128 tokens and
      extrapolated x32 (printed as such);
  (c) the log-prob kernel alone over 32 rows, CUDA events around >= 200 back-to-back launches; bytes read (rows x n_vocab x 4)
      per second against the data sheet's 3.35 TB/s.
The arms of (a) and (b) alternate in one process after a warm-up of every shape, each timed with a host clock around a call that
ends in a device synchronise; medians are printed with the card's name and power limit.

  python profiles/eval_all_time.py [--reps N] [--vocabs 32000,128256]
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

N_EMBD, N_HEAD, N_LAYER, N_FF = 4096, 32, 32, 11008
SEG, N_REQ, REQ_LEN = 2048, 32, 128


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True,
                           timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # the name from torch alone, the limit unknown
        q = f"{torch.cuda.get_device_name(0)}, power limit unknown ({e})"
    return q


def q6k_random(n, k, seed):
    """n rows of k / 256 block_q6_K (210 bytes: ql[128] qh[64] scales[16] d) with random codes and d = 2^-10"""
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, 256, (n, k // 256, 210), dtype=np.uint8)
    rows[:, :, 208:210] = np.frombuffer(np.float16(2 ** -10).tobytes(), np.uint8)
    return ns.Weight.from_q6_K_host(rows.reshape(n, -1), n, k)


def engine(layers, out_w, tok, V, n_ctx, n_seq, rng):
    E = N_EMBD
    eng = ns.Llama(n_vocab=V, n_embd=E, n_head=N_HEAD, n_head_kv=N_HEAD, n_layer=N_LAYER, n_ff=N_FF, n_ctx=n_ctx, norm_eps=1e-5)
    eng.set_f32(ns.Llama.TOK_EMBD, 0, tok)
    eng.set_f32(ns.Llama.OUT_NORM, 0, rng.uniform(0.5, 1.5, E).astype(np.float32))
    eng.set_weight(ns.Llama.OUTPUT, 0, out_w)
    for il in range(N_LAYER):
        eng.set_f32(ns.Llama.ATTN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        eng.set_f32(ns.Llama.FFN_NORM, il, rng.uniform(0.5, 1.5, E).astype(np.float32))
        for t, w in layers[il].items():
            eng.set_weight(t, il, w)
    if n_seq > 1:
        eng.set_sequences(n_seq)
    return eng


def alternate(arms, reps):
    """arms: {name: fn}; warm-up twice, then reps rounds in turn -> {name: median seconds}"""
    for _ in range(2):
        for fn in arms.values():
            fn()
    ts = {k: [] for k in arms}
    for _ in range(reps):
        for k, fn in arms.items():
            t0 = time.perf_counter()
            fn()
            ts[k].append(time.perf_counter() - t0)
    return {k: float(np.median(v)) for k, v in ts.items()}


def log_softmax_host(x, t):
    m = x.max()
    return float(x[t] - m - np.log(np.exp(x - m, dtype=np.float32).sum(dtype=np.float32)))


def kernel_time(V, rows=32, launches=400):
    x = torch.randn(rows, V, device="cuda")
    t = torch.randint(0, V, (rows,), dtype=torch.int32, device="cuda")
    lp = torch.zeros(rows, device="cuda")
    am = torch.zeros(rows, dtype=torch.int32, device="cuda")
    ws = torch.zeros(ns.lib().ns_llama_logprob_workspace_bytes(rows, V), dtype=torch.uint8, device="cuda")
    st = torch.cuda.current_stream().cuda_stream

    def one():
        assert ns.logprob(x.data_ptr(), rows, V, t.data_ptr(), lp.data_ptr(), am.data_ptr(), ws.data_ptr(), st) == 0, ns.last_error()

    for _ in range(20):
        one()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(launches):
        one()
    e1.record()
    torch.cuda.synchronize()
    sec = e0.elapsed_time(e1) / 1e3 / launches
    return sec, rows * V * 4 / sec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5, help="alternating rounds per point")
    ap.add_argument("--vocabs", default="32000,128256")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs the GPU"
    L = ns.lib()
    L.bestla_init()
    print(f"card: {card()}")
    rng = np.random.default_rng(0)
    E, FF = N_EMBD, N_FF
    shapes = {ns.Llama.WQ: (E, E), ns.Llama.WK: (E, E), ns.Llama.WV: (E, E), ns.Llama.WO: (E, E), ns.Llama.W1: (FF, E),
              ns.Llama.W2: (E, FF), ns.Llama.W3: (FF, E)}
    layers = [{t: ns.Weight.random(n, k, group=128, seed=il * 8 + t) for t, (n, k) in shapes.items()} for il in range(N_LAYER)]
    vocabs = [int(v) for v in args.vocabs.split(",")]
    print("(c) log-prob kernel alone, 32 rows, CUDA events over 400 launches")
    for V in vocabs:
        sec, bps = kernel_time(V)
        print(f"    vocab {V:>6}: {sec * 1e6:7.1f} us/launch, {bps / 1e12:.2f} TB/s of logits read ({100 * bps / 3.35e12:.1f} % of 3.35 TB/s)")
    for V in vocabs:
        tok = (rng.standard_normal((V, E), dtype=np.float32) * 0.05).astype(np.float32)
        for head in ("int4", "q6_K"):
            out_w = ns.Weight.random(V, E, group=128, seed=999) if head == "int4" else q6k_random(V, E, 999)
            # (a) one 2048-token segment
            eng = engine(layers, out_w, tok, V, SEG, 1, rng)
            seg = [int(t) for t in rng.integers(3, V, SEG)]
            tg = [seg[1:] + [seg[0]]]
            res = alternate({
                "eval_all targets": lambda: eng.eval_all([0], [seg], [0], targets=tg),
                "eval_all + logits": lambda: eng.eval_all([0], [seg], [0], targets=tg, want_logits=True),
                "eval_batch last row": lambda: eng.eval_batch([0], [seg], [0], want_logits=False),
            }, args.reps)
            base = res["eval_batch last row"]
            print(f"(a) vocab {V} lm_head {head}, one {SEG}-token segment (medians of {args.reps}):")
            for k, v in res.items():
                print(f"    {k:<22} {v * 1e3:9.2f} ms  (+{(v - base) * 1e3:8.2f} ms over the last row only)")
            eng.close()
            # (b) 32 requests of 128 tokens
            eng = engine(layers, out_w, tok, V, REQ_LEN, N_REQ, rng)
            reqs = [[int(t) for t in rng.integers(3, V, REQ_LEN)] for _ in range(N_REQ)]
            tgs = [r[1:] + [r[0]] for r in reqs]
            seqs = list(range(N_REQ))

            def per_token_one_request():
                r, t = reqs[0], tgs[0]
                for p in range(REQ_LEN):
                    lg, _ = eng.eval([r[p]], p)
                    log_softmax_host(lg, t[p])

            res = alternate({
                "one eval_all": lambda: eng.eval_all(seqs, reqs, [0] * N_REQ, targets=tgs),
                "32 eval_all calls": lambda: [eng.eval_all([s], [reqs[s]], [0], targets=[tgs[s]]) for s in seqs],
                "per token (1 request)": per_token_one_request,
            }, max(2, args.reps // 2))
            one = res["one eval_all"]
            print(f"(b) vocab {V} lm_head {head}, {N_REQ} requests x {REQ_LEN} tokens:")
            print(f"    one eval_all (T = {N_REQ * REQ_LEN})    {one * 1e3:9.2f} ms")
            print(f"    {N_REQ} single-segment eval_all {res['32 eval_all calls'] * 1e3:9.2f} ms  ({res['32 eval_all calls'] / one:.2f}x)")
            ext = res["per token (1 request)"] * N_REQ
            print(f"    ns_llama_eval per token + host log-softmax: {res['per token (1 request)'] * 1e3:.1f} ms for one request, "
                  f"x{N_REQ} extrapolated = {ext * 1e3:9.1f} ms  ({ext / one:.1f}x)")
            eng.close()
            del out_w


if __name__ == "__main__":
    main()

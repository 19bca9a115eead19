"""Two-GPU tensor-parallel layer: shards from ns_split_weight, matmuls in libns_b200, NCCL sum all-reduce after o-proj and
down-proj (llama.cpp:592,693).  Needs 2 GPUs; skipped on a single-GPU machine."""
import os
import socket

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import traceback
    try:
        import torch.distributed as dist
        import neural_speed_b200 as ns
        import oracle
        from neural_speed_b200 import tp
        torch.cuda.set_device(rank)
        ns.lib().bestla_init()
        ctx = tp.TPContext(backend="nccl")
        n_embd, n_ff, n_head, g, m = 1024, 2048, 8, 128, 1
        plan = tp.LlamaShardPlan(world, n_embd, n_ff, n_head, n_head, g)
        dims = {"wq": (n_embd, n_embd), "wk": (n_embd, n_embd), "wv": (n_embd, n_embd), "wo": (n_embd, n_embd),
                "w1": (n_ff, n_embd), "w3": (n_ff, n_embd), "w2": (n_embd, n_ff)}
        full = {}
        for i, (name, (nn, kk)) in enumerate(dims.items()):
            w = np.random.default_rng(50 + i).uniform(-0.05, 0.05, (nn, kk)).astype(np.float32)
            full[name] = ns.np_bestla_quantize(w, "int4", g, "sym", "fp32", "fp32")
        sh = plan.shapes()
        shards = {r: {name: tp.split_blob(full[name], *dims[name], world, r, sh[name][0]) for name in dims} for r in range(world)}
        layer = {name: ns.Weight.from_blob(shards[rank][name]) for name in dims}
        x = torch.from_numpy(np.random.default_rng(9).uniform(-0.5, 0.5, (m, n_embd)).astype(np.float32)).cuda()
        eng = tp.TPLlamaMatmuls(plan, [layer], ctx)
        out = eng.layer(0, x)
        torch.cuda.synchronize()
        ns.lib().bestla_device_sync(None)
        # expectation from the dequantised shards (fp32 compute, tolerance 1e-3 as sycl_gemm.cpp:404-442)
        xs = x.cpu().numpy()
        dq = {r: {name: ns.unpack_blob(shards[r][name], sh[name][1], sh[name][2]) for name in dims} for r in range(world)}
        o = sum(oracle.gemm_f64acc(oracle.gemm_f64acc(xs, dq[r]["wq"]), dq[r]["wo"]).astype(np.float64) for r in range(world))
        h = (xs + o).astype(np.float32)

        def mid(r):
            gt = oracle.gemm_f64acc(h, dq[r]["w1"])
            return (gt / (1 + np.exp(-gt)) * oracle.gemm_f64acc(h, dq[r]["w3"])).astype(np.float32)

        dn = sum(oracle.gemm_f64acc(mid(r), dq[r]["w2"]).astype(np.float64) for r in range(world))
        want = h + dn
        err = float(np.abs(out.cpu().numpy() - want).max())
        assert err <= 2e-3, err
        gathered = [torch.empty_like(out) for _ in range(world)]
        dist.all_gather(gathered, out)
        assert all(torch.equal(gathered[0], t) for t in gathered)   # every rank holds the same activation after the all-reduce
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception:
        q.put((rank, traceback.format_exc()))


def _worker_p2p(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    import traceback
    try:
        import time
        import torch.distributed as dist
        import neural_speed_b200 as ns
        from neural_speed_b200 import tp
        torch.cuda.set_device(rank)
        ns.lib().bestla_init()
        ctx = tp.TPContext(backend="nccl")
        assert ctx.enable_p2p(16384)
        g = torch.Generator(device="cuda").manual_seed(100 + rank)
        gsame = torch.Generator(device="cuda").manual_seed(7)      # the residual (layer input) is the same on every rank
        for n in (4096, 8192, 16384, 4):
            for it in range(6):
                x = torch.randn(n, device="cuda", generator=g)
                res = torch.randn(n, device="cuda", generator=gsame) if it % 2 else None
                want = x.clone()
                dist.all_reduce(want)                       # NCCL
                if res is not None:
                    want = want + res
                got = ctx.all_reduce(x.clone(), residual=res)
                torch.cuda.synchronize()
                assert torch.allclose(got, want, rtol=1e-5, atol=1e-5), (n, it, float((got - want).abs().max()))
                gathered = [torch.empty_like(got) for _ in range(world)]
                dist.all_gather(gathered, got)
                assert all(torch.equal(gathered[0], t) for t in gathered)  # fixed rank order -> bit-identical on every rank
        assert ns.lib().ns_comm_status(ctx._comm) == 0
        # latency, 8192 floats (the [1, n_embd] partial of Llama-2-70B), back to back on one stream
        x = torch.randn(8192, device="cuda")
        for fn, name in ((lambda: ctx.all_reduce(x), "p2p"), (lambda: dist.all_reduce(x), "nccl")):
            for _ in range(20):
                fn()
            torch.cuda.synchronize()
            dist.barrier()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(200):
                fn()
            e1.record()
            torch.cuda.synchronize()
            if rank == 0:
                print(f"all-reduce 32 KB {name}: {e0.elapsed_time(e1) / 200 * 1e3:.2f} us", flush=True)
            x.normal_()
        dist.barrier()
        dist.destroy_process_group()
        q.put((rank, "ok"))
    except Exception:
        q.put((rank, traceback.format_exc()))


def test_two_gpu_oneshot_nvlink_all_reduce(capfd):
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker_p2p, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


def test_two_gpu_tensor_parallel_layer():
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    world, port = 2, _free_port()
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    procs = [ctx.Process(target=_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=60)
    assert sorted(res) == [(0, "ok"), (1, "ok")], res


@pytest.mark.parametrize("world", [2, 4, 8])
def test_one_gpu_loopback_of_the_exchange_and_the_k_split(world):
    """The tensor-parallel exchange on ONE device: `world` ranks' communicators live in this process (ns_comm_link_local wires
    their buffers by pointer instead of cudaIpc), every rank runs its all-reduce kernel on its own stream, so the kernels are
    co-resident and really wait on each other's flags.  The partials come from a K-split o-projection (ns_split_weight shards,
    model_files.h:1650-1672): the reduced result must equal the unsplit matmul within the fp32-compute tolerance, every rank must
    hold bit-identical sums, and the step counters must survive many back-to-back steps (both parities, CUDA-graph-style replay)."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import ctypes as C
    import neural_speed_b200 as ns
    import oracle
    from neural_speed_b200 import tp
    L = ns.lib()
    L.bestla_init()
    L.ns_comm_link_local.argtypes = [C.c_void_p, C.c_int]
    n, k, g = 1024, 2048, 128
    rng = np.random.default_rng(77)
    w = rng.uniform(-0.05, 0.05, (n, k)).astype(np.float32)
    blob = ns.np_bestla_quantize(w, "int4", g, "sym", "fp32", "fp32")
    x = rng.uniform(-0.5, 0.5, (1, k)).astype(np.float32)
    res = rng.normal(0, 1, (1, n)).astype(np.float32)
    kl = k // world
    shards = [ns.Weight.from_blob(tp.split_blob(blob, n, k, world, r, tp.SPLIT_K)) for r in range(world)]
    streams = [torch.cuda.Stream() for _ in range(world)]
    comms = [C.c_void_p(L.ns_comm_create(r, world, n, None)) for r in range(world)]
    assert all(c.value for c in comms), ns.last_error()
    arr = (C.c_void_p * world)(*[c.value for c in comms])
    assert L.ns_comm_link_local(arr, world) == 0, ns.last_error()
    xs = [torch.from_numpy(np.ascontiguousarray(x[:, r * kl:(r + 1) * kl])).cuda() for r in range(world)]
    resid = torch.from_numpy(res).cuda()
    parts = [torch.zeros(1, n, device="cuda") for _ in range(world)]
    torch.cuda.synchronize()
    want = None
    for step in range(5):  # both parities of the slot buffers, several wraps of the arrival counters
        for r in range(world):
            q = C.c_void_p(streams[r].cuda_stream)
            ns.mul_mat(shards[r], xs[r].data_ptr(), kl, parts[r].data_ptr(), n, 1, queue=q)
            rc = L.ns_comm_all_reduce_f32(comms[r], C.c_void_p(parts[r].data_ptr()), n, C.c_void_p(resid.data_ptr()), q)
            assert rc == 0, ns.last_error()
        torch.cuda.synchronize()
        got = [p.cpu().numpy().copy() for p in parts]
        for r in range(1, world):
            assert np.array_equal(got[0], got[r]), f"rank {r} differs from rank 0 at step {step}"
        if want is None:
            wdq = ns.unpack_blob(blob, n, k)  # [K, N]
            want = oracle.gemm_f64acc(x, wdq) + res
            # shards are re-quantised slices (bestla_split_weight): compare against THEIR dequantised sum as well
            sh = sum(oracle.gemm_f64acc(np.ascontiguousarray(x[:, r * kl:(r + 1) * kl]),
                                        ns.unpack_blob(tp.split_blob(blob, n, k, world, r, tp.SPLIT_K), n, kl)).astype(np.float64)
                     for r in range(world)) + res
            assert np.abs(got[0] - sh).max() <= 1e-3
            assert np.abs(got[0] - want).max() <= 0.2  # re-quantising the int4 slices moves the weights a little (outputs are O(1))
        for r in range(world):
            assert L.ns_comm_status(comms[r]) == 0
    for c in comms:
        L.ns_comm_free(c)

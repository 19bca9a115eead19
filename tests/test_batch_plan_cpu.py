"""ns_llama_batch_plan (include/ns_b200.h): the host plan of ns_llama_eval_batch on its own, without a device.

Internal order: the one-token segments first, then the longer ones, each group in the caller's order.  Rows carry their position
and KV block; each multi-token segment gets one tile entry per 64 query rows, its first row counted from internal row d (the first
multi-token row).  Every refusal of the call returns NS_E_INVALID with its reason."""
import numpy as np
import pytest

import neural_speed_b200 as ns

E_INVALID = -1


def _want(seqs, n_tokens, n_past):
    order = [i for i in range(len(seqs)) if n_tokens[i] == 1] + [i for i in range(len(seqs)) if n_tokens[i] > 1]
    d = sum(1 for t in n_tokens if t == 1)
    rows, tiles, r = [], [], 0
    for j, i in enumerate(order):
        rows += [(n_past[i] + t, seqs[i]) for t in range(n_tokens[i])]
        if j >= d:
            tiles += [(r - d, n_tokens[i], n_past[i], seqs[i], q0) for q0 in range(0, n_tokens[i], 64)]
        r += n_tokens[i]
    return order, np.array(rows, np.int32).reshape(-1, 2), d, np.array(tiles, np.int32).reshape(-1, 5)


@pytest.mark.parametrize("case", [
    dict(seqs=[3, 0, 5, 1], n_tokens=[1, 7, 1, 130], n_past=[40, 0, 9, 100]),  # decodes between prompts
    dict(seqs=[2], n_tokens=[64], n_past=[0]),                                  # one full tile
    dict(seqs=[2, 7], n_tokens=[65, 63], n_past=[1, 2]),                        # one row past a tile, one row short of one
    dict(seqs=[0, 1, 2], n_tokens=[1, 1, 1], n_past=[0, 5, 255]),               # decode only: no tiles
    dict(seqs=[4, 0, 6, 2, 1], n_tokens=[200, 2, 1, 128, 1], n_past=[56, 0, 255, 128, 0]),
])
def test_order_rows_tiles_and_d(case):
    seqs, n_tokens, n_past = case["seqs"], case["n_tokens"], case["n_past"]
    rc, plan = ns.batch_plan(8, 256, seqs, n_tokens, n_past)
    assert rc == 0, ns.last_error()
    order, rows, d, tiles = _want(seqs, n_tokens, n_past)
    assert list(plan["order"]) == order
    assert plan["d"] == d
    assert np.array_equal(plan["rows"], rows)
    assert np.array_equal(plan["tiles"], tiles)
    # every multi-token row is covered by exactly one tile row, and tiles start at 64-row boundaries of their segment
    covered = np.zeros(len(rows), np.int32)
    for first, ln, _, _, q0 in plan["tiles"]:
        assert q0 % 64 == 0 and q0 < ln
        covered[d + first + q0:d + first + min(q0 + 64, ln)] += 1
    assert np.array_equal(covered[d:], np.ones(len(rows) - d, np.int32)) and not covered[:d].any()


def test_the_order_is_stable_within_each_group():
    rng = np.random.default_rng(3)
    seqs = rng.permutation(32).astype(np.int32)
    n_tokens = rng.choice([1, 1, 2, 9, 70], 32).astype(np.int32)
    n_past = rng.integers(0, 100, 32).astype(np.int32)
    rc, plan = ns.batch_plan(32, 512, seqs, n_tokens, n_past)
    assert rc == 0, ns.last_error()
    ones = [i for i in range(32) if n_tokens[i] == 1]
    assert list(plan["order"]) == ones + [i for i in range(32) if n_tokens[i] > 1]
    assert plan["d"] == len(ones)
    assert np.array_equal(plan["rows"], _want(seqs.tolist(), n_tokens.tolist(), n_past.tolist())[1])


def test_the_row_cap_is_4096():
    rc, plan = ns.batch_plan(2, 4096, [0, 1], [4000, 96], [0, 0])
    assert rc == 0 and len(plan["rows"]) == 4096 and len(plan["tiles"]) == 63 + 2
    assert ns.batch_plan(2, 4096, [0, 1], [4000, 97], [0, 0])[0] == E_INVALID
    assert "4097 rows in one pass, at most 4096" in ns.last_error()


@pytest.mark.parametrize("args,text", [
    ((4, 64, [0, 4], [1, 1], [0, 0]), "sequence id 4 outside [0, 4)"),
    ((4, 64, [-1], [1], [0]), "sequence id -1 outside [0, 4)"),
    ((4, 64, [2, 2], [1, 3], [0, 0]), "sequence id 2 appears twice"),
    ((4, 64, [0, 1, 2, 3, 0], [1] * 5, [0] * 5), "n 5 outside [1, n_seq 4]"),
    ((4, 64, [], [], []), "n 0 outside [1, n_seq 4]"),
    ((4, 64, [1, 2], [1, 0], [0, 0]), "segment 1: n_tokens 0 < 1"),
    ((4, 64, [1], [-3], [0]), "segment 0: n_tokens -3 < 1"),
    ((4, 64, [1], [1], [-1]), "n_past -1"),
    ((4, 64, [1], [5], [60]), "sequence 1: n_past 60 + 5 tokens outside n_ctx 64"),
    ((4, 64, [1], [1], [64]), "outside n_ctx 64"),
    ((0, 64, [0], [1], [0]), "invalid arguments"),
    ((33, 64, [0], [1], [0]), "invalid arguments"),
])
def test_refusals(args, text):
    rc, plan = ns.batch_plan(*args)
    assert rc == E_INVALID and plan is None
    assert text in ns.last_error(), ns.last_error()


def test_null_pointers_are_refused():
    import ctypes as C
    L = ns.lib()
    a = np.zeros(8, np.int32)
    p = a.ctypes.data_as(C.c_void_p)
    for nulled in range(7):
        ptrs = [p] * 7
        ptrs[nulled] = None
        assert L.ns_llama_batch_plan(4, 64, 1, *ptrs) == E_INVALID and "null pointer" in ns.last_error(), nulled

"""The decode GEMV's launch plan (ns_gemv_ring_plan: ns_gemv_ring_choose in csrc/gemv_ring.cu, the one function both ring launchers
and ns_route ask) at real model shapes, without a device.  The table agrees entry for entry with the planning code the launchers
ran before it was gathered into that function, so it pins the plan every launch ran with then: a planner change shows up here first.
Each entry: (wide, weight rows per ring stage, stages, stage-owning consumer warps, CTAs per SM), or None when no plan fits."""
import ctypes as C

import pytest

import neural_speed_b200 as ns

FMTS = {"q4_0": (32, ns.S_F16, 0, ns.COMP_Q8_0), "g32-f32": (32, ns.S_F32, 0, ns.COMP_INT8),
        "g128-bf16-asym": (128, ns.S_BF16, 1, ns.COMP_INT8)}
# name: (mode, activation rows, fused (the kernel quantises fp32 rows) or prepared image, folded RMSNorm)
LAUNCH = {"m1": (0, 1, 1, 0), "m1-prepared": (0, 1, 0, 0), "m1-norm": (0, 1, 1, 1), "m1-gate-up": (2, 1, 1, 0), "m2": (0, 2, 1, 0),
          "m2-norm": (0, 2, 1, 1), "m4": (0, 4, 1, 0), "m4-prepared": (0, 4, 0, 0)}
# launches a tile of that many rows cannot take (ns_gemv_tile_rows) are absent
TABLE = {
    # q4_0
    ("q4_0", 1024): {"m1": (1, 2, 56, 14, 1), "m1-prepared": (0, 2, 28, 7, 2), "m1-norm": (1, 2, 56, 14, 1), "m1-gate-up": (1, 2, 56, 14, 1), "m2": (0, 2, 28, 7, 2), "m2-norm": (0, 2, 28, 7, 2), "m4": (0, 2, 28, 7, 2), "m4-prepared": (0, 2, 28, 7, 2)},
    ("q4_0", 4096): {"m1": (1, 2, 42, 14, 1), "m1-prepared": (0, 2, 21, 7, 2), "m1-norm": (1, 2, 42, 14, 1), "m1-gate-up": (1, 2, 42, 14, 1), "m2": (0, 2, 21, 7, 2), "m2-norm": (0, 2, 21, 7, 2), "m4": (0, 2, 14, 7, 2), "m4-prepared": (0, 2, 14, 7, 2)},
    ("q4_0", 5120): {"m1": (1, 2, 28, 14, 1), "m1-prepared": (0, 2, 14, 7, 2), "m1-norm": (1, 2, 28, 14, 1), "m1-gate-up": (1, 2, 28, 14, 1), "m2": (0, 2, 14, 7, 2), "m2-norm": (0, 2, 14, 7, 2), "m4": (0, 2, 14, 7, 2), "m4-prepared": (0, 2, 14, 7, 2)},
    ("q4_0", 11008): {"m1": (1, 2, 14, 14, 1), "m1-prepared": (0, 2, 7, 7, 2), "m1-norm": (1, 2, 14, 14, 1), "m1-gate-up": (1, 2, 14, 14, 1), "m2": (0, 2, 7, 7, 2), "m2-norm": (0, 2, 7, 7, 2), "m4": (0, 1, 7, 7, 2), "m4-prepared": (0, 1, 7, 7, 2)},
    ("q4_0", 13824): {"m1": (1, 1, 14, 14, 1), "m1-prepared": (0, 1, 7, 7, 2), "m1-norm": (1, 1, 14, 14, 1), "m1-gate-up": (1, 2, 12, 12, 1), "m2": (0, 1, 7, 7, 2), "m2-norm": (0, 1, 7, 7, 2)},
    ("q4_0", 14336): {"m1": (1, 1, 14, 14, 1), "m1-prepared": (0, 1, 7, 7, 2), "m1-norm": (1, 1, 14, 14, 1), "m1-gate-up": (0, 2, 6, 6, 2), "m2": (0, 1, 7, 7, 2), "m2-norm": (0, 1, 7, 7, 2)},
    ("q4_0", 28672): {"m1": (1, 1, 10, 10, 1), "m1-prepared": (0, 1, 4, 4, 2), "m1-norm": (1, 1, 10, 10, 1), "m1-gate-up": (0, 2, 5, 5, 1)},
    ("q4_0", 32768): {"m1": (1, 1, 8, 8, 1), "m1-prepared": (0, 1, 4, 4, 2), "m1-norm": (1, 1, 8, 8, 1), "m1-gate-up": (1, 2, 4, 4, 1)},
    ("q4_0", 49152): {"m1": (0, 1, 5, 5, 1), "m1-prepared": (0, 1, 5, 5, 1), "m1-norm": (0, 1, 5, 5, 1), "m1-gate-up": (1, 2, 2, 2, 1)},
    # g32-f32
    ("g32-f32", 1024): {"m1": (1, 2, 56, 14, 1), "m1-prepared": (0, 2, 28, 7, 2), "m1-norm": (1, 2, 56, 14, 1), "m1-gate-up": (1, 2, 56, 14, 1), "m2": (0, 2, 28, 7, 2), "m2-norm": (0, 2, 28, 7, 2), "m4": (0, 2, 28, 7, 2), "m4-prepared": (0, 2, 28, 7, 2)},
    ("g32-f32", 4096): {"m1": (1, 2, 28, 14, 1), "m1-prepared": (0, 2, 21, 7, 2), "m1-norm": (1, 2, 28, 14, 1), "m1-gate-up": (1, 2, 28, 14, 1), "m2": (0, 2, 14, 7, 2), "m2-norm": (0, 2, 14, 7, 2), "m4": (0, 2, 14, 7, 2), "m4-prepared": (0, 2, 14, 7, 2)},
    ("g32-f32", 5120): {"m1": (1, 2, 28, 14, 1), "m1-prepared": (0, 2, 14, 7, 2), "m1-norm": (1, 2, 28, 14, 1), "m1-gate-up": (1, 2, 28, 14, 1), "m2": (0, 2, 14, 7, 2), "m2-norm": (0, 2, 14, 7, 2), "m4": (0, 2, 14, 7, 2), "m4-prepared": (0, 2, 14, 7, 2)},
    ("g32-f32", 11008): {"m1": (0, 2, 7, 7, 2), "m1-prepared": (0, 2, 7, 7, 2), "m1-norm": (0, 2, 7, 7, 2), "m1-gate-up": (0, 2, 7, 7, 2), "m2": (0, 1, 7, 7, 2), "m2-norm": (0, 1, 7, 7, 2), "m4": (0, 1, 7, 7, 2), "m4-prepared": (0, 1, 7, 7, 2)},
    ("g32-f32", 13824): {"m1": (1, 1, 14, 14, 1), "m1-prepared": (0, 1, 7, 7, 2), "m1-norm": (1, 1, 14, 14, 1), "m1-gate-up": (1, 2, 10, 10, 1), "m2": (0, 1, 7, 7, 2), "m2-norm": (0, 1, 7, 7, 2)},
    ("g32-f32", 14336): {"m1": (1, 1, 14, 14, 1), "m1-prepared": (0, 1, 7, 7, 2), "m1-norm": (1, 1, 14, 14, 1), "m1-gate-up": (1, 2, 10, 10, 1), "m2": (0, 1, 7, 7, 2), "m2-norm": (0, 1, 7, 7, 2)},
    ("g32-f32", 28672): {"m1": (0, 1, 4, 4, 2), "m1-prepared": (0, 1, 4, 4, 2), "m1-norm": (0, 1, 4, 4, 2), "m1-gate-up": (1, 2, 4, 4, 1)},
    ("g32-f32", 32768): {"m1": (0, 1, 7, 7, 1), "m1-prepared": (0, 1, 7, 7, 1), "m1-norm": (0, 1, 7, 7, 1), "m1-gate-up": (0, 2, 3, 3, 1)},
    ("g32-f32", 49152): {"m1": (1, 1, 4, 4, 1), "m1-prepared": (0, 1, 4, 4, 1), "m1-norm": (1, 1, 4, 4, 1), "m1-gate-up": (1, 2, 2, 2, 1)},
    # g128-bf16-asym
    ("g128-bf16-asym", 1024): {"m1": (1, 2, 56, 14, 1), "m1-prepared": (0, 2, 28, 7, 2), "m1-norm": (1, 2, 56, 14, 1), "m1-gate-up": (1, 2, 56, 14, 1), "m2": (0, 2, 28, 7, 2), "m2-norm": (0, 2, 28, 7, 2), "m4": (0, 2, 28, 7, 2), "m4-prepared": (0, 2, 28, 7, 2)},
    ("g128-bf16-asym", 4096): {"m1": (1, 2, 42, 14, 1), "m1-prepared": (0, 2, 21, 7, 2), "m1-norm": (1, 2, 42, 14, 1), "m1-gate-up": (1, 2, 42, 14, 1), "m2": (0, 2, 21, 7, 2), "m2-norm": (0, 2, 21, 7, 2), "m4": (0, 2, 21, 7, 2), "m4-prepared": (0, 2, 21, 7, 2)},
    ("g128-bf16-asym", 5120): {"m1": (1, 2, 28, 14, 1), "m1-prepared": (0, 2, 14, 7, 2), "m1-norm": (1, 2, 28, 14, 1), "m1-gate-up": (1, 2, 28, 14, 1), "m2": (0, 2, 14, 7, 2), "m2-norm": (0, 2, 14, 7, 2), "m4": (0, 2, 14, 7, 2), "m4-prepared": (0, 2, 14, 7, 2)},
    ("g128-bf16-asym", 11008): {"m1": (1, 2, 14, 14, 1), "m1-prepared": (0, 2, 7, 7, 2), "m1-norm": (1, 2, 14, 14, 1), "m1-gate-up": (1, 2, 14, 14, 1), "m2": (0, 2, 7, 7, 2), "m2-norm": (0, 2, 7, 7, 2), "m4": (0, 1, 7, 7, 2), "m4-prepared": (0, 1, 7, 7, 2)},
    ("g128-bf16-asym", 13824): {"m1": (1, 1, 14, 14, 1), "m1-prepared": (0, 1, 7, 7, 2), "m1-norm": (1, 1, 14, 14, 1), "m1-gate-up": (1, 2, 12, 12, 1), "m2": (0, 1, 7, 7, 2), "m2-norm": (0, 1, 7, 7, 2)},
    ("g128-bf16-asym", 14336): {"m1": (1, 1, 14, 14, 1), "m1-prepared": (0, 1, 7, 7, 2), "m1-norm": (1, 1, 14, 14, 1), "m1-gate-up": (1, 2, 12, 12, 1), "m2": (0, 1, 7, 7, 2), "m2-norm": (0, 1, 7, 7, 2)},
    ("g128-bf16-asym", 28672): {"m1": (0, 1, 5, 5, 2), "m1-prepared": (0, 1, 5, 5, 2), "m1-norm": (0, 1, 5, 5, 2), "m1-gate-up": (0, 2, 5, 5, 1)},
    ("g128-bf16-asym", 32768): {"m1": (0, 1, 4, 4, 2), "m1-prepared": (0, 1, 4, 4, 2), "m1-norm": (0, 1, 4, 4, 2), "m1-gate-up": (1, 2, 4, 4, 1)},
    ("g128-bf16-asym", 49152): {"m1": (0, 1, 5, 5, 1), "m1-prepared": (0, 1, 5, 5, 1), "m1-norm": (0, 1, 5, 5, 1), "m1-gate-up": (1, 2, 2, 2, 1)},
}


def plan(k, g, stype, asym, comp, mode, m, fused, norm):
    out = (C.c_int * 5)()
    rc = ns.lib().ns_gemv_ring_plan(k, g, stype, asym, comp, mode, m, fused, norm, out)
    return rc, (tuple(out) if rc == 1 else None)


@pytest.mark.parametrize("key", list(TABLE), ids=[f"{f}-k{k}" for f, k in TABLE])
def test_plan_table(key):
    fmt, k = key
    g, st, asym, comp = FMTS[fmt]
    for name, (mode, m, fused, norm) in LAUNCH.items():
        rc, got = plan(k, g, st, asym, comp, mode, m, fused, norm)
        if name not in TABLE[key]:
            assert rc < 0, (name, rc)
            continue
        assert rc >= 0, (name, ns.last_error())
        assert got == TABLE[key][name], (name, got)
        if m == 3 or m == 4:  # a 3-row tile runs the 4-row template
            assert plan(k, g, st, asym, comp, mode, 3, fused, norm)[1] == got


def test_every_plan_class_is_reached():
    """the classes tests/test_gpu_ring.py asserts per case, each at a real shape"""
    q4, g32 = FMTS["q4_0"], FMTS["g32-f32"]
    assert plan(4096, *q4, 0, 1, 1, 0)[1] == (1, 2, 42, 14, 1)      # wide, row pairs
    assert plan(13824, *q4, 0, 1, 1, 0)[1] == (1, 1, 14, 14, 1)     # wide, single rows
    assert plan(11008, *g32, 0, 1, 1, 0)[1] == (0, 2, 7, 7, 2)      # wide plan of 13 stages (odd) refused: the two-CTA kernel
    assert plan(28672, *g32, 0, 1, 1, 0)[1] == (0, 1, 4, 4, 2)      # two-CTA, single rows, 4 active warps
    assert plan(32768, *g32, 0, 1, 0, 0)[1] == (0, 1, 7, 7, 1)      # prepared image, whole SM on the 7-warp kernel
    assert plan(49152, *q4, 0, 1, 1, 0)[1] == (0, 1, 5, 5, 1)       # fused, wide refused (5 stages), whole SM on the 7-warp kernel


def test_no_plan_and_invalid_launches():
    g32 = FMTS["g32-f32"]
    assert plan(131072, *g32, 0, 1, 1, 0) == (0, None)              # one 65 KB row pitch: no stage fits next to the activations
    assert plan(131072, *g32, 0, 1, 0, 0) == (0, None)
    assert plan(4096, *g32, 0, 1, 1, 0)[0] == 1
    L = ns.lib()
    out = (C.c_int * 5)()
    assert L.ns_gemv_ring_plan(4096, 32, ns.S_F32, 0, ns.COMP_F32, 0, 1, 0, 0, out) < 0   # float compute: the register GEMV
    assert L.ns_gemv_ring_plan(4096, 32, ns.S_F32, 0, ns.COMP_INT8, 0, 3, 0, 1, out) < 0  # a norm folds into <= 2 rows only
    assert L.ns_gemv_ring_plan(4096, 48, ns.S_F32, 0, ns.COMP_INT8, 0, 1, 0, 0, out) < 0  # groups of 32 multiples (or K)
    assert L.ns_gemv_ring_plan(1000, 1000, ns.S_F32, 1, ns.COMP_INT8, 0, 1, 1, 0, out) < 0  # group K = 1000: prepared path only
    assert L.ns_gemv_ring_plan(1000, 1000, ns.S_F32, 1, ns.COMP_INT8, 0, 1, 0, 0, out) == 1
    assert L.ns_gemv_ring_plan(28672, 32, ns.S_F32, 0, ns.COMP_INT8, 0, 2, 1, 0, out) < 0  # tiles of one row at this K

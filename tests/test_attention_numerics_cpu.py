"""The CPU attention model (oracle/llama_model.py) the GPU attention tests compare against.

* rope_mode0_rows and attention_reference are vectorised restatements of rope_mode0 and of the per-(token, head) attention of
  OracleLlama.eval; they are shown equal to those here (RoPE bit for bit, attention up to the fp32 summation order).
* The stated deviations of the tensor-core prompt attention and of the split-context decode attention from the reference's
  soft_max (DESIGN.md section 4): the reference rounds p = e / sum to fp16 BEFORE the V product (ne_compute_forward_soft_max_f32,
  core/ne_layers.c:8887-8954, then mul_mat(V, P) with P converted to fp16, :6943-7083); the kernels accumulate sum e V with the
  exact fp16 e and divide once at the end -- and, with several context ranges [256 r, 256 r + 256), merge per-range
  {max, sum e, sum e V} with exp(max_r - max) weights.  attend_stated restates that; this bounds what it costs."""
import numpy as np
import pytest

from oracle import llama_model as lm


@pytest.mark.parametrize("hd", [32, 64, 80, 128])
@pytest.mark.parametrize("theta,scale", [(10000.0, 1.0), (500000.0, 1.0), (10000.0, 0.25), (500000.0, 4.0)])
def test_vectorised_rope_is_bit_identical_to_rope_mode0(hd, theta, scale):
    r = np.random.default_rng(hd)
    pos = np.array([0, 1, 2, 63, 255, 256, 1000, 2047, 4095, 8190, 8191, 8191])
    x = r.normal(0, 1, (pos.size, 3, hd)).astype(np.float32)
    x[0, 0, :4] = [0.0, -0.0, 1e-30, -3e4]
    got = lm.rope_mode0_rows(x, pos, hd, theta, scale)
    want = np.stack([lm.rope_mode0(x[t], int(p), hd, theta, scale) for t, p in enumerate(pos)])
    assert got.view(np.uint32).tolist() == want.view(np.uint32).tolist()


def test_fmaf_is_correctly_rounded():
    r = np.random.default_rng(5)
    a, b = r.normal(0, 1, 4000).astype(np.float32), r.normal(0, 1, 4000).astype(np.float32)
    c = -(a * b)  # heavy cancellation: the exact residual of the product decides the result
    c[::2] = r.normal(0, 1, 2000).astype(np.float32)
    want = np.array([lm._libm.fmaf(float(x), float(y), float(z)) for x, y, z in zip(a, b, c)], np.float32)
    assert np.array_equal(lm._fmaf(a, b, c), want)


@pytest.mark.parametrize("n_head,n_head_kv,hd,n_past,m", [(4, 4, 64, 0, 1), (4, 2, 128, 37, 1), (2, 1, 64, 5, 6), (3, 3, 96, 20, 4),
                                                         (8, 2, 32, 300, 3)])
def test_vectorised_attention_matches_the_per_row_oracle(n_head, n_head_kv, hd, n_past, m):
    """attention_reference == OracleLlama.eval's loop (vec_dot_f16_rows -> soft_max_f16table -> vec_dot_f16_rows, pinned to the
    reference's engine) up to the fp32 summation order of the two dot products"""
    r = np.random.default_rng(n_past + m)
    L = n_past + m
    q = r.normal(0, 1.5, (m, n_head, hd)).astype(np.float32)
    kc = r.normal(0, 1, (n_head_kv, L + 3, hd)).astype(np.float16)
    vc = r.normal(0, 1, (n_head_kv, L + 3, hd)).astype(np.float16)
    got = lm.attention_reference(q, kc, vc, n_past)
    scale = np.float32(1.0) / np.float32(np.sqrt(np.float32(hd)))
    worst = 0.0
    for t in range(m):
        for h in range(n_head):
            hk = h // (n_head // n_head_kv)
            ln = n_past + t + 1
            s = lm.vec_dot_f16_rows(kc[hk, :ln].astype(np.float32), lm._f16(q[t, h])) * scale
            p = lm.soft_max_f16table(s)
            want = lm.vec_dot_f16_rows(np.ascontiguousarray(vc[hk, :ln].astype(np.float32).T), lm._f16(p))
            worst = max(worst, float(np.abs(got[t, h] - want).max()))
    # fp32 reordering only: measured 9e-8 (|out| ~ 1), a few ulp; no fp16 rounding of a score or a p flips on these inputs
    assert worst <= 1e-6, worst


def test_normalising_after_the_v_product_stays_within_1e3_of_the_reference_order():
    rng = np.random.default_rng(0)
    worst = 0.0
    for length, hd, kind in ((40, 64, "mma"), (300, 128, "mma"), (256, 128, "split"), (300, 128, "split"), (2100, 128, "split"),
                             (8192, 64, "split")):
        for _ in range(4):
            s = rng.normal(0, 2.0, (1, length)).astype(np.float32)
            v = lm._f16(rng.normal(0, 1.0, (length, hd)))
            a, b = lm.attend_reference(s, v), lm.attend_stated(s, v, kind)
            if kind == "split" and length <= lm.SPLIT_KEYS:
                assert np.array_equal(a, b)  # one range: the reference order exactly
            worst = max(worst, float(np.abs(a - b).max() / np.abs(a).max()))
    assert worst <= 1e-3, worst


def test_split_ranges_are_the_kernels_256_aligned_ranges():
    """a score spike in range 1 only: the merge must weight range 0 by exp(max_0 - max_1), with the boundary at 256"""
    s = np.zeros((1, 300), np.float32)
    s[0, 256] = 8.0
    v = np.zeros((300, 2), np.float32)
    v[:256, 0] = 1.0
    v[256:, 1] = 1.0
    got = lm.attend_stated(s, v, "split")[0]
    e_small = float(lm._f16(np.exp(np.float32(-8.0))))  # range 1 away from the spike: fp16(exp(fp16(-8)))
    w0 = float(np.exp(np.float32(-8.0)))               # range 0 (max 0) against the global max 8
    num0, num1 = w0 * 256.0, 1.0 + 43 * e_small
    assert np.allclose(got, [num0 / (num0 + num1), num1 / (num0 + num1)], rtol=1e-6)

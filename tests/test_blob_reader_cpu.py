"""Every host entry that reads a serialized BesTLA blob refuses one whose header disagrees with its buffers, and writes
nothing: BTLAGemmUnPackB, bestla_packweight_copyattr, ns_split_weight_size / ns_split_weight and ns_device_storage_bytes all
go through the one bounds-checked reader.  Each corruption below stays inside the blob's own size field, so a reader that
honours that field never leaves the test's memory."""
import ctypes as C
import functools
import struct

import numpy as np
import pytest

import neural_speed_b200 as ns

N, K, G = 100, 256, 64  # N not a multiple of NTile=48: NPad > N
INT_DTYPES = ["int2", "int3", "int4", "int5", "int6", "int7", "int8"]
FLOAT_DTYPES = ["nf4", "fp4_bnb", "fp4_e2m1"]
COMPS = ["int8", "bf16", "fp16", "fp32"]


def _configs(dtype):
    """(scale dtype, asym, compute dtype, shuffle) of every blob the packers write for this weight dtype"""
    if dtype in FLOAT_DTYPES:
        return [(s, False, c, False) for s in ("fp32", "bf16", "fp16") for c in COMPS]
    plain = [(s, a, c, False) for s in ("fp32", "bf16", "fp16") for a in (False, True) for c in COMPS]
    return plain + [(s, a, c, True) for s in ("fp32", "bf16") for a in (False, True) for c in COMPS]  # qpack: fp32 / bf16 scales


@functools.lru_cache(maxsize=None)
def _blob(dtype, sdt, asym, cdt, shuffle):
    rng = np.random.default_rng(7)
    alg = "asym" if asym else "sym"
    if not shuffle:
        b = ns.np_bestla_quantize(rng.normal(0, 0.05, (N, K)).astype(np.float32), dtype, G, alg, sdt, cdt)
    else:
        full = 1 << (int(dtype[3:]) - 1)
        q = rng.integers(-full, full, (K, N)).astype(np.int8)
        sc = rng.uniform(0.01, 0.02, (K // G, N)).astype(np.float32)
        zp = rng.integers(-full, full, (K // G, N)).astype(np.int8)
        g_idx = rng.permutation(np.repeat(np.arange(K // G), G)).astype(np.int32)
        b = ns.np_bestla_qpack(q, sc, zp, g_idx, dtype, G, alg, sdt, cdt)
    return bytes(b)


def _layout(b):
    """byte offsets of the fields the corruptions touch (bestla_storage.h:98-146, :151-248, :250-357)"""
    (qsz, qoff) = struct.unpack_from("<QQ", b, 48)
    at = 64 + qoff + qsz                       # scaT zpT redT CStep CSize, then the scale buffer
    (ssz, soff) = struct.unpack_from("<QQ", b, at + 24)
    zflag = at + 40 + soff + ssz
    return dict(size=struct.unpack_from("<Q", b, 0)[0], q=48, scale=at + 24, zp=zflag + 1 if b[zflag] else None)


def _set(b, fmt, off, value):
    struct.pack_into(fmt, b, off, value)


def _shorten(b, at):
    """the buffer whose (size, offset) pair sits at `at` starts 64 bytes later and ends where it did: the rest of the blob
    still parses, but the buffer is shorter than the header implies"""
    sz, off = struct.unpack_from("<QQ", b, at)
    struct.pack_into("<QQ", b, at, sz - 64, off + 64)


def _corrupt(blob, how):
    b = bytearray(blob)
    L = _layout(b)
    npad = struct.unpack_from("<i", b, 20)[0]
    if how == "prologue":
        _set(b, "<I", 8, 3)
    elif how in ("q.size", "q.offset", "scale.size", "scale.offset"):
        buf, field = how.split(".")
        _set(b, "<Q", L[buf] + (0 if field == "size" else 8), L["size"])
    elif how == "scale.short":
        _shorten(b, L["scale"])
    elif how == "zp.short":
        _shorten(b, L["zp"])
    elif how == "packrow3":
        b[13] = 3
    elif how == "ntile":
        b[12] += 1
        assert npad % b[12] != 0
    elif how == "n_past_npad":
        _set(b, "<i", 28, npad + 1)
    assert struct.unpack_from("<Q", b, 0)[0] == len(blob)
    return b


CORRUPTIONS = ["prologue", "q.size", "q.offset", "scale.size", "scale.offset", "scale.short", "zp.short", "packrow3", "ntile",
               "n_past_npad"]


def _cases():
    for how in CORRUPTIONS:
        for dtype in INT_DTYPES + FLOAT_DTYPES:
            if how != "zp.short" or dtype in INT_DTYPES:
                yield how, dtype


def _buf(data):
    """64-byte aligned uint8 copy of `data` (the packers align their buffers the same way)"""
    raw = np.zeros(len(data) + 64, np.uint8)
    a = raw[(-raw.ctypes.data) % 64:][:len(data)]
    a[:] = np.frombuffer(bytes(data), np.uint8)
    return a


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.mark.parametrize("how,dtype", list(_cases()))
def test_every_host_reader_refuses_an_inconsistent_blob(how, dtype):
    L = ns.lib()
    w_kn = np.random.default_rng(1).uniform(-0.5, 0.5, (K, N)).astype(np.float32)
    for sdt, asym, cdt, shuffle in _configs(dtype):
        if how == "zp.short" and not asym:
            continue
        cfg = (dtype, sdt, asym, cdt, shuffle)
        good = _buf(_blob(*cfg))
        # the intact blob is read by every entry
        assert L.BTLAGemmUnPackB(_p(np.empty((K, N), np.float32)), _p(good), N, K, N, None), cfg
        assert L.ns_split_weight_size(_p(good), N // 2, K) > 0, cfg
        assert L.ns_device_storage_bytes(_p(good)) > 0, cfg

        bad = _buf(_corrupt(_blob(*cfg), how))
        n, k = struct.unpack_from("<ii", bytes(bad[28:36]))
        out = np.full((k, n), 7.0, np.float32)
        assert not L.BTLAGemmUnPackB(_p(out), _p(bad), n, k, n, None), cfg
        assert np.all(out == 7.0), cfg
        dst = np.full(2 * good.size + 4096, 0xAB, np.uint8)
        L.bestla_packweight_copyattr(_p(w_kn), _p(dst), N, K, N, _p(bad))
        assert np.all(dst == 0xAB), cfg
        assert L.ns_split_weight_size(_p(bad), n // 2, k) == 0, cfg
        assert not L.ns_split_weight(_p(bad), _p(dst), n, k, n // 2, k, 1, 0, False), cfg
        assert np.all(dst == 0xAB), cfg
        assert L.ns_device_storage_bytes(_p(bad)) == 0, cfg

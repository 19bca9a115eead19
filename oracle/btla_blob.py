"""Oracle restatement (numpy) of the serialized BesTLA weight blob -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.

Follows /root/reference/bestla/bestla:
  bestla_storage.h:60-147   ObjectAlignedBuffer / ObjectOptionalBuffer (size, offset-to-64B, pad, data; bool flag)
  bestla_storage.h:151-248  ObjectQuantCorrection (scaT, zpT, redT, CStep, CSize, scale/zp/reduce/dq buffers)
  bestla_storage.h:250-357  IWeightBase / IWeightKBlockBase header fields
  bestla_storage.h:697-834  StorageWeightKBlockNInteger (QBuf, correction, shuffle indices; size padded to 64)
  bestla_prologue_b.h:490-510 + kernel_ref.h:40-58   reorderWeight = padding_interleave(NTile, PackRow)
  kernel_ref.h:155-165      compress_s8_s4 (nibble = q + 8, element 2i low)
  bestla_prologue_b.h:455-470 + kernel_ref.h:2132-2141  reduceWeight / row_reduce_sum
  bestla_prologue_b.h:337-356  setShuffleIndices
  bestla_gemm.h:83-125      CoreAttr id encoding
  bestla_storage.h:724-745 + bestla_prologue_b.h:512-564 + kernel_ref.h:178-345   2/3/5/6/7-bit codes as bit planes
"""
from __future__ import annotations

import struct

import numpy as np

from . import f32_to_bf16_bits, bf16_bits_to_f32

S4_CLIP = 4 | (1 << 8)
S8 = 8 | (1 << 8)
F4_NF4 = 4 | (2 << 16)
F32 = 32
BF16 = 16 | (1 << 16)
F16 = 16

# (NTile, PackRow, KTile, CompType, ISA) of the cores neural_speed can emit (bestla_defs.h:36-54)
CORES = {
    "avx512_vnni_kblock": (48, 4, 4, 4 | (3 << 4), 6),
    "amx_int8_kblock": (48, 4, 64, 4 | (3 << 4), 10),
    "avx2_vnni_kblock": (24, 4, 4, 4 | (3 << 4), 2),
    "amx_bf16": (48, 2, 32, 1 | (1 << 4), 9),
    "amx_fp16": (48, 2, 32, 2 | (2 << 4), 11),
    "avx512f": (48, 1, 1, 0, 4),
    "avx2": (24, 1, 1, 0, 2),
}


def core_id(ntile, packrow, comp, isa):
    return ntile | (packrow << 8) | (comp << 16) | (isa << 32)


def interleave(q_kn: np.ndarray, ntile: int, packrow: int, kpad: int, npad: int) -> np.ndarray:
    """[K,N] int8 -> flat [N/NTile][KPad/PackRow][NTile][PackRow] with zero padding."""
    k, n = q_kn.shape
    p = np.zeros((kpad, npad), np.int8)
    p[:k, :n] = q_kn
    t = p.reshape(kpad // packrow, packrow, npad // ntile, ntile)  # [kb, ii, nb, jj]
    return np.ascontiguousarray(t.transpose(2, 0, 3, 1)).reshape(-1)  # [nb, kb, jj, ii]


def compress_s4(flat: np.ndarray, bias: int = 8) -> np.ndarray:
    u = ((flat.astype(np.int16) + bias) & 0xF).astype(np.uint8)
    return (u[0::2] | (u[1::2] << 4)).astype(np.uint8)


# plane widths per code width, low bits first (compress_{2,3,5,6,7}bit)
PLANES = {2: (2,), 3: (2, 1), 5: (4, 1), 6: (4, 2), 7: (4, 2, 1)}


def compress_planes(flat: np.ndarray, bits: int) -> np.ndarray:
    """flat int8 [E] (values q) -> the plane bytes: u = q + 2^(bits-1); plane i holds its slice of u for every element, element e at
    bit (e % (8/w)) * w of byte e // (8/w); planes laid one after the other (4-bit, 2-bit, 1-bit)."""
    u = (flat.astype(np.int16) + (1 << (bits - 1))).astype(np.uint8)
    out, sh = [], 0
    for w in PLANES[bits]:
        per = 8 // w
        part = ((u >> sh) & ((1 << w) - 1)).reshape(-1, per)
        byte = np.zeros(part.shape[0], np.uint8)
        for j in range(per):
            byte |= (part[:, j] << (j * w)).astype(np.uint8)
        out.append(byte)
        sh += w
    return np.concatenate(out)


def decompress_planes(raw: np.ndarray, bits: int, elt: int) -> np.ndarray:
    """inverse of compress_planes: int32 [elt] values q."""
    u = np.zeros(elt, np.int32)
    at, sh = 0, 0
    for w in PLANES[bits]:
        per = 8 // w
        nbytes = (elt * w + 7) // 8
        plane = raw[at:at + nbytes].astype(np.int32)
        e = np.arange(elt)
        u |= ((plane[e // per] >> ((e % per) * w)) & ((1 << w) - 1)) << sh
        at += nbytes
        sh += w
    return u - (1 << (bits - 1))


def _aligned(buf: bytearray, base_addr: int, data: bytes) -> None:
    buf += struct.pack("<Q", len(data))
    after = base_addr + len(buf) + 8
    off = (-after) % 64
    buf += struct.pack("<Q", off)
    buf += b"\0" * off
    buf += data


def _optional(buf: bytearray, base_addr: int, data) -> None:
    if data is None:
        buf += b"\0"
    else:
        buf += b"\1"
        _aligned(buf, base_addr, data)


def _scale_bytes(sc_pad: np.ndarray, stype: int) -> bytes:
    if stype == F32:
        return sc_pad.astype(np.float32).tobytes()
    if stype == BF16:
        return f32_to_bf16_bits(sc_pad).tobytes()
    return sc_pad.astype(np.float16).tobytes()


def serialize(q_kn, scales, zps, group, core="avx512_vnni_kblock", qtype=S4_CLIP, stype=F32, g_idx=None, base_addr=0) -> bytes:
    """Build the byte image StorageWeightKBlockNInteger/NFloat::serialize would write at address base_addr."""
    ntile, packrow, ktile, comp, isa = CORES[core]
    q_kn = np.asarray(q_kn, np.int8)
    k, n = q_kn.shape
    npad = -(-n // ntile) * ntile
    kpad = -(-k // ktile) * ktile
    is_float = qtype == F4_NF4
    is_int_core = (comp >> 4) & 0xF in (3, 4)
    nk = -(-kpad // group)
    raw_nb = -(-k // group)
    flat = interleave(q_kn, ntile, packrow, kpad, npad)
    qbytes = flat.view(np.uint8).tobytes() if qtype == S8 else compress_s4(flat, 0 if is_float else 8).tobytes()
    sc_pad = np.zeros((nk, npad), np.float32)
    sc_pad[:raw_nb, :n] = scales
    sbytes = _scale_bytes(sc_pad, stype)
    zbytes = None
    if zps is not None:
        zp_pad = np.zeros((nk, npad), np.int8)
        zp_pad[:raw_nb, :n] = zps
        zbytes = zp_pad.tobytes()
    rbytes = None
    if is_int_core and not is_float:
        if stype == BF16:
            s_eff = bf16_bits_to_f32(f32_to_bf16_bits(np.asarray(scales, np.float32)))
        elif stype == F16:
            s_eff = np.asarray(scales, np.float32).astype(np.float16).astype(np.float32)
        else:
            s_eff = np.asarray(scales, np.float32)
        red = np.zeros((nk, npad), np.float32)
        for b in range(raw_nb):
            acc = np.zeros(n, np.float32)
            for kk in range(b * group, min(k, (b + 1) * group)):
                z = zps[b].astype(np.float32) if zps is not None else np.float32(0)
                acc = (acc + (q_kn[kk].astype(np.float32) - z) * s_eff[b]).astype(np.float32)
            red[b, :n] = acc
        rbytes = f32_to_bf16_bits(red).tobytes()
    shbytes = None
    if g_idx is not None and not is_float:
        sh = np.zeros(k, np.int32)
        cnt = np.zeros(raw_nb, np.int64)
        for i, g in enumerate(np.asarray(g_idx)):
            sh[g * group + cnt[g]] = i
            cnt[g] += 1
        shbytes = sh.tobytes()

    buf = bytearray()
    buf += struct.pack("<Q", 0)  # mSize placeholder
    buf += struct.pack("<I", 2 if is_float else 1)
    buf += struct.pack("<Q", core_id(ntile, packrow, comp, isa))
    buf += struct.pack("<iiii", npad, kpad, n, k)
    buf += struct.pack("<I", qtype)
    buf += struct.pack("<ii", group, 0)
    _aligned(buf, base_addr, qbytes)
    buf += struct.pack("<III", stype, 0 if is_float else S8, 0 if is_float else BF16)
    buf += struct.pack("<i", npad)
    buf += struct.pack("<Q", nk * npad)
    _aligned(buf, base_addr, sbytes)
    _optional(buf, base_addr, zbytes)
    _optional(buf, base_addr, rbytes)
    _optional(buf, base_addr, None)
    _optional(buf, base_addr, shbytes)

    def ser_size(nbytes):
        return 16 + nbytes + 64

    total = 8 + 4 + 8 + 16 + 4 + 8 + ser_size(len(qbytes)) + (12 + 4 + 8) + ser_size(len(sbytes))
    total += 1 + (ser_size(len(zbytes)) if zbytes is not None else 0)
    total += 1 + (ser_size(len(rbytes)) if rbytes is not None else 0)
    total += 1
    if not is_float:
        total += 1 + (ser_size(len(shbytes)) if shbytes is not None else 0)
    total = -(-total // 64) * 64
    assert len(buf) <= total, (len(buf), total)
    buf += b"\0" * (total - len(buf))
    buf[0:8] = struct.pack("<Q", total)
    return bytes(buf)


def parse(blob) -> dict:
    """PackedWeightParser::deserialBuffer equivalent: returns header fields and numpy views of the buffers."""
    b = bytes(blob)
    size, prologue = struct.unpack_from("<QI", b, 0)
    (cid,) = struct.unpack_from("<Q", b, 12)
    npad, kpad, n, k = struct.unpack_from("<iiii", b, 20)
    (dtype,) = struct.unpack_from("<I", b, 36)
    blk, dq = struct.unpack_from("<ii", b, 40)
    pos = 48

    def aligned():
        nonlocal pos
        sz, off = struct.unpack_from("<QQ", b, pos)
        pos += 16 + off
        data = b[pos:pos + sz]
        pos += sz
        return data

    def optional():
        nonlocal pos
        flag = b[pos]
        pos += 1
        return aligned() if flag else None

    qbuf = aligned()
    sca_t, zp_t, red_t = struct.unpack_from("<III", b, pos)
    pos += 12
    (cstep,) = struct.unpack_from("<i", b, pos)
    pos += 4
    (csize,) = struct.unpack_from("<Q", b, pos)
    pos += 8
    sbuf = aligned()
    zbuf = optional()
    rbuf = optional()
    dqbuf = optional()
    shbuf = optional()
    return dict(size=size, prologue=prologue, core_id=cid, ntile=cid & 0xFF, packrow=(cid >> 8) & 0xFF,
                comp=(cid >> 16) & 0xFFFF, isa=(cid >> 32) & 0xFF, npad=npad, kpad=kpad, n=n, k=k, dtype=dtype, blocksize=blk,
                dqblocksize=dq, qbuf=qbuf, sca_t=sca_t, zp_t=zp_t, red_t=red_t, cstep=cstep, csize=csize, scale=sbuf, zp=zbuf,
                red=rbuf, dq=dqbuf, shuffle=shbuf)


def codes(blob) -> dict:
    """The stored operands of a blob: q int32 [K,N] (signed integer codes, or the 0..15 codebook codes of a float blob), scale
    fp32 [ceil(K/blk),N] as stored (bf16 / fp16 widened), zp int32 [..] or None, blk, prologue (2: float codebook)."""
    h = parse(blob)
    n, k, npad, kpad, nt, pr, blk = h["n"], h["k"], h["npad"], h["kpad"], h["ntile"], h["packrow"], h["blocksize"]
    raw = np.frombuffer(h["qbuf"], np.uint8)
    if (h["dtype"] & 0xFF) == 8:
        flat = raw.view(np.int8).astype(np.int32)
    elif (h["dtype"] & 0xFF) in PLANES and h["prologue"] == 1:
        flat = decompress_planes(raw, h["dtype"] & 0xFF, npad * kpad)
    else:
        flat = np.empty(raw.size * 2, np.int32)
        flat[0::2] = raw & 0xF
        flat[1::2] = raw >> 4
        if h["prologue"] == 1:
            flat -= 8
    t = flat.reshape(npad // nt, kpad // pr, nt, pr).transpose(1, 3, 0, 2).reshape(kpad, npad)[:k, :n]
    nk = -(-kpad // blk)
    if h["sca_t"] == F32:
        sc = np.frombuffer(h["scale"], np.float32)
    elif h["sca_t"] == BF16:
        sc = bf16_bits_to_f32(np.frombuffer(h["scale"], np.uint16))
    else:
        sc = np.frombuffer(h["scale"], np.float16).astype(np.float32)
    raw_nb = -(-k // blk)
    sc = sc.reshape(nk, h["cstep"])[:raw_nb, :n]
    zp = None
    if h["zp"] is not None:
        zp = np.frombuffer(h["zp"], np.int8).reshape(nk, h["cstep"])[:raw_nb, :n].astype(np.int32)
    return dict(q=np.ascontiguousarray(t), scale=np.ascontiguousarray(sc), zp=zp, blk=blk, prologue=h["prologue"])


def unpack(blob) -> np.ndarray:
    """Dequantise a blob to fp32 [K,N] (unpackWeight semantics)."""
    c = codes(blob)
    t, sc, blk = c["q"], c["scale"], c["blk"]
    gi = np.arange(t.shape[0]) // blk
    if c["prologue"] == 2:
        from . import lib
        lut = np.array([lib().orc_nf4_unpack(c) for c in range(16)], np.float32)
        return (lut[t] * sc[gi]).astype(np.float32)
    if c["zp"] is not None:
        t = t - c["zp"][gi]
    return (t.astype(np.float32) * sc[gi]).astype(np.float32)

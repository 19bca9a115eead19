// btla_blob.h -- the serialized BesTLA weight blob (StorageWeightKBlockNInteger / NFloat, bestla/bestla/bestla_storage.h:697-860),
// host code only.  pack.cpp writes it and owns its one reader: every caller takes the blob's fields from a BlobView that
// parse_blob has checked, so a blob read from a file is bounds-checked the same way on every path.
#pragma once
#include <cstddef>
#include <cstdint>

// codes that are not 4 or 8 bits wide are stored as a sum of power-of-two bit planes (bestla_storage.h:724-745)
struct BlobPlanes {
  int n;  // 0: the codes are nibbles (4 bits) or bytes (8 bits)
  int width[3];
  size_t off[3];  // byte offset of each plane in the q buffer
  size_t bytes;   // total
};

struct BlobView {
  size_t size;
  uint32_t prologue;
  uint64_t core_id;
  int npad, kpad, n, k;
  uint32_t dtype;
  int blocksize, dqblocksize;
  const uint8_t* qbuf;
  size_t qbytes;
  uint32_t sca_t, zp_t, red_t;
  int cstep;
  size_t csize;
  const uint8_t* scale;
  size_t scale_bytes;
  const uint8_t* zp;
  size_t zp_bytes;
  const uint8_t* red;
  size_t red_bytes;
  const uint8_t* dq;
  size_t dq_bytes;
  const int* shuffle;
  size_t shuffle_bytes;
  // derived
  int ntile, packrow, comp_b, comp_a;
  int ne_comp;  // the NS_NE_COMP_* that re-quantising with this blob's attributes asks for (bestla_packweight_copyattr)
  int bits;     // code width
  BlobPlanes planes;
};

// The blob's own size field, or 0 when it is implausible (under 64 bytes or over 1 TiB).
size_t blob_size(const void* blob);

// avail: bytes readable at `blob` (0: unknown -- trust the blob's own size field, as the reference's deserialBuffer does).
// Returns false, with ns_last_error() saying why, unless the header is consistent and every buffer lies inside the size field
// and is as large as the header implies; then every element and correction index of the n x k weight is in bounds.
bool parse_blob(const void* blob, BlobView* v, size_t avail = 0);

// Code of tile-order element e (0 <= e < npad * kpad) of a parsed blob: the 0..15 codebook index of a 4-bit float (NFloat)
// blob, else the signed integer the codes store.
int blob_code(const BlobView& v, size_t e);

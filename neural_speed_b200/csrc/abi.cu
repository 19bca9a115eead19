// abi.cu -- the C-ABI of libns_b200.so (see include/ns_b200.h): device context, weight handles, blob upload,
// host-buffer drop-ins for neural_speed/core/ne_bestla.h and the device set modelled on its NS_SYCL block.
// There is NO CPU compute path in this file: without a usable CUDA device every compute entry point fails loudly.
#include <atomic>
#include <cstdarg>
#include <cstring>
#include <mutex>
#include <unordered_map>
#include <vector>

#include "nsb.cuh"
#include "btla_blob.h"

// ---------------------------------------------------------------------------------------------------- errors / context
static thread_local char g_err[512] = "";
static std::atomic<unsigned long long> g_launches{0};

void ns_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}
[[noreturn]] void ns_fatal(const char* fmt, ...) {
  // the reference prints and assert(0)s on bad input (core/layers/inner_product.cpp:31-35)
  va_list ap;
  va_start(ap, fmt);
  fprintf(stderr, "Err: ");
  vfprintf(stderr, fmt, ap);
  fprintf(stderr, "\n");
  va_end(ap);
  abort();
}
bool ns_cuda_ok(cudaError_t e, const char* what) {
  if (e == cudaSuccess) return true;
  ns_set_error("CUDA error %s: %s (%s)", cudaGetErrorName(e), cudaGetErrorString(e), what);
  return false;
}
void ns_count_launch(int n) { g_launches.fetch_add((unsigned long long)n, std::memory_order_relaxed); }

extern "C" const char* ns_last_error(void) { return g_err; }
extern "C" const char* ns_version(void) { return "ns_b200 0.1 (sm_90a)"; }
extern "C" unsigned long long ns_launch_count(void) { return g_launches.load(); }

struct ns_device {
  int dev;
  cudaStream_t stream;
  bool profile;
};

static std::mutex g_mu;
static int g_dev_state = 0;  // 0 unknown, 1 ok, -1 none
static ns_device g_default = {0, nullptr, false};
// library-owned scratch per stream
struct Scratch {
  void* p = nullptr;
  size_t bytes = 0;
};
static std::unordered_map<cudaStream_t, Scratch> g_scratch;

int ns_ensure_device() {
  if (g_dev_state == 1) return NS_OK;
  std::lock_guard<std::mutex> lk(g_mu);
  if (g_dev_state == 1) return NS_OK;
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    ns_set_error("no CUDA device available (%s); libns_b200 has no CPU fallback", cudaGetErrorString(e));
    cudaGetLastError();
    g_dev_state = -1;
    return NS_E_NODEVICE;
  }
  int dev = 0;
  cudaGetDevice(&dev);
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, dev) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
    ns_set_error("device %d is sm_%d%d; this library carries sm_90a code only", dev, prop.major, prop.minor);
    g_dev_state = -1;
    return NS_E_NODEVICE;
  }
  g_default.dev = dev;
  if (cudaStreamCreateWithFlags(&g_default.stream, cudaStreamNonBlocking) != cudaSuccess) {
    ns_set_error("cudaStreamCreate failed");
    g_dev_state = -1;
    return NS_E_CUDA;
  }
  g_dev_state = 1;
  return NS_OK;
}

int ns_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    if (sms <= 0) sms = 132;
  }
  return sms;
}

static cudaStream_t default_stream() { return g_default.stream; }
static cudaStream_t stream_of(void* queue) { return queue ? (cudaStream_t)queue : default_stream(); }
cudaStream_t ns_stream_of(void* queue) { return stream_of(queue); }

static void* scratch_get(cudaStream_t st, size_t bytes) {
  std::lock_guard<std::mutex> lk(g_mu);
  Scratch& s = g_scratch[st];
  if (s.bytes < bytes) {
    if (s.p) {
      cudaStreamSynchronize(st);
      cudaFree(s.p);
    }
    size_t nb = ns_round_up(bytes + bytes / 4, 1 << 20);
    if (cudaMalloc(&s.p, nb) != cudaSuccess) {
      s.p = nullptr;
      s.bytes = 0;
      ns_set_error("cudaMalloc(%zu) for scratch failed", nb);
      return nullptr;
    }
    s.bytes = nb;
  }
  return s.p;
}

// ---------------------------------------------------------------------------------------------------- weight handles
static size_t stype_size(int stype) { return (size_t)ns_stype_size(stype); }
static void weight_layout(ns_weight* w) { ns_weight_layout(w); }
static size_t weight_image_bytes(const ns_weight* w, bool with_shuffle) {
  size_t b = ns_round_up((size_t)w->n * w->pitch, 256);
  if (with_shuffle) b += ns_round_up((size_t)w->k * 4, 256);
  return b;
}
static void weight_carve(ns_weight* w, void* base, bool with_shuffle) {
  char* p = (char*)base;
  w->rows = (uint8_t*)p;
  p += ns_round_up((size_t)w->n * w->pitch, 256);
  w->shuffle = with_shuffle ? (int*)p : nullptr;
}
// st: the stream the weight is then filled on.  The clearing is ordered before the fill on that stream: a plain cudaMemset runs on
// the legacy default stream, which the library's non-blocking streams do not wait for, and could land after (or during) the repack.
static int weight_alloc(ns_weight* w, bool with_shuffle, cudaStream_t st) {
  w->total_bytes = weight_image_bytes(w, with_shuffle);
  NS_CUDA_TRY(cudaMalloc(&w->base, w->total_bytes));
  // padding bytes of each row are streamed by the GEMV too: keep them defined
  NS_CUDA_TRY(cudaMemsetAsync(w->base, 0, w->total_bytes, st));
  w->external = 0;
  weight_carve(w, w->base, with_shuffle);
  return NS_OK;
}

extern "C" void ns_weight_free(ns_weight* w) {
  if (!w) return;
  if (w->base && !w->external) cudaFree(w->base);
  delete w;
}

extern "C" int ns_weight_info(const ns_weight* w, int* n, int* k, int* group, int* wfmt, int* stype, int* comp, int* asym) {
  if (!w) return NS_E_INVALID;
  if (n) *n = w->n;
  if (k) *k = w->k;
  if (group) *group = w->group;
  if (wfmt) *wfmt = w->wfmt;
  if (stype) *stype = w->stype;
  if (comp) *comp = w->comp;
  if (asym) *asym = w->asym;
  return NS_OK;
}
extern "C" int ns_weight_set_comp(ns_weight* w, int comp) {
  if (!w || comp < 0 || comp > NS_COMP_INT8_S8) return NS_E_INVALID;
  if (w->wfmt == NS_W_NF4 && !(comp == NS_COMP_F32 || comp == NS_COMP_BF16)) {
    ns_set_error("NF4 weights support float compute only (docs/advanced_usage.md:82-83)");
    return NS_E_UNSUPPORTED;
  }
  if (w->wfmt == NS_W_Q8_0 && comp != NS_COMP_Q8_0) {
    ns_set_error("ggml Q8_0 weights have the fixed compute type NS_COMP_Q8_0");
    return NS_E_UNSUPPORTED;
  }
  w->comp = comp;
  return NS_OK;
}
extern "C" size_t ns_weight_algorithmic_bytes(const ns_weight* w) {
  if (w->wfmt == NS_W_Q6K) return (size_t)w->n * (w->k / 256) * 210;  // block_q6_K bytes
  // SURVEY.md 8(d): N*K*bits/8 + N*ceil(K/g)*(scale_bytes [+1 if asym])
  const size_t bits = (w->wfmt == NS_W_S8 || w->wfmt == NS_W_Q8_0) ? 8 : 4;  // Q8_0: N*K + N*K/32*2, block_q8_0's bytes
  return (size_t)w->n * w->k * bits / 8 + (size_t)w->n * w->ngroups * (stype_size(w->stype) + (w->asym ? 1 : 0));
}

// ggml rows of 32-element blocks (block_q4_0: 18 bytes, block_q8_0: 34 bytes) -> NSB rows, repacked on the device
static ns_weight* weight_from_ggml32(bool q8, const void* rows, int n, int k, size_t nb01, int rows_on_device, void* queue) {
  const char* who = q8 ? "ns_weight_from_q8_0" : "ns_weight_from_q4_0";
  if (ns_ensure_device()) return nullptr;
  if (!rows || n <= 0 || k <= 0 || k % 32 != 0 || nb01 < (size_t)k / 32 * (q8 ? 34 : 18)) {
    ns_set_error("%s: invalid arguments (n=%d k=%d nb01=%zu)", who, n, k, nb01);
    return nullptr;
  }
  // the repack kernels read blocks as 16-bit words (fp16 d, then the codes): rows must start on even addresses
  if (nb01 % 2 != 0 || (rows_on_device && ((uintptr_t)rows & 1))) {
    ns_set_error("%s: rows must be 2-byte aligned (nb01=%zu, rows=%p)", who, nb01, rows);
    return nullptr;
  }
  cudaStream_t st = stream_of(queue);
  ns_weight* w = new ns_weight();
  memset(w, 0, sizeof(*w));
  w->n = n;
  w->k = k;
  w->group = 32;
  w->wfmt = q8 ? NS_W_Q8_0 : NS_W_S4;
  w->stype = NS_S_F16;
  w->comp = NS_COMP_Q8_0;
  w->asym = 0;
  weight_layout(w);
  if (weight_alloc(w, false, st)) {
    delete w;
    return nullptr;
  }
  const void* src = rows;
  void* tmp = nullptr;
  if (!rows_on_device) {
    const size_t bytes = (size_t)n * nb01;
    if (!ns_cuda_ok(cudaMalloc(&tmp, bytes), q8 ? "cudaMalloc(q8_0 staging)" : "cudaMalloc(q4_0 staging)") ||
        !ns_cuda_ok(cudaMemcpyAsync(tmp, rows, bytes, cudaMemcpyHostToDevice, st), q8 ? "H2D q8_0 rows" : "H2D q4_0 rows")) {
      if (tmp) cudaFree(tmp);
      ns_weight_free(w);
      return nullptr;
    }
    src = tmp;
  }
  int rc = q8 ? ns_launch_repack_q8_0(src, nb01, w, st) : ns_launch_repack_q4_0(src, nb01, w, st);
  if (tmp) {
    cudaStreamSynchronize(st);
    cudaFree(tmp);
  }
  if (rc) {
    ns_weight_free(w);
    return nullptr;
  }
  return w;
}
extern "C" ns_weight* ns_weight_from_q4_0(const void* rows, int n, int k, size_t nb01, int rows_on_device, void* queue) {
  return weight_from_ggml32(false, rows, n, k, nb01, rows_on_device, queue);
}
extern "C" ns_weight* ns_weight_from_q8_0(const void* rows, int n, int k, size_t nb01, int rows_on_device, void* queue) {
  return weight_from_ggml32(true, rows, n, k, nb01, rows_on_device, queue);
}

extern "C" ns_weight* ns_weight_from_q6_K(const void* rows, int n, int k, size_t nb01, int rows_on_device, void* queue) {
  if (ns_ensure_device()) return nullptr;
  if (!rows || n <= 0 || k <= 0 || k % 256 != 0 || nb01 < (size_t)k / 256 * 210) {
    ns_set_error("ns_weight_from_q6_K: invalid arguments (n=%d k=%d nb01=%zu)", n, k, nb01);
    return nullptr;
  }
  cudaStream_t st = stream_of(queue);
  ns_weight* w = new ns_weight();
  memset(w, 0, sizeof(*w));
  w->n = n;
  w->k = k;
  w->wfmt = NS_W_Q6K;
  w->stype = NS_S_F32;
  w->comp = NS_COMP_Q8_0;  // ggml integer path (Q8_K activations)
  w->asym = 0;
  ns_q6k_layout(w);
  if (weight_alloc(w, false, st)) {
    delete w;
    return nullptr;
  }
  const void* src = rows;
  void* tmp = nullptr;
  if (!rows_on_device) {
    const size_t bytes = (size_t)n * nb01;
    if (!ns_cuda_ok(cudaMalloc(&tmp, bytes), "cudaMalloc(q6_K staging)") ||
        !ns_cuda_ok(cudaMemcpyAsync(tmp, rows, bytes, cudaMemcpyHostToDevice, st), "H2D q6_K rows")) {
      if (tmp) cudaFree(tmp);
      ns_weight_free(w);
      return nullptr;
    }
    src = tmp;
  }
  int rc = ns_launch_repack_q6k(src, nb01, w, st);
  if (tmp) {
    cudaStreamSynchronize(st);
    cudaFree(tmp);
  }
  if (rc) {
    ns_weight_free(w);
    return nullptr;
  }
  return w;
}

extern "C" ns_weight* ns_weight_from_unpacked(const int8_t* q, const float* scales, const int8_t* zp, const int* shuffle,
                                              int n, int k, int group, int wfmt, int stype, int comp, void* queue) {
  if (ns_ensure_device()) return nullptr;
  if (!q || !scales || n <= 0 || k <= 0 || wfmt < 0 || wfmt > NS_W_NF4 || stype < 0 || stype > NS_S_F16) {
    ns_set_error("ns_weight_from_unpacked: invalid arguments");
    return nullptr;
  }
  cudaStream_t st = stream_of(queue);
  ns_weight* w = new ns_weight();
  memset(w, 0, sizeof(*w));
  w->n = n;
  w->k = k;
  w->group = group;
  w->wfmt = wfmt;
  w->stype = stype;
  w->comp = comp;
  w->asym = zp ? 1 : 0;
  weight_layout(w);
  if ((w->group % 32 != 0 && w->group != w->k) || (wfmt == NS_W_NF4 && !(comp == NS_COMP_F32 || comp == NS_COMP_BF16))) {
    ns_set_error("ns_weight_from_unpacked: unsupported group %d / comp %d", group, comp);
    delete w;
    return nullptr;
  }
  if (weight_alloc(w, shuffle != nullptr, st)) {
    delete w;
    return nullptr;
  }
  const size_t qb = (size_t)k * n, sb = (size_t)w->ngroups * n * 4, zb = (size_t)w->ngroups * n;
  char* tmp = nullptr;
  const size_t tot = ns_round_up(qb, 256) + ns_round_up(sb, 256) + ns_round_up(zb, 256);
  bool ok = ns_cuda_ok(cudaMalloc((void**)&tmp, tot), "cudaMalloc(staging)");
  int8_t* dq = (int8_t*)tmp;
  float* ds = (float*)(tmp + ns_round_up(qb, 256));
  int8_t* dz = (int8_t*)(tmp + ns_round_up(qb, 256) + ns_round_up(sb, 256));
  ok = ok && ns_cuda_ok(cudaMemcpyAsync(dq, q, qb, cudaMemcpyHostToDevice, st), "H2D q");
  ok = ok && ns_cuda_ok(cudaMemcpyAsync(ds, scales, sb, cudaMemcpyHostToDevice, st), "H2D scales");
  if (zp) ok = ok && ns_cuda_ok(cudaMemcpyAsync(dz, zp, zb, cudaMemcpyHostToDevice, st), "H2D zp");
  if (shuffle) ok = ok && ns_cuda_ok(cudaMemcpyAsync(w->shuffle, shuffle, (size_t)k * 4, cudaMemcpyHostToDevice, st), "H2D shuffle");
  if (ok) ok = ns_launch_repack_canonical(dq, ds, zp ? dz : nullptr, w, st) == NS_OK;
  cudaStreamSynchronize(st);
  if (tmp) cudaFree(tmp);
  if (!ok) {
    ns_weight_free(w);
    return nullptr;
  }
  return w;
}

// ---- serialized BesTLA blob (btla_blob.h): what the device supports, and the upload ------------------------------------
static int blob_to_weight_meta(const BlobView& v, ns_weight* w) {
  memset(w, 0, sizeof(*w));
  w->n = v.n;
  w->k = v.k;
  w->group = v.blocksize;
  if (v.dtype == NS_BTLA_S4_CLIP || v.dtype == NS_BTLA_S2_CLIP || v.dtype == NS_BTLA_S3_CLIP)
    w->wfmt = NS_W_S4;  // 2- / 3-bit codes ride in the 4-bit container
  else if (v.dtype == NS_BTLA_S8 || v.dtype == NS_BTLA_S5_CLIP || v.dtype == NS_BTLA_S6_CLIP || v.dtype == NS_BTLA_S7_CLIP)
    w->wfmt = NS_W_S8;  // 5- / 6- / 7-bit codes in the 8-bit one
  else if (v.dtype == NS_BTLA_F4_NF4 || v.dtype == NS_BTLA_F4_BNB || v.dtype == NS_BTLA_F4_E2M1) {
    w->wfmt = NS_W_NF4;  // 4-bit codes into a 16-level table: the table is chosen per weight
    w->f4kind = v.dtype == NS_BTLA_F4_NF4 ? NS_F4_NF4 : v.dtype == NS_BTLA_F4_BNB ? NS_F4_BNB : NS_F4_E2M1;
  }
  else {
    ns_set_error("blob: weight dtype 0x%x not supported (int2..int8 / nf4 / fp4 are)", v.dtype);
    return NS_E_UNSUPPORTED;
  }
  if (v.sca_t == NS_BTLA_F32) w->stype = NS_S_F32;
  else if (v.sca_t == NS_BTLA_BF16) w->stype = NS_S_BF16;
  else if (v.sca_t == NS_BTLA_F16) w->stype = NS_S_F16;
  else {
    ns_set_error("blob: scale dtype 0x%x not supported (f32 / bf16 / f16 are)", v.sca_t);
    return NS_E_UNSUPPORTED;
  }
  // CompType B: tFP32=0 tBF16=1 tFP16=2 tS8=3 tU8=4 ; A: tU8=4 / tS8=3 (bestla_gemm.h:22-49)
  if (v.comp_b == 0) w->comp = NS_COMP_F32;
  else if (v.comp_b == 1) w->comp = NS_COMP_BF16;
  else if (v.comp_b == 2) w->comp = NS_COMP_F32;  // fp16 compute cores: evaluated in fp32 here (superset precision)
  else if (v.comp_b == 3 || v.comp_b == 4) w->comp = (v.comp_a == 3) ? NS_COMP_INT8_S8 : NS_COMP_INT8;
  else {
    ns_set_error("blob: compute type %d not supported", v.comp_b);
    return NS_E_UNSUPPORTED;
  }
  if (w->wfmt == NS_W_NF4 && !(w->comp == NS_COMP_F32 || w->comp == NS_COMP_BF16)) w->comp = NS_COMP_F32;
  w->asym = v.zp ? 1 : 0;
  weight_layout(w);
  if (w->group % 32 != 0 && w->group != w->k) {
    ns_set_error("blob: block size %d is not a multiple of 32", w->group);
    return NS_E_UNSUPPORTED;
  }
  return NS_OK;
}

// upload the pieces of a blob and repack into w (whose device pointers are already carved)
static int blob_upload_repack(const BlobView& v, ns_weight* w, cudaStream_t st) {
  // bit-plane codes (2, 3, 5, 6, 7 bits): transcoded on the host, element by element in the blob's own tile order, into the nibble
  // (q + 8) or byte (q) form of the 4- / 8-bit container the repack kernel reads -- the integers, scales and zero points are
  // unchanged, so every matmul path sees exactly the weight the reference would dequantise
  std::vector<uint8_t> trans;
  const uint8_t* qsrc = v.qbuf;
  size_t qbytes = v.qbytes;
  if (v.planes.n) {
    const size_t E = (size_t)v.npad * v.kpad;
    if (w->wfmt == NS_W_S4) {
      trans.assign(E / 2 + 1, 0);
      for (size_t e = 0; e < E; ++e) {
        const unsigned u = (unsigned)(blob_code(v, e) + 8) & 0xfu;
        trans[e >> 1] = (uint8_t)((e & 1) ? (trans[e >> 1] | (u << 4)) : u);
      }
      qbytes = E / 2;
    } else {
      trans.resize(E);
      for (size_t e = 0; e < E; ++e) trans[e] = (uint8_t)(int8_t)blob_code(v, e);
      qbytes = E;
    }
    qsrc = trans.data();
  }
  const size_t qb = ns_round_up(qbytes, 256), sb = ns_round_up(v.scale_bytes, 256), zb = ns_round_up(v.zp_bytes, 256);
  char* tmp = nullptr;
  NS_CUDA_TRY(cudaMalloc((void**)&tmp, qb + sb + zb + 256));
  bool ok = ns_cuda_ok(cudaMemcpyAsync(tmp, qsrc, qbytes, cudaMemcpyHostToDevice, st), "H2D qbuf");
  ok = ok && ns_cuda_ok(cudaMemcpyAsync(tmp + qb, v.scale, v.scale_bytes, cudaMemcpyHostToDevice, st), "H2D scales");
  if (v.zp) ok = ok && ns_cuda_ok(cudaMemcpyAsync(tmp + qb + sb, v.zp, v.zp_bytes, cudaMemcpyHostToDevice, st), "H2D zp");
  if (v.shuffle && w->shuffle)
    ok = ok && ns_cuda_ok(cudaMemcpyAsync(w->shuffle, v.shuffle, (size_t)v.k * 4, cudaMemcpyHostToDevice, st), "H2D shuffle");
  int rc = NS_E_CUDA;
  if (ok)
    rc = ns_launch_repack_btla(tmp, tmp + qb, w->stype, v.zp ? (const int8_t*)(tmp + qb + sb) : nullptr, v.cstep, v.kpad,
                               v.ntile, v.packrow, w->wfmt == NS_W_NF4, w, st);
  cudaStreamSynchronize(st);
  cudaFree(tmp);
  return rc;
}

// nbytes: bytes readable at `blob` (0: unknown, trust the blob's size field); a file-backed blob passes its tensor size so a
// corrupt size field cannot make the parser read past the buffer
extern "C" ns_weight* ns_weight_from_btla_blob_n(const void* blob, size_t nbytes, void* queue) {
  if (ns_ensure_device()) return nullptr;
  BlobView v;
  if (!parse_blob(blob, &v, nbytes)) return nullptr;
  ns_weight* w = new ns_weight();
  if (blob_to_weight_meta(v, w) || weight_alloc(w, v.shuffle != nullptr, stream_of(queue))) {
    delete w;
    return nullptr;
  }
  if (blob_upload_repack(v, w, stream_of(queue))) {
    ns_weight_free(w);
    return nullptr;
  }
  return w;
}

// Benchmark aid: a weight of the given geometry filled with random codes / scales / zero points on the device (the decode path is
// bandwidth bound: speed does not depend on the values; parity tests never use this).
extern "C" ns_weight* ns_weight_random(int n, int k, int group, int wfmt, int stype, int comp, int asym, unsigned seed, void* queue) {
  if (ns_ensure_device()) return nullptr;
  if (n <= 0 || k <= 0 || !(wfmt == NS_W_S4 || wfmt == NS_W_S8 || wfmt == NS_W_NF4 || wfmt == NS_W_Q8_0) || stype < 0 || stype > NS_S_F16 ||
      comp < 0 || comp > NS_COMP_INT8_S8 || (wfmt == NS_W_NF4 && (asym || !(comp == NS_COMP_F32 || comp == NS_COMP_BF16))) ||
      (wfmt == NS_W_Q8_0 && (k % 32 || group != 32 || stype != NS_S_F16 || comp != NS_COMP_Q8_0 || asym))) {
    ns_set_error("ns_weight_random: invalid geometry");
    return nullptr;
  }
  ns_weight* w = new ns_weight();
  memset(w, 0, sizeof(*w));
  w->n = n;
  w->k = k;
  w->group = group;
  w->wfmt = wfmt;
  w->stype = stype;
  w->comp = comp;
  w->asym = asym ? 1 : 0;
  weight_layout(w);
  if (weight_alloc(w, false, stream_of(queue)) || ns_launch_random_weight(w, seed, stream_of(queue))) {
    ns_weight_free(w);
    return nullptr;
  }
  return w;
}

extern "C" ns_weight* ns_weight_from_btla_blob(const void* blob, void* queue) { return ns_weight_from_btla_blob_n(blob, 0, queue); }

extern "C" int ns_weight_dequant_f32(const ns_weight* w, float* dst_dev, int ld, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!w || !dst_dev || ld < w->k) return NS_E_INVALID;
  if (w->wfmt == NS_W_Q6K) return ns_launch_dequant_q6k(w, dst_dev, ld, stream_of(queue));
  return ns_launch_dequant(w, dst_dev, ld, stream_of(queue));
}

// ---------------------------------------------------------------------------------------------------- device matmuls
// Every matmul node runs on one of four kernel paths, and the path fixes the node's numerics class (DESIGN.md section 4):
//   NS_PATH_GEMV  GEMV tiles of <= 4 rows: the TMA ring, or the register GEMV for the formats the ring does not take
//   NS_PATH_IMMA  integer tensor cores, 3..32 rows of int4 weights with an integer compute type or of ggml Q8_0 weights: the
//                 GEMV's exact block sums
//   NS_PATH_TC    wgmma GEMM, bf16 numerics
//   NS_PATH_Q6K   ggml Q6_K x Q8_K in tiles of <= 4 rows, plain nodes only
// ns_route is the one place that picks the path; the workspace of a node and whether an RMSNorm folds into it follow from it.
int ns_route(int kind, const ns_weight* const* w, int m, int flags) {
  if (kind == NS_NODE_PLAIN && w[0]->wfmt == NS_W_Q6K) return NS_PATH_Q6K;  // whatever the flags
  const int nw = kind == NS_NODE_QKV ? 3 : (kind == NS_NODE_FFN && w[1]) ? 2 : 1;  // the weights of the node's first launch
  const int mode = kind == NS_NODE_QKV ? NS_GEMV_CONCAT : nw == 2 ? NS_GEMV_GATE_UP_SILU : NS_GEMV_PLAIN;
  bool gemv_only = false;
  if (!(flags & (NS_MM_FORCE_GEMV | NS_MM_FORCE_TC)) && ns_gemm_imma_supported(w, nw, m)) {
    const bool imma = kind == NS_NODE_PLAIN ||
                      (kind == NS_NODE_QKV && w[0]->n % 2 == 0 && w[1]->n % 2 == 0) ||  // QKV: q and k need an even n
                      (kind == NS_NODE_FFN && ns_gemm_imma_supported(&w[2], 1, m));     // FFN: gate/up and down both, or neither
    if (imma) {
      if (ns_gemm_imma_planned(w, nw, mode, m) && (kind != NS_NODE_FFN || ns_gemm_imma_planned(&w[2], 1, NS_GEMV_PLAIN, m)))
        return NS_PATH_IMMA;
      // a launch the shared-memory planner cannot fit takes GEMV tiles: the same exact block sums, never the bf16 GEMM
      gemv_only = true;
    }
  }
  // The tensor-core GEMM has a fixed cost at small m (pipeline fill, split-K epilogue) while GEMV tiles keep the exact-integer
  // numerics: GEMV tiles up to 16 rows (the reference switches from its GEMV to the blocked GEMM at m > 4)
  bool tc = !gemv_only && !(flags & NS_MM_FORCE_GEMV) && (m > 16 || (flags & NS_MM_FORCE_TC)) && ns_gemm_tc_supported(w[0]);
  if (kind == NS_NODE_QKV)  // one bf16 activation image for all three: equal k, no act-order shuffles
    tc = tc && ns_gemm_tc_supported(w[1]) && ns_gemm_tc_supported(w[2]) && w[1]->k == w[0]->k && w[2]->k == w[0]->k &&
         !w[0]->shuffle && !w[1]->shuffle && !w[2]->shuffle;
  if (kind == NS_NODE_FFN)  // shuffles are checked on gate/up only
    tc = tc && ns_gemm_tc_supported(w[2]) && (!w[1] || ns_gemm_tc_supported(w[1])) && !w[0]->shuffle && !(w[1] && w[1]->shuffle);
  if (tc) return NS_PATH_TC;
  // the weights of the first launch must fit one GEMV launch, and an FFN's down projection one of its own; every tile of both
  // must have a kernel plan, so that a node the ring cannot run is refused before any of its launches is issued
  if (int rc = ns_gemv_check(w, nw, mode)) return rc;
  if (int rc = ns_gemv_planned(w, nw, mode, m, (flags & NS_ROUTE_NORM) != 0)) return rc;
  if (kind == NS_NODE_FFN) {
    if (int rc = ns_gemv_check(&w[2], 1, NS_GEMV_PLAIN)) return rc;
    if (int rc = ns_gemv_planned(&w[2], 1, NS_GEMV_PLAIN, m, false)) return rc;
  }
  return NS_PATH_GEMV;
}

// The RMSNorm in front of a launch of 1..3 weights folds into its activation quantiser when the launch is a ring GEMV that
// quantises its own activations: decode rows (m <= 2, below the tensor-core GEMM) that the integer tensor cores do not take
// (NS_IMMA_MIN_M may hand them 2 rows), k % 8 == 0
static bool norm_foldable(const ns_weight* const* w, int nw, int m) {
  static const bool off = getenv("NS_NO_FUSED_NORM") != nullptr;  // debugging aid: separate rmsnorm launches
  if (off || m < 1 || m > 2 || nw < 1) return false;
  for (int i = 0; i < nw; ++i)
    if (!w[i] || !ns_gemv_fused_quant_ok(w[i]) || w[i]->k % 8) return false;
  const int mode = nw == 3 ? NS_GEMV_CONCAT : nw == 2 ? NS_GEMV_GATE_UP_SILU : NS_GEMV_PLAIN;
  return !(ns_gemm_imma_supported(w, nw, m) && ns_gemm_imma_planned(w, nw, mode, m));
}

// kpad: the widest padded input of the node's launches
static size_t path_workspace_bytes(int path, int m, int kpad) {
  switch (path) {
    case NS_PATH_IMMA: return ns_gemm_imma_workspace_bound(m, kpad);
    case NS_PATH_TC: return ns_gemm_tc_workspace_bytes(m, kpad);  // bf16 [m][kpad]
    case NS_PATH_Q6K: return ns_q6k_workspace_bytes(4, kpad);
    default: return ns_act_workspace_bytes(4, kpad);  // activation images of <= 4-row tiles
  }
}
// Covers every path a node of up to m rows may take (NS_IMMA_MIN_M may hand a single row to the integer tensor cores, which
// take 32 at most), so one workspace serves every smaller call too
extern "C" size_t ns_device_workspace_bytes(int m, int k) {
  const int kpad = (int)ns_round_up((size_t)k, 32), rows = m < 1 ? 1 : m;
  size_t b = 0;
  for (int p = NS_PATH_GEMV; p <= NS_PATH_Q6K; ++p) {
    const size_t s = path_workspace_bytes(p, p == NS_PATH_IMMA && rows > 32 ? 32 : rows, kpad);
    b = s > b ? s : b;
  }
  return b;
}

static void* pick_ws(void* workspace, cudaStream_t st, size_t bytes) { return workspace ? workspace : scratch_get(st, bytes); }

static int norm_unsupported(const char* who) {
  ns_set_error("%s: the RMSNorm can only be folded into the ring GEMV (int4 weights with an integer compute type or Q8_0, <= 2 rows)", who);
  return NS_E_UNSUPPORTED;
}

// One launch of 1..3 weights sharing one activation on its path; mode, epilogue and dst layout as ns_launch_gemv.  The wgmma
// GEMM has no element-wise epilogue (the FFN applies its activation function on its own) and writes weight i at dst + i * m * ldo.
static int launch_set(int path, const ns_weight* const* w, int nw, int mode, const float* act, int lda, float* dst, int ldo, int m,
                      const float* bias, int bcast, const float* residual, int eltop, const float* norm_w, float norm_eps,
                      int one_image, void* ws, cudaStream_t st) {
  if (path == NS_PATH_IMMA) return ns_launch_gemm_imma(w, nw, mode, act, lda, dst, ldo, m, bias, bcast, residual, eltop, ws, st);
  if (path == NS_PATH_TC) {
    if (int rc = ns_launch_act_bf16(w[0], act, lda, m, ws, st)) return rc;
    const float* b = bias;
    for (int i = 0; i < nw; ++i) {
      if (int rc = ns_launch_gemm_tc(w[i], ws, dst + (size_t)i * m * ldo, ldo, m, b, bcast, residual, st)) return rc;
      // a QKV node's broadcast bias is [b_q | b_k | b_v]: each weight adds its own part
      if (b && bcast && mode == NS_GEMV_CONCAT) b += w[i]->n;
    }
    return NS_OK;
  }
  const int tile = path == NS_PATH_Q6K ? 4 : ns_gemv_tile_rows(w[0]);
  const bool fused = path == NS_PATH_GEMV && ns_gemv_fused_quant_ok(w[0]);  // the GEMV quantises the activations itself
  for (int m0 = 0; m0 < m; m0 += tile) {
    const int mt = (m - m0 < tile) ? (m - m0) : tile;
    const float* a = act + (size_t)m0 * lda;
    float* d = dst + (size_t)m0 * ldo;
    const float* b = bias ? (bcast ? bias : bias + (size_t)m0 * ldo) : nullptr;
    const float* r = residual ? residual + (size_t)m0 * ldo : nullptr;
    int rc = NS_OK;
    if (path == NS_PATH_Q6K) {
      rc = ns_launch_mul_mat_q6k(w[0], a, lda, d, ldo, mt, b, bcast, r, ws, st);
    } else {
      if (!fused) rc = ns_launch_act_prep(a, lda, mt, w[0], ws, st);
      if (!rc)
        rc = ns_launch_gemv(w, nw, mode, fused ? nullptr : ws, d, ldo, mt, m, b, bcast, r, nullptr, st, fused ? a : nullptr, lda, eltop,
                            norm_w, norm_eps, one_image);
    }
    if (rc) return rc;
  }
  return NS_OK;
}

static int mul_mat_impl(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* bias,
                        const float* residual, int flags, void* workspace, void* queue, const float* norm_w, float norm_eps,
                        int one_image = 0) {
  if (int rc = ns_ensure_device()) return rc;
  if (!w || !act || !dst || m <= 0 || lda < w->k || ldo < w->n) {
    ns_set_error("ns_mul_mat: invalid arguments (m=%d lda=%d ldo=%d)", m, lda, ldo);
    return NS_E_INVALID;
  }
  if (norm_w && !norm_foldable(&w, 1, m)) return norm_unsupported("ns_rmsnorm_mul_mat");
  const int path = ns_route(NS_NODE_PLAIN, &w, m, (flags & ~NS_ROUTE_NORM) | (norm_w ? NS_ROUTE_NORM : 0));
  if (path < 0) return path;
  cudaStream_t st = stream_of(queue);
  void* ws = pick_ws(workspace, st, path_workspace_bytes(path, m, w->kpad));
  if (!ws) return NS_E_CUDA;
  return launch_set(path, &w, 1, NS_GEMV_PLAIN, act, lda, dst, ldo, m, bias, (flags & NS_MM_BIAS_BCAST) ? 1 : 0, residual,
                    NS_ELT_DEFAULT, norm_w, norm_eps, one_image, ws, st);
}
extern "C" int ns_mul_mat(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* bias,
                          const float* residual, int flags, void* workspace, void* queue) {
  return mul_mat_impl(w, act, lda, dst, ldo, m, bias, residual, flags, workspace, queue, nullptr, 0.f);
}
int ns_mul_mat_engine(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* residual, void* workspace,
                      cudaStream_t st, const float* norm_w, float norm_eps) {
  return mul_mat_impl(w, act, lda, dst, ldo, m, nullptr, residual, 0, workspace, (void*)st, norm_w, norm_eps, 1);
}
extern "C" int ns_mul_mat_engine_image(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* residual,
                                       void* workspace, void* queue) {
  return mul_mat_impl(w, act, lda, dst, ldo, m, nullptr, residual, 0, workspace, queue, nullptr, 0.f, 1);
}
// dst = W * (rms_norm(act) * norm_w) [+ residual]: ne_rms_norm + ne_mul + ne_mul_mat (llama.cpp:205-215, :703-712) as ONE launch
extern "C" int ns_rmsnorm_mul_mat(const ns_weight* w, const float* act, int lda, const float* norm_w, float norm_eps, float* dst,
                                  int ldo, int m, const float* residual, void* workspace, void* queue) {
  if (!norm_w) return NS_E_INVALID;
  return mul_mat_impl(w, act, lda, dst, ldo, m, nullptr, residual, 0, workspace, queue, norm_w, norm_eps);
}

int ns_mul_mat_bias(const ns_weight* w, const float* act, int lda, float* dst, int ldo, int m, const float* bias, void* workspace,
                    cudaStream_t st, const float* norm_w, float norm_eps) {
  return mul_mat_impl(w, act, lda, dst, ldo, m, bias, nullptr, bias ? NS_MM_BIAS_BCAST : 0, workspace, (void*)st, norm_w, norm_eps);
}

// A broadcast bias of a QKV node is read at bias[i * m * ldo + row] by the GEMV and IMMA epilogues (the output's offset in the
// [3][m][ldo] layout): that is [b_q | b_k | b_v] for one row; the wgmma launches take one part each
bool ns_qkv_bias_ok(int path, int m) { return m == 1 || path == NS_PATH_TC; }

int ns_mul_qkv_norm(const ns_weight* wq, const ns_weight* wk, const ns_weight* wv, const float* act, int lda, float* dst, int ldo,
                    int m, void* workspace, void* queue, const float* norm_w, float norm_eps, const float* bias) {
  if (int rc = ns_ensure_device()) return rc;
  if (!wq || !wk || !wv || !act || !dst || m <= 0) return NS_E_INVALID;
  const ns_weight* wl[3] = {wq, wk, wv};
  if (norm_w && !norm_foldable(wl, 3, m)) return norm_unsupported("ns_rmsnorm_mul_qkv");
  const int path = ns_route(NS_NODE_QKV, wl, m, norm_w ? NS_ROUTE_NORM : 0);
  if (path < 0) return path;
  if (bias && (!ns_qkv_bias_ok(path, m) || ldo != wq->n || wk->n != wq->n || wv->n != wq->n)) {
    ns_set_error("ns_mul_qkv: a bias needs one row or the wgmma path, and ldo == n (m=%d path=%d)", m, path);
    return NS_E_UNSUPPORTED;
  }
  cudaStream_t st = stream_of(queue);
  void* ws = pick_ws(workspace, st, path_workspace_bytes(path, m, wq->kpad));
  if (!ws) return NS_E_CUDA;
  return launch_set(path, wl, 3, NS_GEMV_CONCAT, act, lda, dst, ldo, m, bias, bias ? 1 : 0, nullptr, NS_ELT_DEFAULT, norm_w, norm_eps, 0,
                    ws, st);
}
extern "C" int ns_mul_qkv(const ns_weight* wq, const ns_weight* wk, const ns_weight* wv, const float* act, int lda,
                          float* dst, int ldo, int m, void* workspace, void* queue) {
  return ns_mul_qkv_norm(wq, wk, wv, act, lda, dst, ldo, m, workspace, queue, nullptr, 0.f);
}
extern "C" int ns_rmsnorm_mul_qkv(const ns_weight* wq, const ns_weight* wk, const ns_weight* wv, const float* act, int lda,
                                  const float* norm_w, float norm_eps, float* dst, int ldo, int m, void* workspace, void* queue) {
  if (!norm_w) return NS_E_INVALID;
  return ns_mul_qkv_norm(wq, wk, wv, act, lda, dst, ldo, m, workspace, queue, norm_w, norm_eps);
}

// Fused feed-forward.  w3 != NULL: tmp = elt(x W1^T) * (x W3^T), dst = tmp W2^T (SiLu / Gelu_Mul, ip_fusion_ffn.cpp:734-753).
// w3 == NULL: tmp = gelu(x W1^T + b1), dst = tmp W2^T + b2 (GeLu / Add_GeLu, ip_fusion_ffn.cpp:755-779).
// tmp: [2][m][fmid] floats when m > 4 and w3 is given (gate and up GEMM outputs; the product lands in the first half), else [m][fmid]
static int ffn_impl(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, int eltop, const float* b1, const float* b2,
                    int bcast, const float* act, int lda, float* tmp, float* dst, int ldo, int m, void* workspace, void* queue,
                    const float* residual = nullptr, const float* norm_w = nullptr, float norm_eps = 0.f, int one_image = 0) {
  if (int rc = ns_ensure_device()) return rc;
  if (!w1 || !w2 || !act || !tmp || !dst || m <= 0 || w2->k != w1->n || (w3 && (w3->n != w1->n || w3->k != w1->k)) ||
      (w3 && (b1 || b2)) || (!w3 && eltop != NS_ELT_GELU)) {
    ns_set_error("fused FFN: invalid arguments");
    return NS_E_INVALID;
  }
  const ns_weight* wn[3] = {w1, w3, w2};
  const int ngu = w3 ? 2 : 1, fmid = w1->n;
  if (norm_w && !norm_foldable(wn, ngu, m)) return norm_unsupported("fused FFN");
  const int path = ns_route(NS_NODE_FFN, wn, m, norm_w ? NS_ROUTE_NORM : 0);
  if (path < 0) return path;
  cudaStream_t st = stream_of(queue);
  void* ws = pick_ws(workspace, st, path_workspace_bytes(path, m, w1->kpad > w2->kpad ? w1->kpad : w2->kpad));
  if (!ws) return NS_E_CUDA;
  if (int rc = launch_set(path, wn, ngu, w3 ? NS_GEMV_GATE_UP_SILU : NS_GEMV_PLAIN, act, lda, tmp, fmid, m, b1, bcast, nullptr, eltop,
                          norm_w, norm_eps, one_image, ws, st))
    return rc;
  if (path == NS_PATH_TC) {  // gate (and up) landed in tmp as plain GEMM outputs
    float* up = tmp + (size_t)m * fmid;
    int rc = NS_OK;
    // one_image (the eval step: nobody reads tmp): the product goes straight into the down projection's bf16 image (the
    // activation image of gate/up in `ws` is dead once both GEMMs have been issued -- stream order)
    if (w3 && one_image && ns_launch_silu_mul_bf16(w2, tmp, up, m, ws, st, eltop, &rc))
      return rc ? rc : ns_launch_gemm_tc(w2, ws, dst, ldo, m, b2, bcast, residual, st);
    rc = w3 ? ns_launch_silu_mul(tmp, up, tmp, nullptr, (size_t)m * fmid, st, eltop) : ns_launch_gelu(tmp, (size_t)m * fmid, st);
    if (rc) return rc;
  }
  return launch_set(path, &w2, 1, NS_GEMV_PLAIN, tmp, fmid, dst, ldo, m, b2, bcast, residual, NS_ELT_DEFAULT, nullptr, 0.f, one_image,
                    ws, st);
}
// dst = residual + FFN_SiLU(act): the decode engine's "cur = ne_add(ffn, inpFF)" (llama.cpp:698) folded into the down GEMV
int ns_ffn_silu_residual(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda, float* tmp,
                         float* dst, int ldo, int m, const float* residual, void* workspace, cudaStream_t st, const float* norm_w,
                         float norm_eps, int one_image) {
  if (!w3) return NS_E_INVALID;
  return ffn_impl(w1, w2, w3, NS_ELT_DEFAULT, nullptr, nullptr, 0, act, lda, tmp, dst, ldo, m, workspace, (void*)st, residual, norm_w,
                  norm_eps, one_image);
}
extern "C" int ns_ffn_silu_engine_image(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda,
                                        float* tmp, float* dst, int ldo, int m, const float* residual, void* workspace, void* queue) {
  if (!w3) return NS_E_INVALID;
  return ffn_impl(w1, w2, w3, NS_ELT_DEFAULT, nullptr, nullptr, 0, act, lda, tmp, dst, ldo, m, workspace, queue, residual, nullptr, 0.f,
                  1);
}
// dst = residual + FFN_SiLU(rms_norm(act) * norm_w): llama.cpp:601-698 with the norm folded into the gate/up launch
extern "C" int ns_rmsnorm_ffn_silu(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda,
                                   const float* norm_w, float norm_eps, float* tmp, float* dst, int ldo, int m, const float* residual,
                                   void* workspace, void* queue) {
  if (!w3 || !norm_w) return NS_E_INVALID;
  return ffn_impl(w1, w2, w3, NS_ELT_DEFAULT, nullptr, nullptr, 0, act, lda, tmp, dst, ldo, m, workspace, queue, residual, norm_w,
                  norm_eps);
}
// The plan of one ring launch of weight geometry w (n, k, group, wfmt, stype, comp, asym set; mode checked by the caller), as the
// launchers would run it: ns_gemv_ring_plan and ns_gemv_ring_plan_q8_0 differ only in the weights they describe
static int ring_plan_of(const char* who, ns_weight& w, int mode, int m, int fused, int norm, int* out) {
  ns_weight_layout(&w);
  if (w.group % 32 && w.group != w.k) {
    ns_set_error("%s: group size %d is not a multiple of 32", who, w.group);
    return NS_E_INVALID;
  }
  if (m < 1 || m > ns_gemv_tile_rows(&w) || (fused && !ns_gemv_fused_quant_ok(&w)) || (norm && (!fused || m > 2))) {
    ns_set_error("%s: no such launch (m=%d of at most %d, fused=%d, norm=%d)", who, m, ns_gemv_tile_rows(&w), fused, norm);
    return NS_E_INVALID;
  }
  RingChoice c;
  const bool ok = ns_gemv_ring_choose(w.kpad, w.pitch, mode, m >= 3 ? 4 : m, fused != 0, norm != 0, &c);
  out[0] = ok && c.wide, out[1] = ok ? c.plan.rows : 0, out[2] = ok ? c.plan.stages : 0, out[3] = ok ? c.plan.active : 0;
  out[4] = ok ? c.plan.ctas : 0;
  return ok ? 1 : 0;
}
extern "C" int ns_gemv_ring_plan(int k, int group, int stype, int asym, int comp, int mode, int m, int fused, int norm, int* out) {
  ns_weight w;
  memset(&w, 0, sizeof(w));
  w.n = 2, w.k = k, w.group = group, w.wfmt = NS_W_S4, w.stype = stype, w.comp = comp, w.asym = asym ? 1 : 0;
  if (k < 1 || stype < NS_S_F32 || stype > NS_S_F16 || !(comp == NS_COMP_INT8 || comp == NS_COMP_INT8_S8 || comp == NS_COMP_Q8_0) ||
      mode < NS_GEMV_PLAIN || mode > NS_GEMV_GATE_UP_SILU || !out) {
    ns_set_error("ns_gemv_ring_plan: not a ring GEMV launch (k=%d stype=%d comp=%d mode=%d)", k, stype, comp, mode);
    return NS_E_INVALID;
  }
  return ring_plan_of("ns_gemv_ring_plan", w, mode, m, fused, norm, out);
}
extern "C" int ns_gemv_ring_plan_q8_0(int k, int mode, int m, int fused, int norm, int* out) {
  ns_weight w;
  memset(&w, 0, sizeof(w));
  w.n = 2, w.k = k, w.group = 32, w.wfmt = NS_W_Q8_0, w.stype = NS_S_F16, w.comp = NS_COMP_Q8_0, w.asym = 0;
  if (k < 32 || k % 32 || mode < NS_GEMV_PLAIN || mode > NS_GEMV_GATE_UP_SILU || !out) {
    ns_set_error("ns_gemv_ring_plan_q8_0: not a ring GEMV launch (k=%d mode=%d)", k, mode);
    return NS_E_INVALID;
  }
  return ring_plan_of("ns_gemv_ring_plan_q8_0", w, mode, m, fused, norm, out);
}
extern "C" int ns_rmsnorm_fusable(const ns_weight* const* weights, int nw, int m) {
  return (weights && nw >= 1 && nw <= 3 && norm_foldable(weights, nw, m)) ? 1 : 0;
}
extern "C" int ns_ffn_silu(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* act, int lda,
                           float* tmp, float* dst, int ldo, int m, void* workspace, void* queue) {
  if (!w3) return NS_E_INVALID;
  return ffn_impl(w1, w2, w3, NS_ELT_DEFAULT, nullptr, nullptr, 0, act, lda, tmp, dst, ldo, m, workspace, queue);
}
extern "C" int ns_ffn_gelu(const ns_weight* w1, const ns_weight* w2, const ns_weight* w3, const float* b1, const float* b2,
                           int bias_bcast, const float* act, int lda, float* tmp, float* dst, int ldo, int m, void* workspace,
                           void* queue) {
  return ffn_impl(w1, w2, w3, NS_ELT_GELU, b1, b2, bias_bcast, act, lda, tmp, dst, ldo, m, workspace, queue);
}

// ---------------------------------------------------------------------------------------------------- expert-indexed nodes
// ne_mul_mat_id / ne_mul_id_ffn_silu (core/ne_layers.c:2384-2460; compute :7345-7498 ggml types, :7783-7916 BesTLA blobs,
// :8053-8071 fused FFN): dst[t] = W[ids[t * ids_stride + id]] . act[t].  See moe.cu for the grouping scheme.
struct ExpertPlan {
  std::vector<int> order;                 // token indices sorted (stably) by expert
  std::vector<std::pair<int, int>> span;  // per expert: [begin, end) inside `order`
  bool identity;                          // order == 0..m-1: the rows already lie grouped, no gather / scatter
};
static int plan_experts(const int32_t* ids, int ids_stride, int id, int ids_on_device, int m, int n_as, cudaStream_t st, ExpertPlan* pl) {
  if (!ids || ids_stride < 1 || id < 0 || id >= ids_stride || n_as < 1 || n_as > 256 || m < 1) {
    ns_set_error("ns_mul_mat_id: invalid ids (stride=%d id=%d n_as=%d m=%d)", ids_stride, id, n_as, m);
    return NS_E_INVALID;
  }
  std::vector<int32_t> host;
  const int32_t* h = ids;
  if (ids_on_device) {  // the routing decision is needed on the host to size the per-expert launches: one small D2H + sync
    host.resize((size_t)m * ids_stride);
    NS_CUDA_TRY(cudaMemcpyAsync(host.data(), ids, host.size() * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    NS_CUDA_TRY(cudaStreamSynchronize(st));
    h = host.data();
  }
  std::vector<int> count((size_t)n_as, 0);
  for (int t = 0; t < m; ++t) {
    const int e = h[(size_t)t * ids_stride + id];
    if (e < 0 || e >= n_as) {  // NE_ASSERT(row_id >= 0 && row_id < n_as), ne_layers.c:7445
      ns_set_error("ns_mul_mat_id: expert id %d of token %d outside [0, %d)", e, t, n_as);
      return NS_E_INVALID;
    }
    ++count[(size_t)e];
  }
  pl->span.assign((size_t)n_as, {0, 0});
  int at = 0;
  for (int e = 0; e < n_as; ++e) {
    pl->span[(size_t)e] = {at, at};
    at += count[(size_t)e];
  }
  pl->order.assign((size_t)m, 0);
  for (int t = 0; t < m; ++t) pl->order[(size_t)pl->span[(size_t)h[(size_t)t * ids_stride + id]].second++] = t;
  pl->identity = true;
  for (int t = 0; t < m; ++t) pl->identity = pl->identity && pl->order[(size_t)t] == t;
  return NS_OK;
}

// The host-side grouping on its own (no device needed): order[m] = token indices sorted stably by expert, span[2 * n_as] = per
// expert [begin, end) inside order.  Returns 1 when order is the identity (rows already grouped), 0 otherwise, < 0 on bad ids.
extern "C" int ns_moe_plan(const int32_t* ids, int ids_stride, int id, int m, int n_as, int* order, int* span) {
  ExpertPlan pl;
  if (int rc = plan_experts(ids, ids_stride, id, 0, m, n_as, nullptr, &pl)) return rc;
  if (order) memcpy(order, pl.order.data(), (size_t)m * sizeof(int));
  if (span)
    for (int e = 0; e < n_as; ++e) {
      span[2 * e] = pl.span[(size_t)e].first;
      span[2 * e + 1] = pl.span[(size_t)e].second;
    }
  return pl.identity ? 1 : 0;
}

// scratch of a grouped node: [order: m int][xg: m x k][yg: m x n][workspace of the matmuls]
struct ExpertScratch {
  int* order;
  float *xg, *yg;
  void* ws;
};
static int expert_scratch(const ExpertPlan& pl, int m, int k, int n, size_t mm_ws, cudaStream_t st, ExpertScratch* sc) {
  const size_t ob = ns_round_up((size_t)m * 4, 256), xb = ns_round_up((size_t)m * k * 4, 256), yb = ns_round_up((size_t)m * n * 4, 256);
  char* base = (char*)scratch_get(st, ob + xb + yb + mm_ws + 256);
  if (!base) return NS_E_CUDA;
  sc->order = (int*)base;
  sc->xg = (float*)(base + ob);
  sc->yg = (float*)(base + ob + xb);
  sc->ws = base + ob + xb + yb;
  if (!pl.identity) NS_CUDA_TRY(cudaMemcpyAsync(sc->order, pl.order.data(), (size_t)m * 4, cudaMemcpyHostToDevice, st));
  return NS_OK;
}

extern "C" int ns_mul_mat_id(const ns_weight* const* experts, int n_as, const int32_t* ids, int ids_stride, int id, int ids_on_device,
                             const float* act, int lda, float* dst, int ldo, int m, int flags, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!experts || !act || !dst || n_as < 1 || m < 1) return NS_E_INVALID;
  for (int e = 0; e < n_as; ++e)
    if (!experts[e] || experts[e]->n != experts[0]->n || experts[e]->k != experts[0]->k) {  // ne_are_same_shape(as[0], a), ne_layers.c:2409
      ns_set_error("ns_mul_mat_id: expert %d missing or of another shape", e);
      return NS_E_INVALID;
    }
  const int n = experts[0]->n, k = experts[0]->k;
  if (lda < k || ldo < n) return NS_E_INVALID;
  cudaStream_t st = stream_of(queue);
  ExpertPlan pl;
  if (int rc = plan_experts(ids, ids_stride, id, ids_on_device, m, n_as, st, &pl)) return rc;
  ExpertScratch sc;
  if (int rc = expert_scratch(pl, m, k, n, ns_device_workspace_bytes(m, k), st, &sc)) return rc;  // any slice of <= m rows
  const float* x = act;
  float* y = dst;
  int ldx = lda, ldy = ldo;
  if (!pl.identity) {
    if (int rc = ns_launch_move_rows(true, act, lda, sc.order, sc.xg, k, m, k, st)) return rc;
    x = sc.xg, y = sc.yg, ldx = k, ldy = n;
  }
  for (int e = 0; e < n_as; ++e) {
    const int b = pl.span[(size_t)e].first, c = pl.span[(size_t)e].second - b;
    if (c == 0) continue;
    if (int rc = mul_mat_impl(experts[e], x + (size_t)b * ldx, ldx, y + (size_t)b * ldy, ldy, c, nullptr, nullptr, flags, sc.ws, (void*)st,
                              nullptr, 0.f))
      return rc;
  }
  if (!pl.identity) return ns_launch_move_rows(false, sc.yg, n, sc.order, dst, ldo, m, n, st);
  return NS_OK;
}

// ne_mul_id_ffn_silu / _gelu: dst[t] = W2[e] (act(W1[e] x_t) * (W3[e] x_t)), e = ids[t * ids_stride + id].  The reference's
// compute (ne_layers.c:8053-8071, :8093-8111) reads ONE id (token 0) and applies that expert to every row -- exact for the
// decode step it is used in; here every token follows its own id.  tmp: [2][m][fmid] floats.
extern "C" int ns_ffn_id(const ns_weight* const* gate, const ns_weight* const* down, const ns_weight* const* up, int n_as, int gelu,
                         const int32_t* ids, int ids_stride, int id, int ids_on_device, const float* act, int lda, float* tmp,
                         float* dst, int ldo, int m, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!gate || !down || !up || !act || !tmp || !dst || n_as < 1 || m < 1) return NS_E_INVALID;
  for (int e = 0; e < n_as; ++e)
    if (!gate[e] || !down[e] || !up[e] || gate[e]->n != gate[0]->n || gate[e]->k != gate[0]->k || down[e]->n != down[0]->n ||
        down[e]->k != gate[0]->n || up[e]->n != gate[0]->n || up[e]->k != gate[0]->k) {
      ns_set_error("ns_ffn_id: expert %d missing or of another shape", e);
      return NS_E_INVALID;
    }
  const int k = gate[0]->k, fmid = gate[0]->n, n = down[0]->n;
  if (lda < k || ldo < n) return NS_E_INVALID;
  cudaStream_t st = stream_of(queue);
  ExpertPlan pl;
  if (int rc = plan_experts(ids, ids_stride, id, ids_on_device, m, n_as, st, &pl)) return rc;
  ExpertScratch sc;
  if (int rc = expert_scratch(pl, m, k, n, ns_device_workspace_bytes(m, k > fmid ? k : fmid), st, &sc)) return rc;
  const float* x = act;
  float* y = dst;
  int ldx = lda, ldy = ldo;
  if (!pl.identity) {
    if (int rc = ns_launch_move_rows(true, act, lda, sc.order, sc.xg, k, m, k, st)) return rc;
    x = sc.xg, y = sc.yg, ldx = k, ldy = n;
  }
  for (int e = 0; e < n_as; ++e) {
    const int b = pl.span[(size_t)e].first, c = pl.span[(size_t)e].second - b;
    if (c == 0) continue;
    if (int rc = ffn_impl(gate[e], down[e], up[e], gelu ? NS_ELT_GELU : NS_ELT_DEFAULT, nullptr, nullptr, 0, x + (size_t)b * ldx, ldx,
                          tmp + (size_t)2 * b * fmid, y + (size_t)b * ldy, ldy, c, sc.ws, (void*)st))
      return rc;
  }
  if (!pl.identity) return ns_launch_move_rows(false, sc.yg, n, sc.order, dst, ldo, m, n, st);
  return NS_OK;
}

extern "C" int ns_prepare_activation(const ns_weight* w, const float* act, int lda, int m, void* workspace, void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!w || !act || !workspace || m < 1 || m > ns_gemv_tile_rows(w) || lda < w->k) {
    ns_set_error("ns_prepare_activation: invalid arguments (m=%d)", m);
    return NS_E_INVALID;
  }
  return ns_launch_act_prep(act, lda, m, w, workspace, stream_of(queue));
}

extern "C" int ns_matmul_prepared(const ns_weight* const* weights, int nw, int mode, const void* workspace, float* dst,
                                  int ldo, int m, const float* bias, int bias_bcast, const float* residual, float* aux,
                                  void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  if (!weights || nw < 1 || nw > 3 || mode < 0 || mode > 2 || !workspace || !dst) {
    ns_set_error("ns_matmul_prepared: invalid arguments");
    return NS_E_INVALID;
  }
  return ns_launch_gemv(weights, nw, mode, workspace, dst, ldo, m, m, bias, bias_bcast, residual, aux, stream_of(queue));
}

// ---------------------------------------------------------------------------------------------------- CUDA graphs
struct ns_graph {
  cudaGraph_t graph;
  cudaGraphExec_t exec;
};
extern "C" int ns_graph_begin(void* queue) {
  if (int rc = ns_ensure_device()) return rc;
  NS_CUDA_TRY(cudaStreamBeginCapture(stream_of(queue), cudaStreamCaptureModeThreadLocal));
  return NS_OK;
}
extern "C" ns_graph* ns_graph_end(void* queue) {
  cudaGraph_t g = nullptr;
  if (!ns_cuda_ok(cudaStreamEndCapture(stream_of(queue), &g), "cudaStreamEndCapture") || !g) return nullptr;
  cudaGraphExec_t e = nullptr;
  if (!ns_cuda_ok(cudaGraphInstantiate(&e, g, 0), "cudaGraphInstantiate")) {
    cudaGraphDestroy(g);
    return nullptr;
  }
  ns_graph* r = new ns_graph();
  r->graph = g;
  r->exec = e;
  return r;
}
extern "C" int ns_graph_launch(ns_graph* g, void* queue) {
  if (!g) return NS_E_INVALID;
  NS_CUDA_TRY(cudaGraphLaunch(g->exec, stream_of(queue)));
  return NS_OK;
}
extern "C" void ns_graph_free(ns_graph* g) {
  if (!g) return;
  cudaGraphExecDestroy(g->exec);
  cudaGraphDestroy(g->graph);
  delete g;
}

// ---------------------------------------------------------------------------------------------------- device set
extern "C" void bestla_init(void) { (void)ns_ensure_device(); }
extern "C" int bestla_set_threads(int nth) { return nth; }
extern "C" void* bestla_get_thread_handle(void) { return nullptr; }
extern "C" void bestla_timer(bool) {}

extern "C" void* bestla_create_device(bool profile) {
  if (ns_ensure_device()) ns_fatal("bestla_create_device: %s", g_err);
  ns_device* d = new ns_device();
  d->dev = g_default.dev;
  d->profile = profile;
  if (cudaStreamCreateWithFlags(&d->stream, cudaStreamNonBlocking) != cudaSuccess) ns_fatal("cudaStreamCreate failed");
  return d;
}
extern "C" void* bestla_get_device_queue(void* device) { return device ? (void*)((ns_device*)device)->stream : nullptr; }
extern "C" void bestla_release_device(void* device) {
  if (!device) return;
  ns_device* d = (ns_device*)device;
  cudaStreamSynchronize(d->stream);
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_scratch.find(d->stream);
    if (it != g_scratch.end()) {
      cudaFree(it->second.p);
      g_scratch.erase(it);
    }
  }
  cudaStreamDestroy(d->stream);
  delete d;
}
extern "C" size_t bestla_device_gmem_size(void* device) {
  (void)device;
  if (ns_ensure_device()) return 0;
  size_t fr = 0, tot = 0;
  cudaMemGetInfo(&fr, &tot);
  return tot;
}
extern "C" void* bestla_device_malloc(size_t size, void* queue) {
  (void)queue;
  if (ns_ensure_device()) ns_fatal("bestla_device_malloc: %s", g_err);
  void* p = nullptr;
  if (cudaMalloc(&p, size) != cudaSuccess) return nullptr;
  return p;
}
extern "C" void bestla_device_free(void* ptr, void* queue) {
  if (!ptr) return;
  cudaStreamSynchronize(stream_of(queue));
  cudaFree(ptr);
}
extern "C" void bestla_device_memcpy(void* dstptr, const void* srcptr, size_t size, void* queue) {
  if (ns_ensure_device()) ns_fatal("bestla_device_memcpy: %s", g_err);
  if (cudaMemcpyAsync(dstptr, srcptr, size, cudaMemcpyDefault, stream_of(queue)) != cudaSuccess)
    ns_fatal("bestla_device_memcpy failed: %s", cudaGetErrorString(cudaGetLastError()));
}
extern "C" void bestla_device_memcpy_sync(void* dstptr, const void* srcptr, size_t size, void* queue) {
  bestla_device_memcpy(dstptr, srcptr, size, queue);
  cudaStreamSynchronize(stream_of(queue));
}
extern "C" void bestla_device_sync(void* queue) {
  if (ns_ensure_device()) ns_fatal("bestla_device_sync: %s", g_err);
  if (cudaStreamSynchronize(stream_of(queue)) != cudaSuccess)
    ns_fatal("bestla_device_sync: %s", cudaGetErrorString(cudaGetLastError()));
}
extern "C" size_t bestla_device_storage_size(void) { return sizeof(ns_weight); }
extern "C" size_t ns_device_storage_bytes(const void* hoststor) {
  BlobView v;
  ns_weight w;
  if (!parse_blob(hoststor, &v) || blob_to_weight_meta(v, &w)) return 0;
  return weight_image_bytes(&w, v.shuffle != nullptr);
}
extern "C" void bestla_device_load_storage(void* hoststor, void* devstor, void* deviceptr, void* queue) {
  if (ns_ensure_device()) ns_fatal("bestla_device_load_storage: %s", g_err);
  BlobView v;
  ns_weight* w = (ns_weight*)devstor;
  if (!devstor || !deviceptr || !parse_blob(hoststor, &v) || blob_to_weight_meta(v, w))
    ns_fatal("bestla_device_load_storage: invalid parameters (%s)", g_err);
  w->base = deviceptr;
  w->external = 1;
  w->total_bytes = weight_image_bytes(w, v.shuffle != nullptr);
  weight_carve(w, deviceptr, v.shuffle != nullptr);
  if (cudaMemsetAsync(deviceptr, 0, w->total_bytes, stream_of(queue)) != cudaSuccess) ns_fatal("cudaMemset failed");
  if (blob_upload_repack(v, w, stream_of(queue))) ns_fatal("bestla_device_load_storage: %s", g_err);
}
extern "C" void bestla_device_f32f32_forward(float* activation, void* weiptr, float* output, int m, int n, int k, int lda,
                                             int ldo, void* workspace, void* queue) {
  const ns_weight* w = (const ns_weight*)weiptr;
  if (!w || w->n != n || w->k != k) ns_fatal("invalid parameters");
  (void)lda;  // the reference ignores lda and uses K (bestla_gemm.cpp:44,95)
  if (ns_mul_mat(w, activation, k, output, ldo, m, nullptr, nullptr, 0, workspace, queue))
    ns_fatal("bestla_device_f32f32_forward: %s", g_err);
}

// ---------------------------------------------------------------------------------------------------- host drop-ins
// Host blobs / ggml rows are uploaded and repacked once and cached by address (weights are immutable for the lifetime of
// the model context in the reference: model_files.h:1490-1499).
struct CacheEntry {
  ns_weight* w;
  size_t tag;
};
static std::unordered_map<const void*, CacheEntry> g_cache;

// Identity check so a recycled address holding a different tensor is re-uploaded: FNV-1a over the header bytes AND 256 eight-byte
// samples spread over the whole payload (two layers' wq share every header field; only the weights differ), plus the size.
// Reads stay inside [blob, blob + nbytes).  ns_host_cache_clear() drops every entry (call it when a model is freed).
static size_t blob_tag(const void* blob, size_t nbytes) {
  size_t t = 1469598103934665603ull;
  const unsigned char* p = (const unsigned char*)blob;
  const size_t head = nbytes < 64 ? nbytes : 64;
  for (size_t i = 0; i < head; ++i) t = (t ^ p[i]) * 1099511628211ull;
  if (nbytes > 72) {
    const size_t span = nbytes - 8, steps = 256;
    for (size_t j = 0; j < steps; ++j) {
      const size_t off = 64 + (size_t)((__uint128_t)(span - 64) * j / steps);
      unsigned long long v;
      memcpy(&v, p + off, 8);
      t = (t ^ (size_t)v) * 1099511628211ull;
    }
  }
  return (t ^ nbytes) * 1099511628211ull;
}

static const ns_weight* cached_blob(const void* blob) {
  if (ns_ensure_device()) ns_fatal("%s", g_err);
  const size_t msize = blob_size(blob);  // an implausible size field: hash the header only (the upload then refuses the blob)
  const size_t tag = blob_tag(blob, msize ? msize : 64);
  {
    std::lock_guard<std::mutex> lk(g_mu);
    auto it = g_cache.find(blob);
    if (it != g_cache.end() && it->second.tag == tag) return it->second.w;
  }
  ns_weight* w = ns_weight_from_btla_blob(blob, nullptr);
  if (!w) return nullptr;
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_cache.find(blob);
  if (it != g_cache.end()) ns_weight_free(it->second.w);
  g_cache[blob] = CacheEntry{w, tag};
  return w;
}

struct HostIO {  // device staging for host-buffer calls
  float* act = nullptr;
  float* out = nullptr;
  float* tmp = nullptr;
  float* bias = nullptr;
  size_t act_elems = 0, out_elems = 0, tmp_elems = 0, bias_elems = 0;
};
static HostIO g_io;
static bool io_reserve(float** p, size_t* have, size_t need) {
  if (*have >= need) return true;
  if (*p) cudaFree(*p);
  *p = nullptr;
  *have = 0;
  if (cudaMalloc((void**)p, need * sizeof(float)) != cudaSuccess) return false;
  *have = need;
  return true;
}

extern "C" unsigned long long bestla_f32f32_get_workspace_size(int m, int n, int k, void* wptr) {
  (void)n;
  (void)wptr;
  return (unsigned long long)m * ns_round_up((size_t)k, 128) * 4;  // inner_product.cpp:20-25
}

static void host_forward(float* activation, const ns_weight* w, float* bias, bool bias_bcast, float* output, int m, int n,
                         int k, int ldo) {
  cudaStream_t st = default_stream();
  if (!io_reserve(&g_io.act, &g_io.act_elems, (size_t)m * k) || !io_reserve(&g_io.out, &g_io.out_elems, (size_t)m * n + (bias ? (size_t)m * n : 0)))
    ns_fatal("device staging allocation failed");
  float* dbias = nullptr;
  if (cudaMemcpyAsync(g_io.act, activation, (size_t)m * k * 4, cudaMemcpyHostToDevice, st) != cudaSuccess) ns_fatal("H2D failed");
  if (bias) {
    dbias = g_io.out + (size_t)m * n;
    const size_t nb = bias_bcast ? (size_t)n : (size_t)m * n;
    if (bias_bcast) {
      cudaMemcpyAsync(dbias, bias, nb * 4, cudaMemcpyHostToDevice, st);
    } else {
      cudaMemcpy2DAsync(dbias, (size_t)n * 4, bias, (size_t)ldo * 4, (size_t)n * 4, m, cudaMemcpyHostToDevice, st);
    }
  }
  if (ns_mul_mat(w, g_io.act, k, g_io.out, n, m, dbias, nullptr, bias_bcast ? NS_MM_BIAS_BCAST : 0, nullptr, st))
    ns_fatal("%s", g_err);
  if (cudaMemcpy2DAsync(output, (size_t)ldo * 4, g_io.out, (size_t)n * 4, (size_t)n * 4, m, cudaMemcpyDeviceToHost, st) != cudaSuccess)
    ns_fatal("D2H failed");
  if (cudaStreamSynchronize(st) != cudaSuccess) ns_fatal("kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
}

extern "C" void bestla_f32f32_forward(float* activation, void* weiptr, float* output, int m, int n, int k, int lda, int ldo,
                                      void* workspace) {
  (void)lda;
  (void)workspace;
  const ns_weight* w = cached_blob(weiptr);
  if (!w || w->n != n || w->k != k || !activation || !output || m <= 0 || ldo < n) {
    printf("Err: invalid parameters\n");
    ns_fatal("bestla_f32f32_forward(m=%d n=%d k=%d): %s", m, n, k, g_err);
  }
  host_forward(activation, w, nullptr, false, output, m, n, k, ldo);
}

extern "C" bool bestla_fusion_add_f32f32_support(void* weiptr, int m, int n, int k) {
  (void)m;
  BlobView v;
  ns_weight w;
  return parse_blob(weiptr, &v) && blob_to_weight_meta(v, &w) == NS_OK && v.n == n && v.k == k;
}
extern "C" void bestla_fusion_add_f32f32_forward(float* activation, void* weiptr, float* bias, float* output, int m, int n,
                                                 int k, int lda, int ldo, bool boardcast_bias, void* workspace) {
  (void)lda;
  (void)workspace;
  const ns_weight* w = cached_blob(weiptr);
  if (!w || w->n != n || w->k != k || !activation || !output || !bias) ns_fatal("invalid parameters (%s)", g_err);
  host_forward(activation, w, bias, boardcast_bias, output, m, n, k, ldo);
}

extern "C" unsigned long long bestla_fusion_QKV_f32f32_get_workspace_size(int m, int n, int k, void* w1ptr) {
  return bestla_f32f32_get_workspace_size(m, n, k, w1ptr);  // ip_fusion_qkv.cpp:155-161
}
extern "C" bool bestla_fusion_QKV_f32f32_support(void* wqptr, void* wkptr, void* wvptr, int m, int n, int k) {
  (void)m;
  BlobView v[3];
  ns_weight w[3];
  void* ptrs[3] = {wqptr, wkptr, wvptr};
  for (int i = 0; i < 3; ++i) {
    if (!parse_blob(ptrs[i], &v[i]) || blob_to_weight_meta(v[i], &w[i]) != NS_OK) return false;
    if (v[i].n != n || v[i].k != k) return false;
    // same core / prologue for all three and no activation shuffle (ip_fusion_qkv.cpp:170-186)
    if (v[i].core_id != v[0].core_id || v[i].prologue != v[0].prologue || v[i].shuffle) return false;
    if (w[i].group != w[0].group || w[i].wfmt != w[0].wfmt || w[i].stype != w[0].stype || w[i].asym != w[0].asym) return false;
  }
  return (n % 2) == 0;
}
extern "C" void bestla_fusion_QKV_f32f32_forward(float* activation, void* wqptr, void* wkptr, void* wvptr, float* output,
                                                 int m, int n, int k, int lda, int ldo, void* workspace) {
  (void)lda;
  (void)workspace;
  const ns_weight* wq = cached_blob(wqptr);
  const ns_weight* wk = cached_blob(wkptr);
  const ns_weight* wv = cached_blob(wvptr);
  if (!wq || !wk || !wv || wq->n != n || wq->k != k) ns_fatal("invalid parameters (%s)", g_err);
  cudaStream_t st = default_stream();
  if (!io_reserve(&g_io.act, &g_io.act_elems, (size_t)m * k) || !io_reserve(&g_io.out, &g_io.out_elems, (size_t)3 * m * ldo))
    ns_fatal("device staging allocation failed");
  cudaMemcpyAsync(g_io.act, activation, (size_t)m * k * 4, cudaMemcpyHostToDevice, st);
  if (ns_mul_qkv(wq, wk, wv, g_io.act, k, g_io.out, ldo, m, nullptr, st)) ns_fatal("%s", g_err);
  cudaMemcpyAsync(output, g_io.out, (size_t)3 * m * ldo * 4, cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) ns_fatal("kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
}

extern "C" unsigned long long bestla_fusion_FFN_f32f32_get_workspace_size(int seq, int fin, int fmid, int fout, void* w1ptr,
                                                                          void* w2ptr) {
  (void)fout;
  (void)w1ptr;
  (void)w2ptr;
  const int kmax = fin > fmid ? fin : fmid;
  return (unsigned long long)seq * ns_round_up((size_t)kmax, 128) * 4;
}
extern "C" bool bestla_fusion_FFN_SiLu_f32f32_support(void* w1ptr, void* w2ptr, void* w3ptr, int seq, int fin, int fmid,
                                                      int fout) {
  (void)seq;
  BlobView v[3];
  ns_weight w[3];
  void* ptrs[3] = {w1ptr, w2ptr, w3ptr};
  for (int i = 0; i < 3; ++i)
    if (!parse_blob(ptrs[i], &v[i]) || blob_to_weight_meta(v[i], &w[i]) != NS_OK || v[i].shuffle) return false;
  if (v[0].n != fmid || v[0].k != fin || v[2].n != fmid || v[2].k != fin || v[1].n != fout || v[1].k != fmid) return false;
  if (v[0].core_id != v[2].core_id || v[0].core_id != v[1].core_id) return false;
  return w[0].group == w[2].group && w[0].wfmt == w[2].wfmt && w[0].stype == w[2].stype && w[0].asym == w[2].asym;
}
extern "C" void bestla_fusion_FFN_SiLu_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, void* w3ptr, float* tmp1,
                                                      float* tmp2, float* output, int seq, int fin, int fmid, int fout,
                                                      void* workspace) {
  (void)workspace;
  (void)tmp1;
  const ns_weight* w1 = cached_blob(w1ptr);
  const ns_weight* w2 = cached_blob(w2ptr);
  const ns_weight* w3 = cached_blob(w3ptr);
  if (!w1 || !w2 || !w3 || w1->n != fmid || w1->k != fin || w2->n != fout || w2->k != fmid) ns_fatal("invalid parameters (%s)", g_err);
  cudaStream_t st = default_stream();
  if (!io_reserve(&g_io.act, &g_io.act_elems, (size_t)seq * fin) || !io_reserve(&g_io.out, &g_io.out_elems, (size_t)seq * fout) ||
      !io_reserve(&g_io.tmp, &g_io.tmp_elems, (size_t)2 * seq * fmid))
    ns_fatal("device staging allocation failed");
  cudaMemcpyAsync(g_io.act, activation, (size_t)seq * fin * 4, cudaMemcpyHostToDevice, st);
  if (ns_ffn_silu(w1, w2, w3, g_io.act, fin, g_io.tmp, g_io.out, fout, seq, nullptr, st)) ns_fatal("%s", g_err);
  cudaMemcpyAsync(output, g_io.out, (size_t)seq * fout * 4, cudaMemcpyDeviceToHost, st);
  if (tmp2) cudaMemcpyAsync(tmp2, g_io.tmp, (size_t)seq * fmid * 4, cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) ns_fatal("kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
}

static bool ffn2_support(void* w1ptr, void* w2ptr, int fin, int fmid, int fout) {
  BlobView v[2];
  ns_weight w[2];
  void* ptrs[2] = {w1ptr, w2ptr};
  for (int i = 0; i < 2; ++i)
    if (!parse_blob(ptrs[i], &v[i]) || blob_to_weight_meta(v[i], &w[i]) != NS_OK || v[i].shuffle) return false;
  if (v[0].n != fmid || v[0].k != fin || v[1].n != fout || v[1].k != fmid) return false;
  return v[0].core_id == v[1].core_id;  // ffn_2w::bestla_fusion_ffn_f32f32_support, ip_fusion_ffn.cpp:33-77
}
static void ffn_host(float* activation, void* w1ptr, void* w2ptr, void* w3ptr, int eltop, float* b1, float* b2, bool bcast,
                     float* tmp1, float* tmp2, float* output, int seq, int fin, int fmid, int fout) {
  const ns_weight* w1 = cached_blob(w1ptr);
  const ns_weight* w2 = cached_blob(w2ptr);
  const ns_weight* w3 = w3ptr ? cached_blob(w3ptr) : nullptr;
  if (!w1 || !w2 || (w3ptr && !w3) || w1->n != fmid || w1->k != fin || w2->n != fout || w2->k != fmid)
    ns_fatal("invalid parameters (%s)", g_err);
  cudaStream_t st = default_stream();
  const size_t nb1 = b1 ? (bcast ? (size_t)fmid : (size_t)seq * fmid) : 0, nb2 = b2 ? (bcast ? (size_t)fout : (size_t)seq * fout) : 0;
  if (!io_reserve(&g_io.act, &g_io.act_elems, (size_t)seq * fin) || !io_reserve(&g_io.out, &g_io.out_elems, (size_t)seq * fout) ||
      !io_reserve(&g_io.tmp, &g_io.tmp_elems, (size_t)2 * seq * fmid) || !io_reserve(&g_io.bias, &g_io.bias_elems, nb1 + nb2 + 1))
    ns_fatal("device staging allocation failed");
  cudaMemcpyAsync(g_io.act, activation, (size_t)seq * fin * 4, cudaMemcpyHostToDevice, st);
  if (b1) cudaMemcpyAsync(g_io.bias, b1, nb1 * 4, cudaMemcpyHostToDevice, st);
  if (b2) cudaMemcpyAsync(g_io.bias + nb1, b2, nb2 * 4, cudaMemcpyHostToDevice, st);
  if (ffn_impl(w1, w2, w3, eltop, b1 ? g_io.bias : nullptr, b2 ? g_io.bias + nb1 : nullptr, bcast ? 1 : 0, g_io.act, fin, g_io.tmp,
               g_io.out, fout, seq, nullptr, st))
    ns_fatal("%s", g_err);
  cudaMemcpyAsync(output, g_io.out, (size_t)seq * fout * 4, cudaMemcpyDeviceToHost, st);
  // the reference leaves the activated intermediate in tmp1 (2w) / the gated product in tmp2 (3w)
  float* tmp_host = w3 ? tmp2 : tmp1;
  if (tmp_host) cudaMemcpyAsync(tmp_host, g_io.tmp, (size_t)seq * fmid * 4, cudaMemcpyDeviceToHost, st);
  if (cudaStreamSynchronize(st) != cudaSuccess) ns_fatal("kernel failed: %s", cudaGetErrorString(cudaGetLastError()));
}
extern "C" bool bestla_fusion_FFN_Gelu_Mul_f32f32_support(void* w1ptr, void* w2ptr, void* w3ptr, int seq, int fin, int fmid,
                                                          int fout) {
  return bestla_fusion_FFN_SiLu_f32f32_support(w1ptr, w2ptr, w3ptr, seq, fin, fmid, fout);
}
extern "C" void bestla_fusion_FFN_Gelu_Mul_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, void* w3ptr, float* tmp1,
                                                          float* tmp2, float* output, int seq, int fin, int fmid, int fout,
                                                          void* workspace) {
  (void)workspace;
  ffn_host(activation, w1ptr, w2ptr, w3ptr, NS_ELT_GELU, nullptr, nullptr, false, tmp1, tmp2, output, seq, fin, fmid, fout);
}
extern "C" bool bestla_fusion_FFN_GeLu_f32f32_support(void* w1ptr, void* w2ptr, int seq, int fin, int fmid, int fout) {
  (void)seq;
  return ffn2_support(w1ptr, w2ptr, fin, fmid, fout);
}
extern "C" void bestla_fusion_FFN_GeLu_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, float* tmp1, float* output,
                                                      int seq, int fin, int fmid, int fout, void* workspace) {
  (void)workspace;
  ffn_host(activation, w1ptr, w2ptr, nullptr, NS_ELT_GELU, nullptr, nullptr, false, tmp1, nullptr, output, seq, fin, fmid, fout);
}
extern "C" bool bestla_fusion_FFN_Add_GeLu_f32f32_support(void* w1ptr, void* w2ptr, int seq, int fin, int fmid, int fout) {
  (void)seq;
  return ffn2_support(w1ptr, w2ptr, fin, fmid, fout);
}
extern "C" void bestla_fusion_FFN_Add_GeLu_f32f32_forward(float* activation, void* w1ptr, void* w2ptr, float* b1ptr, float* b2ptr,
                                                          float* tmp1, float* output, int seq, int fin, int fmid, int fout,
                                                          bool boardcast_bias, void* workspace) {
  (void)workspace;
  ffn_host(activation, w1ptr, w2ptr, nullptr, NS_ELT_GELU, b1ptr, b2ptr, boardcast_bias, tmp1, nullptr, output, seq, fin, fmid, fout);
}

extern "C" void bestla_unpackweight_fp32(void* wptr, int n, int k, float* fp32data, int ld) {
  const ns_weight* w = cached_blob(wptr);
  if (!w || w->n != n || w->k != k || ld < k) ns_fatal("bestla_unpackweight_fp32: invalid parameters (%s)", g_err);
  cudaStream_t st = default_stream();
  float* d = nullptr;
  if (cudaMalloc((void**)&d, (size_t)n * k * 4) != cudaSuccess) ns_fatal("cudaMalloc failed");
  if (ns_launch_dequant(w, d, k, st)) ns_fatal("%s", g_err);
  cudaMemcpy2DAsync(fp32data, (size_t)ld * 4, d, (size_t)k * 4, (size_t)k * 4, n, cudaMemcpyDeviceToHost, st);
  cudaStreamSynchronize(st);
  cudaFree(d);
}

// drops every device copy the host drop-ins cached by address (model free / reload); the device memory is released
extern "C" void ns_host_cache_clear(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto& kv : g_cache) ns_weight_free(kv.second.w);
  g_cache.clear();
}
extern "C" size_t ns_host_cache_entries(void) {
  std::lock_guard<std::mutex> lk(g_mu);
  return g_cache.size();
}

// ggml host drop-in; type: which block the rows hold
enum { GG_Q4_0 = 0, GG_Q6_K = 1, GG_Q8_0 = 2 };
static int gg_block_elems(int type) { return type == GG_Q6_K ? 256 : 32; }
static size_t gg_block_bytes(int type) { return type == GG_Q6_K ? 210 : type == GG_Q8_0 ? 34 : 18; }
static const ns_weight* ggml_cached_weight(int type, const void* src0_rows, size_t nb01, int ne00, int ne01) {
  const size_t tag = blob_tag(src0_rows, (size_t)(ne01 - 1) * nb01 + (size_t)(ne00 / gg_block_elems(type)) * gg_block_bytes(type)) ^
                     ((size_t)ne00 << 32) ^ (size_t)ne01 ^ ((size_t)type << 62);
  std::unique_lock<std::mutex> lk(g_mu);
  auto it = g_cache.find(src0_rows);
  if (it != g_cache.end() && it->second.tag == tag) return it->second.w;
  lk.unlock();
  ns_weight* nw = type == GG_Q6_K   ? ns_weight_from_q6_K(src0_rows, ne01, ne00, nb01, 0, nullptr)
                  : type == GG_Q8_0 ? ns_weight_from_q8_0(src0_rows, ne01, ne00, nb01, 0, nullptr)
                                    : ns_weight_from_q4_0(src0_rows, ne01, ne00, nb01, 0, nullptr);
  if (!nw) return nullptr;
  lk.lock();
  auto it2 = g_cache.find(src0_rows);
  if (it2 != g_cache.end()) ns_weight_free(it2->second.w);
  g_cache[src0_rows] = CacheEntry{nw, tag};
  return nw;
}
static int ggml_mul_mat_host(int type, const void* src0_rows, size_t nb01, const float* src1, float* dst, int ne00, int ne01, int ne11) {
  if (int rc = ns_ensure_device()) return rc;
  if (!src0_rows || !src1 || !dst || ne00 % gg_block_elems(type) != 0 || ne01 <= 0 || ne11 <= 0) {
    ns_set_error("ggml host matmul: invalid arguments");
    return NS_E_INVALID;
  }
  const ns_weight* w = ggml_cached_weight(type, src0_rows, nb01, ne00, ne01);
  if (!w) return NS_E_CUDA;
  cudaStream_t st = default_stream();
  if (!io_reserve(&g_io.act, &g_io.act_elems, (size_t)ne11 * ne00) || !io_reserve(&g_io.out, &g_io.out_elems, (size_t)ne11 * ne01)) {
    ns_set_error("device staging allocation failed");
    return NS_E_CUDA;
  }
  NS_CUDA_TRY(cudaMemcpyAsync(g_io.act, src1, (size_t)ne11 * ne00 * 4, cudaMemcpyHostToDevice, st));
  if (int rc = ns_mul_mat(w, g_io.act, ne00, g_io.out, ne01, ne11, nullptr, nullptr, 0, nullptr, st)) return rc;
  NS_CUDA_TRY(cudaMemcpyAsync(dst, g_io.out, (size_t)ne11 * ne01 * 4, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  return NS_OK;
}
extern "C" int ns_mul_mat_q4_0_f32_host(const void* src0_rows, size_t nb01, const float* src1, float* dst, int ne00, int ne01,
                                        int ne11) {
  return ggml_mul_mat_host(GG_Q4_0, src0_rows, nb01, src1, dst, ne00, ne01, ne11);
}
extern "C" int ns_mul_mat_q6_K_f32_host(const void* src0_rows, size_t nb01, const float* src1, float* dst, int ne00, int ne01,
                                        int ne11) {
  return ggml_mul_mat_host(GG_Q6_K, src0_rows, nb01, src1, dst, ne00, ne01, ne11);
}
extern "C" int ns_mul_mat_q8_0_f32_host(const void* src0_rows, size_t nb01, const float* src1, float* dst, int ne00, int ne01,
                                        int ne11) {
  return ggml_mul_mat_host(GG_Q8_0, src0_rows, nb01, src1, dst, ne00, ne01, ne11);
}
// ne_compute_forward_mul_mat_id_q_f32 (ne_layers.c:7345-7498) on host buffers: expert_rows[e] = dst->opt[e]->data (Q4_0 rows of
// pitch nb01), ids = ids->data with ids_stride = ids->nb[1] / 4 int32 per token, id = dst->op_params[0]
extern "C" int ns_mul_mat_id_q4_0_f32_host(const void* const* expert_rows, int n_as, size_t nb01, const int32_t* ids, int ids_stride,
                                           int id, const float* src1, float* dst, int ne00, int ne01, int ne11) {
  if (int rc = ns_ensure_device()) return rc;
  if (!expert_rows || !ids || !src1 || !dst || n_as < 1 || n_as > 256 || ne00 % 32 != 0 || ne01 <= 0 || ne11 <= 0) {
    ns_set_error("ggml host mul_mat_id: invalid arguments");
    return NS_E_INVALID;
  }
  std::vector<const ns_weight*> ws((size_t)n_as, nullptr);
  for (int e = 0; e < n_as; ++e) {
    if (!expert_rows[e]) return NS_E_INVALID;
    ws[(size_t)e] = ggml_cached_weight(GG_Q4_0, expert_rows[e], nb01, ne00, ne01);
    if (!ws[(size_t)e]) return NS_E_CUDA;
  }
  cudaStream_t st = default_stream();
  if (!io_reserve(&g_io.act, &g_io.act_elems, (size_t)ne11 * ne00) || !io_reserve(&g_io.out, &g_io.out_elems, (size_t)ne11 * ne01)) {
    ns_set_error("device staging allocation failed");
    return NS_E_CUDA;
  }
  NS_CUDA_TRY(cudaMemcpyAsync(g_io.act, src1, (size_t)ne11 * ne00 * 4, cudaMemcpyHostToDevice, st));
  if (int rc = ns_mul_mat_id(ws.data(), n_as, ids, ids_stride, id, 0, g_io.act, ne00, g_io.out, ne01, ne11, 0, st)) return rc;
  NS_CUDA_TRY(cudaMemcpyAsync(dst, g_io.out, (size_t)ne11 * ne01 * 4, cudaMemcpyDeviceToHost, st));
  NS_CUDA_TRY(cudaStreamSynchronize(st));
  return NS_OK;
}

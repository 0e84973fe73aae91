// Library-wide state of libicaf_b200: version, thread-local error string, device properties.
#include <atomic>
#include <cstdlib>
#include <cstring>

#include "icaf_internal.cuh"

namespace icaf {

static thread_local char g_err[512] = "";

int set_error(int code, const char* msg) {
  snprintf(g_err, sizeof(g_err), "%s", msg);
  return code;
}
int set_cuda_error(cudaError_t e, const char* where) {
  snprintf(g_err, sizeof(g_err), "%s: %s (%s)", where, cudaGetErrorString(e), cudaGetErrorName(e));
  return ICAF_ERR_CUDA;
}
bool pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("ICAF_PDL");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0;
}
int current_device() {
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  return dev;
}
int sm_count_cached() {
  static int sms[kMaxDevices] = {0};
  const int dev = current_device();
  if (dev < 0 || dev >= kMaxDevices) return 148;
  if (sms[dev] <= 0) {
    int n = 0;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 148;
    sms[dev] = n;
  }
  return sms[dev];
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// 256-byte L2 promotion pulls the neighbouring 128-byte line along with every miss: right for dense rows (the neighbour
// is the next K block or the next pixel of the same box), wrong for a channel slice of a wider buffer whose last line
// is followed by channels this tensor does not own (ncu: 2x DRAM reads on the 64-of-128-channel C3 inputs).
static CUtensorMapL2promotion l2_promotion(uint64_t row_bytes, uint64_t pitch_bytes) {
  return (pitch_bytes > row_bytes && (row_bytes % 256) != 0) ? CU_TENSOR_MAP_L2_PROMOTION_L2_128B : CU_TENSOR_MAP_L2_PROMOTION_L2_256B;
}

static std::atomic<long long> g_launches{0};
void count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
long long launches_so_far() { return g_launches.load(std::memory_order_relaxed); }

// The one cuTensorMapEncodeTiled call behind the encoders below: fp16, no interleave, zero fill out of bounds.  Staged rows
// are box[0] halfs wide and the swizzle span equals the row (64 / 32 / 16 halfs -> 128 / 64 / 32 B); the L2 promotion
// follows the innermost row and its pitch (strides[0]).
static int encode_tmap(CUtensorMap* out, const void* base, cuuint32_t rank, const cuuint64_t* dims, const cuuint64_t* strides,
                       const cuuint32_t* box, const cuuint32_t* estr) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return set_error(ICAF_ERR_CUDA, "cuTensorMapEncodeTiled entry point not available");
  const CUtensorMapSwizzle swz = box[0] >= 64 ? CU_TENSOR_MAP_SWIZZLE_128B : (box[0] == 32 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, rank, const_cast<void*>(base), dims, strides, box, estr,
                  CU_TENSOR_MAP_INTERLEAVE_NONE, swz, l2_promotion(dims[0] * 2, strides[0]), CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char msg[512];      // room for four dimensions of 64-bit sizes and pitches
    int n = snprintf(msg, sizeof(msg), "cuTensorMapEncodeTiled(%ud, size/pitch/box/step per dim:", rank);
    for (cuuint32_t i = 0; i < rank; ++i)
      n += snprintf(msg + n, sizeof(msg) - n, " %llu/%lluB/%u/%u", (unsigned long long)dims[i], i ? (unsigned long long)strides[i - 1] : 2ull,
                    box[i], estr[i]);
    snprintf(msg + n, sizeof(msg) - n, ") failed: %d", int(r));
    return set_error(ICAF_ERR_CUDA, msg);
  }
  return ICAF_OK;
}

int encode_tmap_2d(CUtensorMap* out, const void* base, uint64_t inner, uint64_t rows, uint64_t row_pitch_bytes,
                   uint32_t box_inner, uint32_t box_rows) {
  const cuuint64_t dims[2] = {inner, rows};
  const cuuint64_t strides[1] = {row_pitch_bytes};
  const cuuint32_t box[2] = {box_inner, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return encode_tmap(out, base, 2, dims, strides, box, estr);
}

int encode_tmap_3d(CUtensorMap* out, const void* base, const uint64_t (&dims)[3], uint64_t pitch1_bytes, uint64_t pitch2_bytes,
                   const uint32_t (&box)[3]) {
  const cuuint64_t gdims[3] = {dims[0], dims[1], dims[2]};
  const cuuint64_t strides[2] = {pitch1_bytes, pitch2_bytes};
  const cuuint32_t gbox[3] = {box[0], box[1], box[2]};
  const cuuint32_t estr[3] = {1, 1, 1};
  return encode_tmap(out, base, 3, gdims, strides, gbox, estr);
}

int encode_tmap_nhwc(CUtensorMap* out, const void* base, int C, int W, int H, int B, int64_t ld, uint32_t box_c,
                     uint32_t box_w, uint32_t box_h, uint32_t sw, uint32_t sh) {
  const cuuint64_t dims[4] = {cuuint64_t(C), cuuint64_t(W), cuuint64_t(H), cuuint64_t(B)};
  const cuuint64_t strides[3] = {cuuint64_t(ld) * 2, cuuint64_t(ld) * 2 * W, cuuint64_t(ld) * 2 * W * H};
  const cuuint32_t box[4] = {box_c, box_w, box_h, 1};
  const cuuint32_t estr[4] = {1, sw, sh, 1};
  return encode_tmap(out, base, 4, dims, strides, box, estr);
}

}  // namespace icaf

extern "C" int icaf_version(void) { return 100; }   // 0.1.0
extern "C" const char* icaf_last_error(void) { return icaf::g_err; }
extern "C" long long icaf_kernel_launches(void) { return icaf::launches_so_far(); }
extern "C" int icaf_sm_count(void) {
  int dev = 0, sms = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return -1;
  return sms;
}

// Device-side offset added to every dropout seed (read by the kernels at run time): a captured CUDA graph of the training step
// keeps its host-side seeds, so the caller bumps this counter on the device between replays to draw fresh masks.
static const uint32_t* g_seed_offset = nullptr;
namespace icaf { const uint32_t* seed_offset_ptr() { return g_seed_offset; } }
extern "C" int icaf_set_seed_offset(const void* device_u32) {
  g_seed_offset = (const uint32_t*)device_u32;
  return ICAF_OK;
}


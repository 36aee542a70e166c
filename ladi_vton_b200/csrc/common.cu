// Error channel + TMA tensor-map encoding (driver entry point fetched through the runtime: no -lcuda link dependency).
#include "common.h"

#include <stdarg.h>

#include <atomic>
#include <stdlib.h>
#include <string.h>

static thread_local char g_err[512] = "";

void ladi_set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

extern "C" const char* ladi_last_error(void) { return g_err; }

// kernels launched (or recorded into a CUDA graph being captured) by this process through the library, whichever entry point issued them --
// an op-level call is 1-3 launches, ladi_unet_forward ~400.  bench.py's `gpu_launches` is a difference of this counter.
static std::atomic<long long> g_launches{0};
void ladi_count_launch() { g_launches.fetch_add(1, std::memory_order_relaxed); }
extern "C" long long ladi_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }
extern "C" int ladi_abi_version(void) { return 2; }

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || p == nullptr) return nullptr;
  fn = reinterpret_cast<EncodeTiledFn>(p);
  return fn;
}

static int encode_tmap(CUtensorMapDataType dtype, CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                       const uint64_t* strides_bytes, const uint32_t* box, int swizzle_bytes) {
  EncodeTiledFn enc = get_encode();
  if (!enc) {
    ladi_set_error("cuTensorMapEncodeTiled unavailable (no CUDA driver?)");
    return LADI_ERR_CUDA;
  }
  if ((reinterpret_cast<uintptr_t>(base) & 15) != 0) {
    ladi_set_error("tensor base %p not 16-byte aligned", base);
    return LADI_ERR_INVALID;
  }
  cuuint64_t d[5], s[5];
  cuuint32_t b[5], e[5];
  for (int i = 0; i < rank; ++i) {
    d[i] = dims[i];
    b[i] = box[i];
    e[i] = 1;
    if (i + 1 < rank) {
      s[i] = strides_bytes[i];
      if (s[i] % 16 != 0) {
        ladi_set_error("tensor stride %llu (dim %d) not a multiple of 16 bytes", (unsigned long long)s[i], i + 1);
        return LADI_ERR_INVALID;
      }
    }
  }
  CUresult r = enc(out, dtype, (cuuint32_t)rank, const_cast<void*>(base), d, s, b, e,
                   CU_TENSOR_MAP_INTERLEAVE_NONE, swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                   CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    ladi_set_error("cuTensorMapEncodeTiled failed (%d): rank=%d dims=[%llu,%llu,%llu,%llu] box=[%u,%u,%u,%u] stride1=%llu", (int)r,
                   rank, (unsigned long long)d[0], (unsigned long long)(rank > 1 ? d[1] : 0),
                   (unsigned long long)(rank > 2 ? d[2] : 0), (unsigned long long)(rank > 3 ? d[3] : 0), b[0], rank > 1 ? b[1] : 0,
                   rank > 2 ? b[2] : 0, rank > 3 ? b[3] : 0, (unsigned long long)(rank > 1 ? s[0] : 0));
    return LADI_ERR_CUDA;
  }
  return LADI_OK;
}

int ladi_encode_tmap_bf16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                          const uint32_t* box, int swizzle_bytes) {
  return encode_tmap(CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, out, base, rank, dims, strides_bytes, box, swizzle_bytes);
}

int ladi_encode_tmap_f32(CUtensorMap* out, const void* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes,
                         const uint32_t* box) {
  return encode_tmap(CU_TENSOR_MAP_DATA_TYPE_FLOAT32, out, base, rank, dims, strides_bytes, box, 128);
}

int ladi_num_sms() {
  static int sms = 0;
  if (sms == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0)
      sms = 132;
  }
  return sms;
}

int ladi_pdl_enabled() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("LADI_PDL");
    v = (e != nullptr && e[0] == '0') ? 0 : 1;
  }
  return v;
}

int ladi_conv_pair_default() {
  static int v = -1;
  if (v < 0) {
    const char* e = getenv("LADI_CONV_2CTA");
    v = (e != nullptr && e[0] == '1') ? 1 : 0;  // off unless LADI_CONV_2CTA=1 (A/B timing)
  }
  return v;
}

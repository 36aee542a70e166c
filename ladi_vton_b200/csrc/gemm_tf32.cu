// TF32 tensor-core GEMM of the fp32 metric networks (metrics.py, precision="tf32"): out[M, c_off : c_off + N] = relu?(A[M, K] W[N, K]^T + bias),
// every operand fp32, accumulation fp32.  This is the precision cuDNN runs clean-fid's and torchmetrics' fp32 convolutions in on Ampere and
// Hopper (torch.backends.cudnn.allow_tf32 defaults to True).
//
// A CTA owns a 128 x BN output tile (BN 64 or 128).  Warp 0 is the TMA producer: 128-byte-swizzled [rows][32 fp32] tiles of A and W
// (BK = 32: one 128-byte row per operand row) into a ring of shared-memory stages guarded by full / empty mbarriers; TMA zero-fills the
// columns past K and the rows past M and N.  Warpgroups 1 and 2 consume, each owning 64 rows of the tile: they round the stage's
// operands to TF32 in place (cvt.rna.tf32.f32, round to nearest with ties away from zero -- the tensor core itself would drop the low 13
// mantissa bits, a truncation biased towards zero), then issue wgmma.m64nBNk8.f32.tf32.tf32 from shared memory, both operands K-major.
// Every output element is summed by one thread in K order, so two runs give the same bits.
#include "common.h"
#include "ptx.cuh"

namespace {

// D (+)= A[smem] * B[smem]^T, both K-major, TF32 operands, fp32 accumulators (fragment layout as in wgmma.cuh)
template <int N> struct WgmmaTf32;

template <> struct WgmmaTf32<64> {
  __device__ __forceinline__ static void ss(float (&d)[32], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};

template <> struct WgmmaTf32<128> {
  __device__ __forceinline__ static void ss(float (&d)[64], uint64_t a, uint64_t b, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(a), "l"(b), "r"(accumulate));
  }
};

constexpr int TF_BM = 128, TF_BK = 32, TF_STAGES = 4, TF_THREADS = 384;
constexpr int TF_A_BYTES = TF_BM * TF_BK * 4;
template <int BN> constexpr int tf_smem_bytes() { return 1024 + TF_STAGES * (TF_A_BYTES + BN * TF_BK * 4) + 2 * 8 * TF_STAGES; }

__device__ __forceinline__ uint32_t tf32_rna(uint32_t bits) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(__uint_as_float(bits)));
  return r;
}

// rounds `chunks` 16-byte chunks from shared address `base` to TF32 in place, chunk i by thread i % nthreads
__device__ __forceinline__ void round_tf32_smem(uint32_t base, int chunks, int t, int nthreads) {
  for (int i = t; i < chunks; i += nthreads) {
    uint4 v = ptx::ld_shared_v4(base + 16 * i);
    v.x = tf32_rna(v.x); v.y = tf32_rna(v.y); v.z = tf32_rna(v.z); v.w = tf32_rna(v.w);
    ptx::st_shared_v4(base + 16 * i, v);
  }
}

template <int BN>
__global__ void __launch_bounds__(TF_THREADS, 1)
gemm_tf32_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmW, int m, int n, int k,
                 const float* __restrict__ bias, int relu, float* __restrict__ out, int out_pitch) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int B_BYTES = BN * TF_BK * 4;
  uint8_t* sA = smem;
  uint8_t* sB = sA + TF_STAGES * TF_A_BYTES;
  const uint32_t full0 = ptx::smem_u32(sB + TF_STAGES * B_BYTES), empty0 = full0 + 8 * TF_STAGES;
  const int wg = threadIdx.x >> 7;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * TF_BM;
  const int nkb = (k + TF_BK - 1) / TF_BK;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmA);
    ptx::prefetch_tmap(&tmW);
    for (int s = 0; s < TF_STAGES; ++s) {
      ptx::mbar_init(full0 + 8 * s, 1);
      ptx::mbar_init(empty0 + 8 * s, 2);  // one arrival per consumer warpgroup
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::pdl_wait();

  if (wg == 0) {
    // ------------------------------------------------------------------------ producer: warp 0, all lanes in the loop, one issues
    if (threadIdx.x < 32) {
      uint32_t stage = 0, phase = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        ptx::mbar_wait(empty0 + 8 * stage, phase ^ 1);
        const uint32_t fb = full0 + 8 * stage;
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(fb, TF_A_BYTES + B_BYTES);  // the full boxes: zero-filled elements count
          ptx::tma_load_2d(&tmA, ptx::smem_u32(sA + stage * TF_A_BYTES), fb, kb * TF_BK, m0);
          ptx::tma_load_2d(&tmW, ptx::smem_u32(sB + stage * B_BYTES), fb, kb * TF_BK, n0);
        }
        __syncwarp();
        if (++stage == (uint32_t)TF_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    return;
  }

  // -------------------------------------------------------------------------- consumers
  const int cw = wg - 1, t = threadIdx.x & 127;  // rows [64 cw, 64 cw + 64) of the tile
  const bool signaller = t == 0;
  uint32_t stage = 0, phase = 0, prev = 0;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int kb = 0; kb < nkb; ++kb) {
    ptx::mbar_wait(full0 + 8 * stage, phase);
    const uint32_t a_s = ptx::smem_u32(sA + stage * TF_A_BYTES + cw * (TF_A_BYTES / 2)), b_s = ptx::smem_u32(sB + stage * B_BYTES);
    // this warpgroup's 64 rows of A, and half of the W tile each
    round_tf32_smem(a_s, TF_A_BYTES / 2 / 16, t, 128);
    round_tf32_smem(b_s, B_BYTES / 16, threadIdx.x - 128, 256);
    ptx::fence_proxy_async_smem();        // the generic-proxy stores are visible to wgmma's reads
    ptx::named_barrier_sync(1, 256);      // ... and both warpgroups have rounded their part of W
    const uint64_t adesc = ptx::smem_desc_sw128(a_s), bdesc = ptx::smem_desc_sw128(b_s);
    ptx::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < TF_BK / 8; ++kk) WgmmaTf32<BN>::ss(acc, adesc + 2 * kk, bdesc + 2 * kk, (kb | kk) != 0);  // 32 bytes per k8
    ptx::wgmma_commit();
    if (kb > 0) {
      ptx::wgmma_wait<1>();  // the MMAs of the previous K block have read their stage
      if (signaller) ptx::mbar_arrive(empty0 + 8 * prev);
    }
    prev = stage;
    if (++stage == (uint32_t)TF_STAGES) { stage = 0; phase ^= 1; }
  }
  ptx::wgmma_wait<0>();
  ptx::reg_fence(acc);
  if (signaller) ptx::mbar_arrive(empty0 + 8 * prev);  // no producer waits on it; keeps the ring's accounting whole
  ptx::pdl_trigger();

  // -------------------------------------------------------------------------- epilogue from the accumulator fragment
  const int lane = t & 31, q = lane & 3;
  const int r0 = m0 + 64 * cw + 16 * (t >> 5) + (lane >> 2);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    const int col = n0 + 8 * j + 2 * q;
    if (col >= n) continue;  // n is even: a pair is wholly inside or outside
    const float b0 = bias ? __ldg(bias + col) : 0.f, b1 = bias ? __ldg(bias + col + 1) : 0.f;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int row = r0 + 8 * h;
      if (row >= m) continue;
      float v0 = acc[4 * j + 2 * h] + b0, v1 = acc[4 * j + 2 * h + 1] + b1;
      if (relu) { v0 = fmaxf(v0, 0.f); v1 = fmaxf(v1, 0.f); }
      *reinterpret_cast<float2*>(out + (long long)row * out_pitch + col) = make_float2(v0, v1);
    }
  }
}

template <int BN>
int launch_tf32(const float* a, int m, int k, int a_pitch, const float* w, int n, int w_pitch, const float* bias, int relu, float* out,
                int out_pitch, cudaStream_t stream) {
  static bool attr_set = false;
  if (!attr_set) {
    LADI_CUDA(cudaFuncSetAttribute(gemm_tf32_kernel<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, tf_smem_bytes<BN>()));
    attr_set = true;
  }
  CUtensorMap tmA, tmW;
  const uint64_t da[2] = {(uint64_t)k, (uint64_t)m}, sa[1] = {(uint64_t)a_pitch * 4};
  const uint64_t dw[2] = {(uint64_t)k, (uint64_t)n}, sw[1] = {(uint64_t)w_pitch * 4};
  const uint32_t ba[2] = {TF_BK, TF_BM}, bw[2] = {TF_BK, BN};
  int rc = ladi_encode_tmap_f32(&tmA, a, 2, da, sa, ba);
  if (rc != LADI_OK) return rc;
  rc = ladi_encode_tmap_f32(&tmW, w, 2, dw, sw, bw);
  if (rc != LADI_OK) return rc;
  const dim3 grid((n + BN - 1) / BN, (m + TF_BM - 1) / TF_BM);
  LADI_CUDA(ladi_launch(gemm_tf32_kernel<BN>, grid, dim3(TF_THREADS), tf_smem_bytes<BN>(), stream, tmA, tmW, m, n, k, bias, relu, out,
                        out_pitch));
  return LADI_OK;
}

bool aligned_to(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

}  // namespace

extern "C" int ladi_gemm_tf32(const float* a, int m, int k, int a_pitch, const float* w, int n, int w_pitch, const float* bias, int relu,
                              float* out, int out_pitch, int c_off, void* stream) {
  LADI_CHECK(a && w && out && m > 0 && k > 0 && n > 0, "gemm_tf32: bad extent (m %d, k %d, n %d)", m, k, n);
  LADI_CHECK(relu == 0 || relu == 1, "gemm_tf32: relu must be 0 or 1");
  LADI_CHECK(a_pitch >= k && a_pitch % 4 == 0, "gemm_tf32: a_pitch %d must be >= k and a multiple of 4", a_pitch);
  LADI_CHECK(w_pitch >= k && w_pitch % 4 == 0, "gemm_tf32: w_pitch %d must be >= k and a multiple of 4", w_pitch);
  LADI_CHECK(n % 4 == 0 && c_off >= 0 && c_off % 4 == 0 && out_pitch % 4 == 0 && out_pitch >= c_off + n,
             "gemm_tf32: n %d, c_off %d and out_pitch %d must be multiples of 4 with c_off + n <= out_pitch", n, c_off, out_pitch);
  LADI_CHECK((m + TF_BM - 1) / TF_BM <= 65535, "gemm_tf32: m %d exceeds 65535 row tiles", m);
  LADI_CHECK(aligned_to(a, 16), "gemm_tf32: a %p must be 16-byte aligned", a);
  LADI_CHECK(aligned_to(w, 16), "gemm_tf32: w %p must be 16-byte aligned", w);
  LADI_CHECK(aligned_to(out, 16), "gemm_tf32: out %p must be 16-byte aligned", out);
  LADI_CHECK(!bias || aligned_to(bias, 4), "gemm_tf32: bias %p must be 4-byte aligned", bias);
  const cudaStream_t s = reinterpret_cast<cudaStream_t>(stream);
  // 128-wide N tiles for the wide Mixed_6/7 outputs (256-448), 64 for the narrow ones (32-192) that a 128 tile would half waste
  if (n >= 256) return launch_tf32<128>(a, m, k, a_pitch, w, n, w_pitch, bias, relu, out + c_off, out_pitch, s);
  return launch_tf32<64>(a, m, k, a_pitch, w, n, w_pitch, bias, relu, out + c_off, out_pitch, s);
}

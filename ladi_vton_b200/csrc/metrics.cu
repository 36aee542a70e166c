// Kernels of the image-quality metrics (ladi_vton_b200/metrics.py, the engine form of the reference's src/utils/val_metrics.py):
// the im2col / pooling glue of the FID Inception-v3 and of the LPIPS AlexNet (their convolutions run on the wgmma GEMMs: convgemm.cu for
// bf16 activations, gemm_tf32.cu for fp32), the LPIPS distance layer, SSIM, and torch-fidelity's TF1-style bilinear resize for the
// Inception Score.  The im2col, pooling and LPIPS kernels are templates on the activation type (bf16 or fp32); a thread moves 16 bytes
// of channels (8 bf16 or 4 fp32).  Every reduction has a fixed order (no floating-point atomics), so two runs give identical bits.
#include "common.h"
#include "ptx.cuh"

namespace {

inline int grid_for(long long total) {
  long long g = (total + 255) / 256;
  const long long cap = (long long)ladi_num_sms() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

// 16 bytes of activations as floats: 8 bf16 or 4 fp32
template <typename T> struct Vec16;
template <> struct Vec16<bf16> {
  static constexpr int N = 8, LOG_N = 3;
  __device__ __forceinline__ static void unpack(uint4 u, float (&f)[8]) {
    f[0] = ptx::bf16_lo(u.x); f[1] = ptx::bf16_hi(u.x); f[2] = ptx::bf16_lo(u.y); f[3] = ptx::bf16_hi(u.y);
    f[4] = ptx::bf16_lo(u.z); f[5] = ptx::bf16_hi(u.z); f[6] = ptx::bf16_lo(u.w); f[7] = ptx::bf16_hi(u.w);
  }
  __device__ __forceinline__ static uint4 pack(const float (&f)[8]) {
    uint4 r;
    r.x = ptx::pack_bf16(f[0], f[1]); r.y = ptx::pack_bf16(f[2], f[3]);
    r.z = ptx::pack_bf16(f[4], f[5]); r.w = ptx::pack_bf16(f[6], f[7]);
    return r;
  }
};
template <> struct Vec16<float> {
  static constexpr int N = 4, LOG_N = 2;
  __device__ __forceinline__ static void unpack(uint4 u, float (&f)[4]) {
    f[0] = __uint_as_float(u.x); f[1] = __uint_as_float(u.y); f[2] = __uint_as_float(u.z); f[3] = __uint_as_float(u.w);
  }
  __device__ __forceinline__ static uint4 pack(const float (&f)[4]) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]), __float_as_uint(f[3]));
  }
};
__device__ __forceinline__ float to_f32(bf16 v) { return __bfloat162float(v); }
__device__ __forceinline__ float to_f32(float v) { return v; }
template <typename T> __device__ __forceinline__ T from_f32(float v);
template <> __device__ __forceinline__ bf16 from_f32<bf16>(float v) { return __float2bfloat16(v); }
template <> __device__ __forceinline__ float from_f32<float>(float v) { return v; }

// NHWC [n,h,w,pitch] -> rows [n*oh*ow, k_pad], column (ky*kw + kx)*c + ch, 16 bytes of channels per thread; c % V == 0.
template <typename T>
__global__ void __launch_bounds__(256) im2col_nhwc_kernel(const T* __restrict__ x, int h, int w, int c, int pitch, int kh, int kw, int sh,
                                                          int sw, int ph, int pw, int oh, int ow, long long rows, T* __restrict__ out,
                                                          int k_pad) {
  ptx::pdl_wait();
  constexpr int V = Vec16<T>::N;
  const int groups = k_pad >> Vec16<T>::LOG_N, k_true = kh * kw * c;
  const long long total = rows * groups;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int col = (int)(i % groups) * V;
    const long long r = i / groups;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (col < k_true) {
      const int tap = col / c, ch = col - tap * c, ky = tap / kw, kx = tap - ky * kw;
      const int ox = (int)(r % ow), oy = (int)((r / ow) % oh);
      const long long b = r / ((long long)ow * oh);
      const int iy = oy * sh - ph + ky, ix = ox * sw - pw + kx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w)
        v = __ldg(reinterpret_cast<const uint4*>(x + ((b * h + iy) * w + ix) * pitch + ch));
    }
    *reinterpret_cast<uint4*>(out + r * k_pad + col) = v;
  }
}

// NCHW fp32 pixels -> the same rows; (x - shift[ch]) / scale[ch] is applied to in-image pixels BEFORE the zero padding.
template <typename T>
__global__ void __launch_bounds__(256) im2col_pixels_kernel(const float* __restrict__ x, int c, int h, int w, int kh, int kw, int sh, int sw,
                                                            int ph, int pw, int oh, int ow, long long rows, const float* __restrict__ shift,
                                                            const float* __restrict__ scale, T* __restrict__ out, int k_pad) {
  ptx::pdl_wait();
  const int k_true = kh * kw * c;
  const long long total = rows * k_pad;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int col = (int)(i % k_pad);
    const long long r = i / k_pad;
    float v = 0.f;
    if (col < k_true) {
      const int tap = col / c, ch = col - tap * c, ky = tap / kw, kx = tap - ky * kw;
      const int ox = (int)(r % ow), oy = (int)((r / ow) % oh);
      const long long b = r / ((long long)ow * oh);
      const int iy = oy * sh - ph + ky, ix = ox * sw - pw + kx;
      if (iy >= 0 && iy < h && ix >= 0 && ix < w) v = (__ldg(x + ((b * c + ch) * h + iy) * w + ix) - __ldg(shift + ch)) / __ldg(scale + ch);
    }
    out[i] = from_f32<T>(v);
  }
}

// torch max_pool2d / avg_pool2d (ceil_mode=False) on NHWC, 16 bytes of channels per thread, output into channels [c_off, c_off + c) of
// `out` [n, oh, ow, out_pitch].  Average: fp32 sum in window order, divided by the window size counted as torch does.
template <typename T>
__global__ void __launch_bounds__(256) pool2d_kernel(const T* __restrict__ x, int h, int w, int c, int pitch, int k, int s, int p, int mode,
                                                     int oh, int ow, long long pixels, T* __restrict__ out, int out_pitch, int c_off) {
  ptx::pdl_wait();
  constexpr int V = Vec16<T>::N;
  const int nv = c >> Vec16<T>::LOG_N;
  const long long total = pixels * nv;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int v = (int)(i % nv);
    const long long px = i / nv;
    const int ox = (int)(px % ow), oy = (int)((px / ow) % oh);
    const long long b = px / ((long long)ow * oh);
    int y0 = oy * s - p, x0 = ox * s - p;
    int y1 = min(y0 + k, h + p), x1 = min(x0 + k, w + p);
    const int padded = (y1 - y0) * (x1 - x0);
    y0 = max(y0, 0); x0 = max(x0, 0); y1 = min(y1, h); x1 = min(x1, w);
    float acc[V];
#pragma unroll
    for (int j = 0; j < V; ++j) acc[j] = mode == LADI_POOL_MAX ? -INFINITY : 0.f;
    for (int yy = y0; yy < y1; ++yy)
      for (int xx = x0; xx < x1; ++xx) {
        float f[V];
        Vec16<T>::unpack(__ldg(reinterpret_cast<const uint4*>(x + ((b * h + yy) * w + xx) * pitch + v * V)), f);
#pragma unroll
        for (int j = 0; j < V; ++j) acc[j] = mode == LADI_POOL_MAX ? fmaxf(acc[j], f[j]) : acc[j] + f[j];
      }
    if (mode != LADI_POOL_MAX) {
      const float inv = 1.f / (float)(mode == LADI_POOL_AVG ? padded : (y1 - y0) * (x1 - x0));
#pragma unroll
      for (int j = 0; j < V; ++j) acc[j] *= inv;
    }
    *reinterpret_cast<uint4*>(out + px * out_pitch + c_off + v * V) = Vec16<T>::pack(acc);
  }
}

// adaptive_avg_pool2d(x, 1).flatten(1): out fp32 [n, out_pitch], one thread per (image, channel), pixels summed in order.
template <typename T>
__global__ void __launch_bounds__(256) global_avg_kernel(const T* __restrict__ x, int n, int hw, int c, int pitch, float* __restrict__ out,
                                                         int out_pitch) {
  ptx::pdl_wait();
  const long long total = (long long)n * c;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ch = (int)(i % c);
    const long long b = i / c;
    const T* p = x + b * hw * pitch + ch;
    float acc = 0.f;
    for (int q = 0; q < hw; ++q) acc += to_f32(p[(long long)q * pitch]);
    out[b * out_pitch + ch] = acc / (float)hw;
  }
}

// One LPIPS layer (lpips.LPIPS.forward, version 0.1): per pixel na = a / (|a| + 1e-10), nb likewise, d = sum_c lin[c] (na - nb)^2;
// acc[b] += mean over pixels of d.  One block per image; warp w takes pixels w, w + 16, ...; warps combined in index order.
constexpr int LPIPS_WARPS = 16;
template <typename T>
__global__ void __launch_bounds__(LPIPS_WARPS * 32) lpips_layer_kernel(const T* __restrict__ fa, const T* __restrict__ fb, int hw, int c,
                                                                       int pitch, const float* __restrict__ lin, float* __restrict__ acc) {
  ptx::pdl_wait();
  __shared__ float part[LPIPS_WARPS];
  const int b = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const T* A = fa + (long long)b * hw * pitch;
  const T* B = fb + (long long)b * hw * pitch;
  float mine = 0.f;
  for (int q = warp; q < hw; q += LPIPS_WARPS) {
    const T* pa = A + (long long)q * pitch;
    const T* pb = B + (long long)q * pitch;
    float sa = 0.f, sb = 0.f;
    for (int ch = lane; ch < c; ch += 32) {
      const float a = to_f32(pa[ch]), bb = to_f32(pb[ch]);
      sa = fmaf(a, a, sa);
      sb = fmaf(bb, bb, sb);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      sa += __shfl_xor_sync(0xffffffffu, sa, o);
      sb += __shfl_xor_sync(0xffffffffu, sb, o);
    }
    const float ra = 1.f / (sqrtf(sa) + 1e-10f), rb = 1.f / (sqrtf(sb) + 1e-10f);
    float d = 0.f;
    for (int ch = lane; ch < c; ch += 32) {
      const float t = to_f32(pa[ch]) * ra - to_f32(pb[ch]) * rb;
      d = fmaf(__ldg(lin + ch), t * t, d);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
    mine += d;
  }
  if (lane == 0) part[warp] = mine;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int i = 0; i < LPIPS_WARPS; ++i) t += part[i];
    acc[b] += t / (float)hw;
  }
}

// SSIM (torchmetrics StructuralSimilarityIndexMeasure, gaussian 11 x 11, sigma 1.5): one 16 x 16 tile of valid positions (window fully
// inside the image) per block, all channels; separable filtering through shared memory; the block's sum goes to partial[b][tile].
constexpr int SSIM_T = 16, SSIM_K = 11, SSIM_S = SSIM_T + SSIM_K - 1;
__global__ void __launch_bounds__(SSIM_T * SSIM_T) ssim_tile_kernel(const float* __restrict__ x, const float* __restrict__ y, int c, int h, int w,
                                                                    float* __restrict__ partial) {
  ptx::pdl_wait();
  __shared__ float g[SSIM_K];
  __shared__ float sx[SSIM_S][SSIM_S], sy[SSIM_S][SSIM_S];
  __shared__ float hs[5][SSIM_S][SSIM_T];
  __shared__ float red[SSIM_T * SSIM_T];
  const int tx = threadIdx.x, ty = threadIdx.y, t = ty * SSIM_T + tx;
  const int b = blockIdx.z, x0 = blockIdx.x * SSIM_T, y0 = blockIdx.y * SSIM_T;
  const int vh = h - SSIM_K + 1, vw = w - SSIM_K + 1;
  if (t == 0) {
    float s = 0.f;
    for (int k = 0; k < SSIM_K; ++k) {
      const float d = ((float)k - 5.f) / 1.5f;
      g[k] = expf(-0.5f * d * d);
      s += g[k];
    }
    for (int k = 0; k < SSIM_K; ++k) g[k] /= s;
  }
  const float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
  float mine = 0.f;
  for (int ch = 0; ch < c; ++ch) {
    __syncthreads();
    const float* X = x + ((long long)b * c + ch) * h * w;
    const float* Y = y + ((long long)b * c + ch) * h * w;
    for (int i = t; i < SSIM_S * SSIM_S; i += SSIM_T * SSIM_T) {
      const int r = i / SSIM_S, q = i - r * SSIM_S, gy = y0 + r, gx = x0 + q;
      const bool in = gy < h && gx < w;
      sx[r][q] = in ? __ldg(X + (long long)gy * w + gx) : 0.f;
      sy[r][q] = in ? __ldg(Y + (long long)gy * w + gx) : 0.f;
    }
    __syncthreads();
    for (int r = ty; r < SSIM_S; r += SSIM_T) {
      float m0 = 0.f, m1 = 0.f, m2 = 0.f, m3 = 0.f, m4 = 0.f;
#pragma unroll
      for (int k = 0; k < SSIM_K; ++k) {
        const float a = sx[r][tx + k], bb = sy[r][tx + k], gk = g[k];
        m0 = fmaf(gk, a, m0);
        m1 = fmaf(gk, bb, m1);
        m2 = fmaf(gk, a * a, m2);
        m3 = fmaf(gk, bb * bb, m3);
        m4 = fmaf(gk, a * bb, m4);
      }
      hs[0][r][tx] = m0; hs[1][r][tx] = m1; hs[2][r][tx] = m2; hs[3][r][tx] = m3; hs[4][r][tx] = m4;
    }
    __syncthreads();
    if (y0 + ty < vh && x0 + tx < vw) {
      float m[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < SSIM_K; ++k)
#pragma unroll
        for (int q = 0; q < 5; ++q) m[q] = fmaf(g[k], hs[q][ty + k][tx], m[q]);
      const float mxx = m[0] * m[0], myy = m[1] * m[1], mxy = m[0] * m[1];
      const float vx = m[2] - mxx, vy = m[3] - myy, cxy = m[4] - mxy;
      mine += ((2.f * mxy + C1) * (2.f * cxy + C2)) / ((mxx + myy + C1) * (vx + vy + C2));
    }
  }
  red[t] = mine;
  __syncthreads();
  for (int o = SSIM_T * SSIM_T / 2; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) partial[(long long)b * gridDim.x * gridDim.y + blockIdx.y * gridDim.x + blockIdx.x] = red[0];
}

// second pass: out[b] = (sum of the image's tile partials, fixed tree order) / (c * valid positions)
__global__ void __launch_bounds__(256) ssim_reduce_kernel(const float* __restrict__ partial, int tiles, float inv_count, float* __restrict__ out) {
  ptx::pdl_wait();
  __shared__ float red[256];
  const int b = blockIdx.x, t = threadIdx.x;
  float s = 0.f;
  for (int i = t; i < tiles; i += 256) s += partial[(long long)b * tiles + i];
  red[t] = s;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  if (t == 0) out[b] = red[0] * inv_count;
}

// torch-fidelity's TF1 bilinear resize of (x * 255).byte() (torchmetrics InceptionScore, normalize=True): source coordinate
// o * (in / out) with no half-pixel offset, upper neighbour clamped to the edge; NCHW fp32 in [0, 1] -> NCHW fp32 in [0, 255].
__global__ void __launch_bounds__(256) resize_tf1_kernel(const float* __restrict__ x, int h, int w, int oh, int ow, long long planes,
                                                         float* __restrict__ out) {
  ptx::pdl_wait();
  const float sy = (float)h / (float)oh, sx = (float)w / (float)ow;
  const long long total = planes * oh * ow;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ox = (int)(i % ow), oy = (int)((i / ow) % oh);
    const long long pl = i / ((long long)ow * oh);
    const float fy = (float)oy * sy, fx = (float)ox * sx;
    const int iy0 = min((int)floorf(fy), h - 1), ix0 = min((int)floorf(fx), w - 1);
    const int iy1 = min(iy0 + 1, h - 1), ix1 = min(ix0 + 1, w - 1);
    const float ly = fy - (float)iy0, lx = fx - (float)ix0;
    const float* P = x + pl * h * w;
    auto px = [&](int yy, int xx) { return truncf(fminf(fmaxf(__fmul_rn(__ldg(P + (long long)yy * w + xx), 255.f), 0.f), 255.f)); };
    const float tl = px(iy0, ix0), tr = px(iy0, ix1), bl = px(iy1, ix0), br = px(iy1, ix1);
    const float top = tl + (tr - tl) * lx, bot = bl + (br - bl) * lx;
    out[i] = top + (bot - top) * ly;
  }
}

// Mean absolute difference of two fp32 row-pitched tensors (nn.L1Loss of the TPS trainer's validation and of its VGG loss):
// pass 1, block k sums |a - b| over the V-wide column groups k*256 + t, k*256 + t + gridDim*256, ... in thread order, then a fixed tree
// over its 256 threads -> partial[k]; pass 2, one block sums the partials in the same fixed tree and adds weight * (sum / count) to
// *acc.  The grid depends on the shape only, so two runs on any device give the same bits.  Pitch padding is never read.
constexpr int L1_THREADS = 256;
__device__ __forceinline__ float block_sum_fixed(float v, float* red) {
  const int t = threadIdx.x;
  red[t] = v;
  __syncthreads();
  for (int o = L1_THREADS / 2; o > 0; o >>= 1) {
    if (t < o) red[t] += red[t + o];
    __syncthreads();
  }
  return red[0];
}
template <int V>
__global__ void __launch_bounds__(L1_THREADS) l1_partial_kernel(const float* __restrict__ a, long long a_pitch, const float* __restrict__ b,
                                                                long long b_pitch, int groups_per_row, long long groups,
                                                                float* __restrict__ partial) {
  ptx::pdl_wait();
  __shared__ float red[L1_THREADS];
  float s = 0.f;
  for (long long i = (long long)blockIdx.x * L1_THREADS + threadIdx.x; i < groups; i += (long long)gridDim.x * L1_THREADS) {
    const long long r = i / groups_per_row;
    const int col = (int)(i - r * groups_per_row) * V;
    if constexpr (V == 4) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(a + r * a_pitch + col));
      const float4 y = __ldg(reinterpret_cast<const float4*>(b + r * b_pitch + col));
      s += fabsf(x.x - y.x);
      s += fabsf(x.y - y.y);
      s += fabsf(x.z - y.z);
      s += fabsf(x.w - y.w);
    } else {
      s += fabsf(__ldg(a + r * a_pitch + col) - __ldg(b + r * b_pitch + col));
    }
  }
  const float t = block_sum_fixed(s, red);
  if (threadIdx.x == 0) partial[blockIdx.x] = t;
}
__global__ void __launch_bounds__(L1_THREADS) l1_final_kernel(const float* __restrict__ partial, int blocks, double count, float weight,
                                                              float* __restrict__ acc) {
  ptx::pdl_wait();
  __shared__ float red[L1_THREADS];
  float s = 0.f;
  for (int i = threadIdx.x; i < blocks; i += L1_THREADS) s += partial[i];
  const float t = block_sum_fixed(s, red);
  if (threadIdx.x == 0) *acc += weight * (float)((double)t / count);
}

}  // namespace

static bool aligned_to(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

#define STREAM reinterpret_cast<cudaStream_t>(stream)

extern "C" int ladi_im2col_bf16(const void* x, int x_is_f32_nchw, int n, int c, int h, int w, int pitch, int kh, int kw, int sh, int sw, int ph,
                                int pw, const float* shift, const float* scale, void* out, int k_pad, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h > 0 && w > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 && ph >= 0 && pw >= 0, "im2col: bad extent");
  const int oh = (h + 2 * ph - kh) / sh + 1, ow = (w + 2 * pw - kw) / sw + 1;
  LADI_CHECK(h + 2 * ph >= kh && w + 2 * pw >= kw && oh > 0 && ow > 0, "im2col: window larger than the padded image");
  LADI_CHECK(k_pad % 8 == 0 && k_pad >= kh * kw * c, "im2col: k_pad must be a multiple of 8 and >= kh*kw*c");
  const long long rows = (long long)n * oh * ow;
  if (x_is_f32_nchw) {
    LADI_CHECK(shift && scale, "im2col: the pixel form needs shift and scale");
    LADI_CHECK(aligned_to(x, 4), "im2col: x %p must be 4-byte aligned (fp32 pixels)", x);
    LADI_CHECK(aligned_to(shift, 4), "im2col: shift %p must be 4-byte aligned", shift);
    LADI_CHECK(aligned_to(scale, 4), "im2col: scale %p must be 4-byte aligned", scale);
    LADI_CHECK(aligned_to(out, 2), "im2col: out %p must be 2-byte aligned", out);
    LADI_CUDA(ladi_launch(im2col_pixels_kernel<bf16>, dim3(grid_for(rows * k_pad)), dim3(256), 0, STREAM, (const float*)x, c, h, w, kh, kw, sh, sw, ph,
                          pw, oh, ow, rows, shift, scale, (bf16*)out, k_pad));
  } else {
    LADI_CHECK(!shift && !scale, "im2col: shift / scale apply to the fp32 pixel form only");
    LADI_CHECK(c % 8 == 0 && pitch % 8 == 0 && pitch >= c, "im2col: C and pitch must be multiples of 8");
    LADI_CHECK(aligned_to(x, 16), "im2col: x %p must be 16-byte aligned", x);
    LADI_CHECK(aligned_to(out, 16), "im2col: out %p must be 16-byte aligned", out);
    LADI_CUDA(ladi_launch(im2col_nhwc_kernel<bf16>, dim3(grid_for(rows * (k_pad / 8))), dim3(256), 0, STREAM, (const bf16*)x, h, w, c, pitch, kh, kw, sh,
                          sw, ph, pw, oh, ow, rows, (bf16*)out, k_pad));
  }
  return LADI_OK;
}

extern "C" int ladi_pool2d_bf16(const void* x, int n, int h, int w, int c, int x_pitch, int k, int s, int p, int mode, void* out, int out_pitch,
                                int c_off, void* stream) {
  LADI_CHECK(x && out && n > 0 && h > 0 && w > 0 && c > 0, "pool2d: bad extent");
  LADI_CHECK(c % 8 == 0 && x_pitch % 8 == 0 && x_pitch >= c, "pool2d: C and pitch must be multiples of 8");
  if (mode == LADI_POOL_GLOBAL_AVG_F32) {
    LADI_CHECK(out_pitch >= c_off + c, "pool2d: channel window outside the output pitch");
    LADI_CHECK(aligned_to(x, 2), "pool2d: x %p must be 2-byte aligned", x);
    LADI_CHECK(aligned_to(out, 4), "pool2d: out %p must be 4-byte aligned (fp32 features)", out);
    LADI_CUDA(ladi_launch(global_avg_kernel<bf16>, dim3(grid_for((long long)n * c)), dim3(256), 0, STREAM, (const bf16*)x, n, h * w, c, x_pitch,
                          (float*)out + c_off, out_pitch));
    return LADI_OK;
  }
  LADI_CHECK(mode == LADI_POOL_MAX || mode == LADI_POOL_AVG || mode == LADI_POOL_AVG_EXCLUDE_PAD, "pool2d: unknown mode %d", mode);
  LADI_CHECK(k > 0 && s > 0 && p >= 0 && 2 * p <= k && h + 2 * p >= k && w + 2 * p >= k, "pool2d: bad window (k %d, s %d, p %d)", k, s, p);
  LADI_CHECK(out_pitch % 8 == 0 && c_off % 8 == 0 && out_pitch >= c_off + c, "pool2d: output pitch / channel offset must be multiples of 8");
  LADI_CHECK(aligned_to(x, 16), "pool2d: x %p must be 16-byte aligned", x);
  LADI_CHECK(aligned_to(out, 16), "pool2d: out %p must be 16-byte aligned", out);
  const int oh = (h + 2 * p - k) / s + 1, ow = (w + 2 * p - k) / s + 1;
  const long long pixels = (long long)n * oh * ow;
  LADI_CUDA(ladi_launch(pool2d_kernel<bf16>, dim3(grid_for(pixels * (c / 8))), dim3(256), 0, STREAM, (const bf16*)x, h, w, c, x_pitch, k, s, p, mode, oh,
                        ow, pixels, (bf16*)out, out_pitch, c_off));
  return LADI_OK;
}

extern "C" int ladi_lpips_layer(const void* fa, const void* fb, int n, int h, int w, int c, int pitch, const float* lin, float* acc, void* stream) {
  LADI_CHECK(fa && fb && lin && acc && n > 0 && h > 0 && w > 0 && c > 0 && pitch >= c, "lpips_layer: bad extent");
  LADI_CHECK(aligned_to(fa, 2), "lpips_layer: fa %p must be 2-byte aligned", fa);
  LADI_CHECK(aligned_to(fb, 2), "lpips_layer: fb %p must be 2-byte aligned", fb);
  LADI_CHECK(aligned_to(lin, 4), "lpips_layer: lin %p must be 4-byte aligned", lin);
  LADI_CHECK(aligned_to(acc, 4), "lpips_layer: acc %p must be 4-byte aligned", acc);
  LADI_CUDA(ladi_launch(lpips_layer_kernel<bf16>, dim3(n), dim3(LPIPS_WARPS * 32), 0, STREAM, (const bf16*)fa, (const bf16*)fb, h * w, c, pitch, lin, acc));
  return LADI_OK;
}

extern "C" int ladi_im2col_f32(const float* x, int x_is_nchw_pixels, int n, int c, int h, int w, int pitch, int kh, int kw, int sh, int sw,
                               int ph, int pw, const float* shift, const float* scale, float* out, int k_pad, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h > 0 && w > 0 && kh > 0 && kw > 0 && sh > 0 && sw > 0 && ph >= 0 && pw >= 0,
             "im2col_f32: bad extent");
  const int oh = (h + 2 * ph - kh) / sh + 1, ow = (w + 2 * pw - kw) / sw + 1;
  LADI_CHECK(h + 2 * ph >= kh && w + 2 * pw >= kw && oh > 0 && ow > 0, "im2col_f32: window larger than the padded image");
  LADI_CHECK(k_pad % 4 == 0 && k_pad >= kh * kw * c, "im2col_f32: k_pad must be a multiple of 4 and >= kh*kw*c");
  const long long rows = (long long)n * oh * ow;
  if (x_is_nchw_pixels) {
    LADI_CHECK(shift && scale, "im2col_f32: the pixel form needs shift and scale");
    LADI_CHECK(aligned_to(x, 4), "im2col_f32: x %p must be 4-byte aligned", x);
    LADI_CHECK(aligned_to(shift, 4), "im2col_f32: shift %p must be 4-byte aligned", shift);
    LADI_CHECK(aligned_to(scale, 4), "im2col_f32: scale %p must be 4-byte aligned", scale);
    LADI_CHECK(aligned_to(out, 4), "im2col_f32: out %p must be 4-byte aligned", out);
    LADI_CUDA(ladi_launch(im2col_pixels_kernel<float>, dim3(grid_for(rows * k_pad)), dim3(256), 0, STREAM, x, c, h, w, kh, kw, sh, sw, ph, pw,
                          oh, ow, rows, shift, scale, out, k_pad));
  } else {
    LADI_CHECK(!shift && !scale, "im2col_f32: shift / scale apply to the pixel form only");
    LADI_CHECK(c % 4 == 0 && pitch % 4 == 0 && pitch >= c, "im2col_f32: C and pitch must be multiples of 4");
    LADI_CHECK(aligned_to(x, 16), "im2col_f32: x %p must be 16-byte aligned", x);
    LADI_CHECK(aligned_to(out, 16), "im2col_f32: out %p must be 16-byte aligned", out);
    LADI_CUDA(ladi_launch(im2col_nhwc_kernel<float>, dim3(grid_for(rows * (k_pad / 4))), dim3(256), 0, STREAM, x, h, w, c, pitch, kh, kw, sh, sw,
                          ph, pw, oh, ow, rows, out, k_pad));
  }
  return LADI_OK;
}

extern "C" int ladi_pool2d_f32(const float* x, int n, int h, int w, int c, int x_pitch, int k, int s, int p, int mode, float* out, int out_pitch,
                               int c_off, void* stream) {
  LADI_CHECK(x && out && n > 0 && h > 0 && w > 0 && c > 0, "pool2d_f32: bad extent");
  LADI_CHECK(c % 4 == 0 && x_pitch % 4 == 0 && x_pitch >= c, "pool2d_f32: C and pitch must be multiples of 4");
  if (mode == LADI_POOL_GLOBAL_AVG_F32) {
    LADI_CHECK(out_pitch >= c_off + c, "pool2d_f32: channel window outside the output pitch");
    LADI_CHECK(aligned_to(x, 4), "pool2d_f32: x %p must be 4-byte aligned", x);
    LADI_CHECK(aligned_to(out, 4), "pool2d_f32: out %p must be 4-byte aligned", out);
    LADI_CUDA(ladi_launch(global_avg_kernel<float>, dim3(grid_for((long long)n * c)), dim3(256), 0, STREAM, x, n, h * w, c, x_pitch, out + c_off,
                          out_pitch));
    return LADI_OK;
  }
  LADI_CHECK(mode == LADI_POOL_MAX || mode == LADI_POOL_AVG || mode == LADI_POOL_AVG_EXCLUDE_PAD, "pool2d_f32: unknown mode %d", mode);
  LADI_CHECK(k > 0 && s > 0 && p >= 0 && 2 * p <= k && h + 2 * p >= k && w + 2 * p >= k, "pool2d_f32: bad window (k %d, s %d, p %d)", k, s, p);
  LADI_CHECK(out_pitch % 4 == 0 && c_off % 4 == 0 && out_pitch >= c_off + c, "pool2d_f32: output pitch / channel offset must be multiples of 4");
  LADI_CHECK(aligned_to(x, 16), "pool2d_f32: x %p must be 16-byte aligned", x);
  LADI_CHECK(aligned_to(out, 16), "pool2d_f32: out %p must be 16-byte aligned", out);
  const int oh = (h + 2 * p - k) / s + 1, ow = (w + 2 * p - k) / s + 1;
  const long long pixels = (long long)n * oh * ow;
  LADI_CUDA(ladi_launch(pool2d_kernel<float>, dim3(grid_for(pixels * (c / 4))), dim3(256), 0, STREAM, x, h, w, c, x_pitch, k, s, p, mode, oh, ow,
                        pixels, out, out_pitch, c_off));
  return LADI_OK;
}

extern "C" int ladi_lpips_layer_f32(const float* fa, const float* fb, int n, int h, int w, int c, int pitch, const float* lin, float* acc,
                                    void* stream) {
  LADI_CHECK(fa && fb && lin && acc && n > 0 && h > 0 && w > 0 && c > 0 && pitch >= c, "lpips_layer_f32: bad extent");
  LADI_CHECK(aligned_to(fa, 4), "lpips_layer_f32: fa %p must be 4-byte aligned", fa);
  LADI_CHECK(aligned_to(fb, 4), "lpips_layer_f32: fb %p must be 4-byte aligned", fb);
  LADI_CHECK(aligned_to(lin, 4), "lpips_layer_f32: lin %p must be 4-byte aligned", lin);
  LADI_CHECK(aligned_to(acc, 4), "lpips_layer_f32: acc %p must be 4-byte aligned", acc);
  LADI_CUDA(ladi_launch(lpips_layer_kernel<float>, dim3(n), dim3(LPIPS_WARPS * 32), 0, STREAM, fa, fb, h * w, c, pitch, lin, acc));
  return LADI_OK;
}

extern "C" int ladi_ssim_partials(int h, int w) {
  if (h < SSIM_K || w < SSIM_K) return -1;
  return ((h - SSIM_K + 1 + SSIM_T - 1) / SSIM_T) * ((w - SSIM_K + 1 + SSIM_T - 1) / SSIM_T);
}

extern "C" int ladi_ssim_f32(const float* x, const float* y, int n, int c, int h, int w, float* ws, float* out, void* stream) {
  LADI_CHECK(x && y && ws && out && n > 0 && c > 0, "ssim: bad arguments");
  LADI_CHECK(h >= SSIM_K && w >= SSIM_K, "ssim: images must be at least 11 x 11 (got %d x %d)", h, w);
  LADI_CHECK(n <= 65535, "ssim: n %d exceeds 65535 images per call (one grid.z slice per image)", n);
  LADI_CHECK(aligned_to(x, 4), "ssim: x %p must be 4-byte aligned", x);
  LADI_CHECK(aligned_to(y, 4), "ssim: y %p must be 4-byte aligned", y);
  LADI_CHECK(aligned_to(ws, 4), "ssim: ws %p must be 4-byte aligned", ws);
  LADI_CHECK(aligned_to(out, 4), "ssim: out %p must be 4-byte aligned", out);
  const dim3 grid((w - SSIM_K + 1 + SSIM_T - 1) / SSIM_T, (h - SSIM_K + 1 + SSIM_T - 1) / SSIM_T, n);
  LADI_CUDA(ladi_launch(ssim_tile_kernel, grid, dim3(SSIM_T, SSIM_T), 0, STREAM, x, y, c, h, w, ws));
  const float inv = (float)(1.0 / ((double)c * (h - SSIM_K + 1) * (w - SSIM_K + 1)));
  LADI_CUDA(ladi_launch(ssim_reduce_kernel, dim3(n), dim3(256), 0, STREAM, (const float*)ws, (int)(grid.x * grid.y), inv, out));
  return LADI_OK;
}

extern "C" int ladi_resize_tf1_u8(const float* x, int n, int c, int h, int w, int oh, int ow, float* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h > 0 && w > 0 && oh > 0 && ow > 0, "resize_tf1: bad extent");
  LADI_CHECK(aligned_to(x, 4), "resize_tf1: x %p must be 4-byte aligned", x);
  LADI_CHECK(aligned_to(out, 4), "resize_tf1: out %p must be 4-byte aligned", out);
  LADI_CUDA(ladi_launch(resize_tf1_kernel, dim3(grid_for((long long)n * c * oh * ow)), dim3(256), 0, STREAM, x, h, w, oh, ow, (long long)n * c, out));
  return LADI_OK;
}

extern "C" int ladi_l1_mean_f32(const float* a, int a_pitch, const float* b, int b_pitch, long long rows, int cols, float weight, float* ws,
                                float* acc, void* stream) {
  LADI_CHECK(a && b && ws && acc && rows > 0 && cols > 0 && a_pitch >= cols && b_pitch >= cols, "l1_mean_f32: bad extent");
  LADI_CHECK(aligned_to(a, 4) && aligned_to(b, 4) && aligned_to(ws, 4) && aligned_to(acc, 4), "l1_mean_f32: operands must be 4-byte aligned");
  const bool vec = cols % 4 == 0 && a_pitch % 4 == 0 && b_pitch % 4 == 0 && aligned_to(a, 16) && aligned_to(b, 16);
  const int v = vec ? 4 : 1;
  const long long groups = rows * (cols / v);
  const long long want = (groups + (long long)L1_THREADS * 4 - 1) / ((long long)L1_THREADS * 4);  // ~4 groups per thread
  const int blocks = (int)(want < 1 ? 1 : (want > LADI_L1_MEAN_WS ? LADI_L1_MEAN_WS : want));
  if (vec)
    LADI_CUDA(ladi_launch(l1_partial_kernel<4>, dim3(blocks), dim3(L1_THREADS), 0, STREAM, a, (long long)a_pitch, b, (long long)b_pitch, cols / 4,
                          groups, ws));
  else
    LADI_CUDA(ladi_launch(l1_partial_kernel<1>, dim3(blocks), dim3(L1_THREADS), 0, STREAM, a, (long long)a_pitch, b, (long long)b_pitch, cols,
                          groups, ws));
  LADI_CUDA(ladi_launch(l1_final_kernel, dim3(1), dim3(L1_THREADS), 0, STREAM, (const float*)ws, blocks, (double)rows * cols, weight, acc));
  return LADI_OK;
}

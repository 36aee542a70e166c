// Kernels of the cloth-warping front-end (SURVEY.md section 8(f) row 2): src/models/ConvNet_TPS.py (feature extraction, correlation,
// thin-plate-spline grid), the batch body of src/inference.py:236-266 (antialiased resizes, grid_sample) and the refinement U-Net of
// src/models/UNet.py + unet_parts.py.  All convolutions / the regression linear run on the wgmma implicit-GEMM kernel (convgemm.cu);
// these are the HBM-bound pieces around them.  NHWC bf16 activations, fp32 geometry (control points, grids, sampling coordinates).
#include "common.h"
#include "ptx.cuh"

namespace {

// ---- torch's antialiased separable "bilinear" (aten upsample_bilinear2d_aa, align_corners=False): triangle filter whose support
// grows with the down-scale factor; weights renormalised at the borders.  Returns first tap, tap count and fills w[] (<= MAXT taps).
constexpr int AA_MAXT = 12;  // support * 2 + 1 taps: down-scale factors up to 5
struct AATaps {
  int first, count;
  float w[AA_MAXT];
};
__device__ __forceinline__ void aa_taps(int o, int in_size, int out_size, AATaps& t) {
  const float scale = (float)in_size / (float)out_size;
  const float support = scale >= 1.f ? scale : 1.f;
  const float invscale = scale >= 1.f ? 1.f / scale : 1.f;
  const float center = scale * ((float)o + 0.5f);
  int lo = (int)(center - support + 0.5f);  // truncation toward zero, as the int64 cast in aten
  if (lo < 0) lo = 0;
  int hi = (int)(center + support + 0.5f);
  if (hi > in_size) hi = in_size;
  int cnt = hi - lo;
  if (cnt > AA_MAXT) cnt = AA_MAXT;
  float total = 0.f;
  for (int j = 0; j < cnt; ++j) {
    float x = ((float)(j + lo) - center + 0.5f) * invscale;
    x = fabsf(x);
    const float w = x < 1.f ? 1.f - x : 0.f;
    t.w[j] = w;
    total += w;
  }
  const float inv = total != 0.f ? 1.f / total : 0.f;
  for (int j = 0; j < cnt; ++j) t.w[j] *= inv;
  t.first = lo;
  t.count = cnt;
}

// src/inference.py:265-271: resize((cloth + 1) / 2, (224, 224), antialias=True).clamp(0, 1), then the CLIP image processor's
// (x - mean) / std, fused: x NCHW fp32 in [-1,1] -> out NCHW fp32 [n,c,oh,ow].  The filter is linear, so the (x+1)/2 affine commutes
// with it.  `quantise` != 0 reproduces a processor that round-trips the [0,1] floats through uint8 (floor(v * 255) / 255).
__global__ void __launch_bounds__(256) clip_preprocess_kernel(const float* __restrict__ x, int n, int c, int h, int w, int oh, int ow,
                                                              const float* __restrict__ mean, const float* __restrict__ stdev,
                                                              int quantise, float* __restrict__ out) {
  ptx::pdl_wait();
  const long long total = (long long)n * oh * ow;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ox = (int)(i % ow), oy = (int)((i / ow) % oh), b = (int)(i / ((long long)ow * oh));
    AATaps ty, tx;
    aa_taps(oy, h, oh, ty);
    aa_taps(ox, w, ow, tx);
    for (int ch = 0; ch < c; ++ch) {
      const float* src = x + ((size_t)b * c + ch) * h * w;
      float acc = 0.f;
      for (int a = 0; a < ty.count; ++a) {
        const float* row = src + (size_t)(ty.first + a) * w + tx.first;
        float r = 0.f;
        for (int k = 0; k < tx.count; ++k) r = fmaf(tx.w[k], __ldg(row + k), r);
        acc = fmaf(ty.w[a], r, acc);
      }
      float v = fminf(fmaxf(fmaf(acc, 0.5f, 0.5f), 0.f), 1.f);
      if (quantise) v = floorf(v * 255.f) * (1.f / 255.f);
      out[(((size_t)b * c + ch) * oh + oy) * ow + ox] = (v - __ldg(mean + ch)) / __ldg(stdev + ch);
    }
  }
}

// Where the resampling kernels write output pixel `px` (flat over n*oh*ow) of channel ch: NHWC bf16 channels [c_off, c_off+c) of a
// pitched tensor (the TPS / refinement inputs), or NCHW fp32 [n, c, oh, ow] (the TPS trainer's validation, which reads them unrounded).
template <typename T> struct ResampleOut;
template <> struct ResampleOut<bf16> {
  bf16* p;
  int pitch, c_off;
  __device__ __forceinline__ void put(long long px, int, int ch, int, long long, float v) const {
    p[(size_t)px * pitch + c_off + ch] = __float2bfloat16(v);
  }
};
template <> struct ResampleOut<float> {
  float* p;
  __device__ __forceinline__ void put(long long px, int b, int ch, int c, long long hw, float v) const {
    p[((size_t)b * c + ch) * hw + (px - (long long)b * hw)] = v;
  }
};

// x NCHW fp32 [n,c,h,w] -> out (ResampleOut) [n,oh,ow]   (torchvision resize(..., BILINEAR, antialias=True))
template <typename T>
__global__ void __launch_bounds__(256) resize_aa_kernel(const float* __restrict__ x, int n, int c, int h, int w, int oh, int ow,
                                                        const ResampleOut<T> out) {
  ptx::pdl_wait();
  const long long total = (long long)n * oh * ow;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ox = (int)(i % ow), oy = (int)((i / ow) % oh), b = (int)(i / ((long long)ow * oh));
    AATaps ty, tx;
    aa_taps(oy, h, oh, ty);
    aa_taps(ox, w, ow, tx);
    for (int ch = 0; ch < c; ++ch) {
      const float* src = x + ((size_t)b * c + ch) * h * w;
      float acc = 0.f;
      for (int a = 0; a < ty.count; ++a) {
        const float* row = src + (size_t)(ty.first + a) * w + tx.first;
        float r = 0.f;
        for (int k = 0; k < tx.count; ++k) r = fmaf(tx.w[k], __ldg(row + k), r);
        acc = fmaf(ty.w[a], r, acc);
      }
      out.put(i, b, ch, c, (long long)oh * ow, acc);
    }
  }
}

// NHWC bf16 [n,h,w,c] (pitch) -> [n,h/2,w/2,4c] (pitch), channel (sy*2+sx)*c + ch  <-  pixel (2y+sy, 2x+sx): turns a 4x4 stride-2 pad-1
// convolution into a 3x3 stride-1 pad-1 one over 4c channels (weights re-indexed at load time, see warp.py).
__global__ void __launch_bounds__(256) s2d_kernel(const bf16* __restrict__ x, int n, int h, int w, int c, int x_pitch, bf16* __restrict__ out,
                                                  int out_pitch) {
  ptx::pdl_wait();
  const int oh = h >> 1, ow = w >> 1, oc = 4 * c;
  const long long total = (long long)n * oh * ow * oc;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int k = (int)(i % oc);
    const long long px = i / oc;
    const int ox = (int)(px % ow), oy = (int)((px / ow) % oh), b = (int)(px / ((long long)ow * oh));
    const int s = k / c, ch = k - s * c;
    const int iy = 2 * oy + (s >> 1), ix = 2 * ox + (s & 1);
    out[(size_t)px * out_pitch + k] = x[(((size_t)b * h + iy) * w + ix) * x_pitch + ch];
  }
}

// in place: x[row, c] = x[row, c] * s[c] + t[c]   (eval-mode BatchNorm that FOLLOWS a ReLU, ConvNet_TPS.py:33-42)
__global__ void __launch_bounds__(256) channel_affine_kernel(bf16* __restrict__ x, long long rows, int c, int pitch, const float* __restrict__ s,
                                                             const float* __restrict__ t) {
  ptx::pdl_wait();
  const int nv = c >> 3;
  const long long total = rows * nv;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int v = (int)(i % nv);
    const long long r = i / nv;
    uint4* p = reinterpret_cast<uint4*>(x + (size_t)r * pitch + v * 8);
    uint4 u = *p;
    const float4 s0 = __ldg(reinterpret_cast<const float4*>(s + v * 8)), s1 = __ldg(reinterpret_cast<const float4*>(s + v * 8 + 4));
    const float4 t0 = __ldg(reinterpret_cast<const float4*>(t + v * 8)), t1 = __ldg(reinterpret_cast<const float4*>(t + v * 8 + 4));
    u.x = ptx::pack_bf16(fmaf(ptx::bf16_lo(u.x), s0.x, t0.x), fmaf(ptx::bf16_hi(u.x), s0.y, t0.y));
    u.y = ptx::pack_bf16(fmaf(ptx::bf16_lo(u.y), s0.z, t0.z), fmaf(ptx::bf16_hi(u.y), s0.w, t0.w));
    u.z = ptx::pack_bf16(fmaf(ptx::bf16_lo(u.z), s1.x, t1.x), fmaf(ptx::bf16_hi(u.z), s1.y, t1.y));
    u.w = ptx::pack_bf16(fmaf(ptx::bf16_lo(u.w), s1.z, t1.z), fmaf(ptx::bf16_hi(u.w), s1.w, t1.w));
    *p = u;
  }
}

// FeatureL2Norm (ConvNet_TPS.py:58-66): one warp per pixel, x / sqrt(sum_c x^2 + 1e-6), in place.
__global__ void __launch_bounds__(256) l2norm_kernel(bf16* __restrict__ x, long long rows, int c, int pitch) {
  ptx::pdl_wait();
  const long long row = (long long)blockIdx.x * 8 + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31, nv = c >> 3;
  bf16* p = x + (size_t)row * pitch;
  float ss = 0.f;
  for (int v = lane; v < nv; v += 32) {
    const uint4 u = *reinterpret_cast<const uint4*>(p + v * 8);
    const float f[8] = {ptx::bf16_lo(u.x), ptx::bf16_hi(u.x), ptx::bf16_lo(u.y), ptx::bf16_hi(u.y),
                        ptx::bf16_lo(u.z), ptx::bf16_hi(u.z), ptx::bf16_lo(u.w), ptx::bf16_hi(u.w)};
#pragma unroll
    for (int i = 0; i < 8; ++i) ss = fmaf(f[i], f[i], ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  const float inv = 1.f / sqrtf(ss + 1e-6f);
  for (int v = lane; v < nv; v += 32) {
    uint4 u = *reinterpret_cast<const uint4*>(p + v * 8);
    u.x = ptx::pack_bf16(ptx::bf16_lo(u.x) * inv, ptx::bf16_hi(u.x) * inv);
    u.y = ptx::pack_bf16(ptx::bf16_lo(u.y) * inv, ptx::bf16_hi(u.y) * inv);
    u.z = ptx::pack_bf16(ptx::bf16_lo(u.z) * inv, ptx::bf16_hi(u.z) * inv);
    u.w = ptx::pack_bf16(ptx::bf16_lo(u.w) * inv, ptx::bf16_hi(u.w) * inv);
    *reinterpret_cast<uint4*>(p + v * 8) = u;
  }
}

// FeatureCorrelation (ConvNet_TPS.py:69-81): out[b, yB, xB, xA*h + yA] = sum_c B[b,yB,xB,c] * A[b,yA,xA,c]  (NHWC in, NHWC out with
// h*w channels: exactly the [b, h*w, h, w] tensor of the reference seen channels-last).
__global__ void __launch_bounds__(256) correlation_kernel(const bf16* __restrict__ fa, const bf16* __restrict__ fb, int n, int h, int w, int c,
                                                          bf16* __restrict__ out, int out_pitch) {
  ptx::pdl_wait();
  const int hw = h * w;
  const long long total = (long long)n * hw * hw;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ia = (int)(i % hw);              // = xA * h + yA
    const int ib = (int)((i / hw) % hw);       // = yB * w + xB
    const int b = (int)(i / ((long long)hw * hw));
    const int xa = ia / h, ya = ia - xa * h;
    const uint4* pa = reinterpret_cast<const uint4*>(fa + ((size_t)b * hw + (ya * w + xa)) * c);
    const uint4* pb = reinterpret_cast<const uint4*>(fb + ((size_t)b * hw + ib) * c);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    for (int v = 0; v < (c >> 3); ++v) {
      const uint4 ua = __ldg(pa + v), ub = __ldg(pb + v);
      a0 = fmaf(ptx::bf16_lo(ua.x), ptx::bf16_lo(ub.x), a0); a1 = fmaf(ptx::bf16_hi(ua.x), ptx::bf16_hi(ub.x), a1);
      a2 = fmaf(ptx::bf16_lo(ua.y), ptx::bf16_lo(ub.y), a2); a3 = fmaf(ptx::bf16_hi(ua.y), ptx::bf16_hi(ub.y), a3);
      a0 = fmaf(ptx::bf16_lo(ua.z), ptx::bf16_lo(ub.z), a0); a1 = fmaf(ptx::bf16_hi(ua.z), ptx::bf16_hi(ub.z), a1);
      a2 = fmaf(ptx::bf16_lo(ua.w), ptx::bf16_lo(ub.w), a2); a3 = fmaf(ptx::bf16_hi(ua.w), ptx::bf16_hi(ub.w), a3);
    }
    out[((size_t)b * hw + ib) * out_pitch + ia] = __float2bfloat16((a0 + a1) + (a2 + a3));
  }
}

// BoundedGridLocNet tanh (ConvNet_TPS.py:122) + TPSGridGen.forward (:183-193):  points = tanh(theta);  mapping = inverse_kernel @
// [points; 0 0 0];  grid[b, p, :] = target_coordinate_repr[p, :] @ mapping.   grid = (blocks over points, images).
constexpr int TPS_MAXN = 64;
__global__ void __launch_bounds__(256) tps_grid_kernel(const float* __restrict__ theta, int theta_pitch, const float* __restrict__ inv_kernel,
                                                       const float* __restrict__ repr, int n_ctrl, int n_points, float* __restrict__ points,
                                                       float* __restrict__ grid) {
  ptx::pdl_wait();
  __shared__ float pts[TPS_MAXN * 2], mapping[(TPS_MAXN + 3) * 2];
  const int b = blockIdx.y, t = threadIdx.x, nk = n_ctrl + 3;
  if (t < n_ctrl * 2) {
    const float v = tanhf(theta[(size_t)b * theta_pitch + t]);
    pts[t] = v;
    if (blockIdx.x == 0) points[(size_t)b * n_ctrl * 2 + t] = v;
  }
  __syncthreads();
  if (t < nk * 2) {
    const int r = t >> 1, d = t & 1;
    float acc = 0.f;
    for (int k = 0; k < n_ctrl; ++k) acc = fmaf(inv_kernel[r * nk + k], pts[2 * k + d], acc);  // the 3 padding rows of Y are zero
    mapping[t] = acc;
  }
  __syncthreads();
  const int p = blockIdx.x * 256 + t;
  if (p < n_points) {
    const float* rr = repr + (size_t)p * nk;
    float gx = 0.f, gy = 0.f;
    for (int k = 0; k < nk; ++k) {
      const float r = __ldg(rr + k);
      gx = fmaf(r, mapping[2 * k], gx);
      gy = fmaf(r, mapping[2 * k + 1], gy);
    }
    float* g = grid + ((size_t)b * n_points + p) * 2;
    g[0] = gx;
    g[1] = gy;
  }
}

// src/inference.py:252-257: highres_grid = resize(low_grid, (H, W), BILINEAR, antialias=True) ; warped = grid_sample(cloth, highres_grid,
// mode bilinear, padding_mode 'border', align_corners False).  low_grid [n, gh, gw, 2] fp32, cloth NCHW fp32 [n, c, H, W] (sampled in
// place at its own resolution), out (ResampleOut) [n, H, W].
template <typename T>
__global__ void __launch_bounds__(256) warp_sample_kernel(const float* __restrict__ low_grid, int gh, int gw, const float* __restrict__ cloth, int n,
                                                          int c, int H, int W, const ResampleOut<T> out) {
  ptx::pdl_wait();
  const long long total = (long long)n * H * W;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int ox = (int)(i % W), oy = (int)((i / W) % H), b = (int)(i / ((long long)W * H));
    AATaps ty, tx;
    aa_taps(oy, gh, H, ty);
    aa_taps(ox, gw, W, tx);
    float gx = 0.f, gy = 0.f;
    for (int a = 0; a < ty.count; ++a) {
      const float* row = low_grid + (((size_t)b * gh + ty.first + a) * gw + tx.first) * 2;
      float rx = 0.f, ry = 0.f;
      for (int k = 0; k < tx.count; ++k) {
        rx = fmaf(tx.w[k], __ldg(row + 2 * k), rx);
        ry = fmaf(tx.w[k], __ldg(row + 2 * k + 1), ry);
      }
      gx = fmaf(ty.w[a], rx, gx);
      gy = fmaf(ty.w[a], ry, gy);
    }
    // grid_sample: unnormalise (align_corners=False), clip to the border, bilinear
    float ix = ((gx + 1.f) * (float)W - 1.f) * 0.5f, iy = ((gy + 1.f) * (float)H - 1.f) * 0.5f;
    ix = fminf(fmaxf(ix, 0.f), (float)(W - 1));
    iy = fminf(fmaxf(iy, 0.f), (float)(H - 1));
    const float fx = floorf(ix), fy = floorf(iy);
    const int x0 = (int)fx, y0 = (int)fy, x1 = x0 + 1, y1 = y0 + 1;
    const float wx1 = ix - fx, wy1 = iy - fy, wx0 = 1.f - wx1, wy0 = 1.f - wy1;
    const bool okx = x1 < W, oky = y1 < H;
    for (int ch = 0; ch < c; ++ch) {
      const float* src = cloth + ((size_t)b * c + ch) * H * W;
      float v = wy0 * wx0 * __ldg(src + (size_t)y0 * W + x0);
      if (okx) v = fmaf(wy0 * wx1, __ldg(src + (size_t)y0 * W + x1), v);
      if (oky) v = fmaf(wy1 * wx0, __ldg(src + (size_t)y1 * W + x0), v);
      if (okx && oky) v = fmaf(wy1 * wx1, __ldg(src + (size_t)y1 * W + x1), v);
      out.put(i, b, ch, c, (long long)H * W, v);
    }
  }
}

// NaN-propagating, as nn.MaxPool2d: a NaN anywhere in the window gives NaN (fmaxf would return the other operand)
__device__ __forceinline__ uint32_t max2(uint32_t a, uint32_t b) {
  const __nv_bfloat162 r = __hmax2_nan(*reinterpret_cast<const __nv_bfloat162*>(&a), *reinterpret_cast<const __nv_bfloat162*>(&b));
  return *reinterpret_cast<const uint32_t*>(&r);
}
// nn.MaxPool2d(2) on NHWC bf16 (unet_parts.py:31-34)
__global__ void __launch_bounds__(256) maxpool2_kernel(const bf16* __restrict__ x, int n, int h, int w, int c, bf16* __restrict__ out) {
  ptx::pdl_wait();
  const int oh = h >> 1, ow = w >> 1, nv = c >> 3;
  const long long total = (long long)n * oh * ow * nv;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int v = (int)(i % nv);
    const long long px = i / nv;
    const int ox = (int)(px % ow), oy = (int)((px / ow) % oh), b = (int)(px / ((long long)ow * oh));
    const bf16* p = x + (((size_t)b * h + 2 * oy) * w + 2 * ox) * c + v * 8;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(p)), bq = __ldg(reinterpret_cast<const uint4*>(p + c));
    const uint4 cq = __ldg(reinterpret_cast<const uint4*>(p + (size_t)w * c)), d = __ldg(reinterpret_cast<const uint4*>(p + (size_t)w * c + c));
    uint4 r;
    r.x = max2(max2(a.x, bq.x), max2(cq.x, d.x));
    r.y = max2(max2(a.y, bq.y), max2(cq.y, d.y));
    r.z = max2(max2(a.z, bq.z), max2(cq.z, d.z));
    r.w = max2(max2(a.w, bq.w), max2(cq.w, d.w));
    *reinterpret_cast<uint4*>(out + (size_t)px * c + v * 8) = r;
  }
}

__device__ __forceinline__ uint32_t lerp4(uint32_t a, uint32_t b, uint32_t c, uint32_t d, float w00, float w01, float w10, float w11) {
  const float lo = w00 * ptx::bf16_lo(a) + w01 * ptx::bf16_lo(b) + w10 * ptx::bf16_lo(c) + w11 * ptx::bf16_lo(d);
  const float hi = w00 * ptx::bf16_hi(a) + w01 * ptx::bf16_hi(b) + w10 * ptx::bf16_hi(c) + w11 * ptx::bf16_hi(d);
  return ptx::pack_bf16(lo, hi);
}
// nn.Upsample(scale_factor=2, mode='bilinear', align_corners=True) on NHWC bf16 (unet_parts.py:47)
__global__ void __launch_bounds__(256) upsample2x_ac_kernel(const bf16* __restrict__ x, int n, int h, int w, int c, bf16* __restrict__ out) {
  ptx::pdl_wait();
  const int oh = 2 * h, ow = 2 * w, nv = c >> 3;
  const float sy = oh > 1 ? (float)(h - 1) / (float)(oh - 1) : 0.f, sx = ow > 1 ? (float)(w - 1) / (float)(ow - 1) : 0.f;
  const long long total = (long long)n * oh * ow * nv;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int v = (int)(i % nv);
    const long long px = i / nv;
    const int ox = (int)(px % ow), oy = (int)((px / ow) % oh), b = (int)(px / ((long long)ow * oh));
    const float fy = sy * (float)oy, fx = sx * (float)ox;
    const int y0 = (int)fy, x0 = (int)fx;
    const int y1 = min(y0 + 1, h - 1), x1 = min(x0 + 1, w - 1);
    const float wy = fy - (float)y0, wx = fx - (float)x0;
    const float w00 = (1.f - wy) * (1.f - wx), w01 = (1.f - wy) * wx, w10 = wy * (1.f - wx), w11 = wy * wx;
    const bf16* base = x + (size_t)b * h * w * c + v * 8;
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)y0 * w + x0) * c));
    const uint4 bq = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)y0 * w + x1) * c));
    const uint4 cq = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)y1 * w + x0) * c));
    const uint4 d = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)y1 * w + x1) * c));
    uint4 r;
    r.x = lerp4(a.x, bq.x, cq.x, d.x, w00, w01, w10, w11);
    r.y = lerp4(a.y, bq.y, cq.y, d.y, w00, w01, w10, w11);
    r.z = lerp4(a.z, bq.z, cq.z, d.z, w00, w01, w10, w11);
    r.w = lerp4(a.w, bq.w, cq.w, d.w, w00, w01, w10, w11);
    *reinterpret_cast<uint4*>(out + (size_t)px * c + v * 8) = r;
  }
}

// x NHWC fp32 [n, hw, pitch] (first c channels) -> NCHW fp32 clamped to [lo, hi]   (inference.py:262: warped_cloth.clamp(-1, 1))
__global__ void __launch_bounds__(256) nhwc_to_nchw_clamp_kernel(const float* __restrict__ x, int n, int c, int hw, int pitch, float lo, float hi,
                                                                 float* __restrict__ out) {
  ptx::pdl_wait();
  const long long total = (long long)n * c * hw;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const long long px = i % hw, r = i / hw;
    const int ch = (int)(r % c);
    const long long b = r / c;
    out[i] = ptx::clamp_keep_nan(x[(b * hw + px) * pitch + ch], lo, hi);  // torch.clamp keeps NaN
  }
}

inline int grid_for(long long total) {
  long long g = (total + 255) / 256;
  const long long cap = (long long)ladi_num_sms() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

#define STREAM reinterpret_cast<cudaStream_t>(stream)

extern "C" int ladi_clip_preprocess(const float* x, int n, int c, int h, int w, int oh, int ow, const float* mean, const float* stdev,
                                    int quantise, float* out, void* stream) {
  LADI_CHECK(x && out && mean && stdev && n > 0 && c > 0 && h > 0 && w > 0 && oh > 0 && ow > 0, "clip_preprocess: bad extent");
  LADI_CHECK((float)h / oh <= 5.f && (float)w / ow <= 5.f, "clip_preprocess: down-scale factors above 5 are not supported");
  LADI_CUDA(ladi_launch(clip_preprocess_kernel, dim3(grid_for((long long)n * oh * ow)), dim3(256), 0, STREAM, x, n, c, h, w, oh, ow, mean,
                        stdev, quantise, out));
  return LADI_OK;
}

extern "C" int ladi_resize_aa(const float* x, int n, int c, int h, int w, int oh, int ow, void* out, int out_pitch, int c_off, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h > 0 && w > 0 && oh > 0 && ow > 0, "resize_aa: bad extent");
  LADI_CHECK(out_pitch >= c_off + c, "resize_aa: channel window outside the output pitch");
  LADI_CHECK((float)h / oh <= 5.f && (float)w / ow <= 5.f, "resize_aa: down-scale factors above 5 are not supported");
  LADI_CUDA(ladi_launch(resize_aa_kernel<bf16>, dim3(grid_for((long long)n * oh * ow)), dim3(256), 0, STREAM, x, n, c, h, w, oh, ow,
                        ResampleOut<bf16>{(bf16*)out, out_pitch, c_off}));
  return LADI_OK;
}

extern "C" int ladi_resize_aa_f32(const float* x, int n, int c, int h, int w, int oh, int ow, float* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h > 0 && w > 0 && oh > 0 && ow > 0, "resize_aa_f32: bad extent");
  LADI_CHECK((float)h / oh <= 5.f && (float)w / ow <= 5.f, "resize_aa_f32: down-scale factors above 5 are not supported");
  LADI_CUDA(ladi_launch(resize_aa_kernel<float>, dim3(grid_for((long long)n * oh * ow)), dim3(256), 0, STREAM, x, n, c, h, w, oh, ow,
                        ResampleOut<float>{out}));
  return LADI_OK;
}

extern "C" int ladi_space_to_depth2(const void* x, int n, int h, int w, int c, int x_pitch, void* out, int out_pitch, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h % 2 == 0 && w % 2 == 0 && h > 0 && w > 0, "space_to_depth2: H and W must be even");
  LADI_CHECK(x_pitch >= c && out_pitch >= 4 * c, "space_to_depth2: pitch too small");
  LADI_CUDA(ladi_launch(s2d_kernel, dim3(grid_for((long long)n * (h / 2) * (w / 2) * 4 * c)), dim3(256), 0, STREAM, (const bf16*)x, n, h, w, c,
                        x_pitch, (bf16*)out, out_pitch));
  return LADI_OK;
}

extern "C" int ladi_channel_affine(void* x, long long rows, int c, int pitch, const float* scale, const float* shift, void* stream) {
  LADI_CHECK(x && scale && shift && rows > 0 && c % 8 == 0 && pitch % 8 == 0 && pitch >= c, "channel_affine: C and pitch must be multiples of 8");
  LADI_CHECK(aligned16(x), "channel_affine: x %p must be 16-byte aligned", x);
  LADI_CHECK(aligned16(scale), "channel_affine: scale %p must be 16-byte aligned (read as float4)", scale);
  LADI_CHECK(aligned16(shift), "channel_affine: shift %p must be 16-byte aligned (read as float4)", shift);
  LADI_CUDA(ladi_launch(channel_affine_kernel, dim3(grid_for(rows * (c / 8))), dim3(256), 0, STREAM, (bf16*)x, rows, c, pitch, scale, shift));
  return LADI_OK;
}

extern "C" int ladi_l2norm_channels(void* x, long long rows, int c, int pitch, void* stream) {
  LADI_CHECK(x && rows > 0 && c % 8 == 0 && pitch % 8 == 0 && pitch >= c, "l2norm: C and pitch must be multiples of 8");
  LADI_CHECK(aligned16(x), "l2norm: x %p must be 16-byte aligned", x);
  LADI_CUDA(ladi_launch(l2norm_kernel, dim3((unsigned)((rows + 7) / 8)), dim3(256), 0, STREAM, (bf16*)x, rows, c, pitch));
  return LADI_OK;
}

extern "C" int ladi_feature_correlation(const void* feat_a, const void* feat_b, int n, int h, int w, int c, void* out, int out_pitch,
                                        void* stream) {
  LADI_CHECK(feat_a && feat_b && out && n > 0 && h > 0 && w > 0 && c % 8 == 0, "correlation: C must be a multiple of 8");
  LADI_CHECK(out_pitch >= h * w, "correlation: output pitch below h*w");
  LADI_CHECK(aligned16(feat_a), "correlation: fa %p must be 16-byte aligned", feat_a);
  LADI_CHECK(aligned16(feat_b), "correlation: fb %p must be 16-byte aligned", feat_b);
  LADI_CUDA(ladi_launch(correlation_kernel, dim3(grid_for((long long)n * h * w * h * w)), dim3(256), 0, STREAM, (const bf16*)feat_a,
                        (const bf16*)feat_b, n, h, w, c, (bf16*)out, out_pitch));
  return LADI_OK;
}

extern "C" int ladi_tps_grid(const float* theta, int theta_pitch, const float* inverse_kernel, const float* target_coordinate_repr, int n,
                             int n_ctrl, int n_points, float* points, float* grid, void* stream) {
  LADI_CHECK(theta && inverse_kernel && target_coordinate_repr && points && grid && n > 0 && n_points > 0, "tps_grid: bad arguments");
  LADI_CHECK(n_ctrl > 0 && n_ctrl <= TPS_MAXN && theta_pitch >= 2 * n_ctrl, "tps_grid: 1..64 control points");
  LADI_CHECK(n <= 65535, "tps_grid: n %d exceeds 65535 images per call (one grid.y slice per image)", n);
  LADI_CUDA(ladi_launch(tps_grid_kernel, dim3((n_points + 255) / 256, n), dim3(256), 0, STREAM, theta, theta_pitch, inverse_kernel,
                        target_coordinate_repr, n_ctrl, n_points, points, grid));
  return LADI_OK;
}

extern "C" int ladi_warp_grid_sample(const float* low_grid, int gh, int gw, const float* cloth, int n, int c, int h, int w, void* out,
                                     int out_pitch, int c_off, void* stream) {
  LADI_CHECK(low_grid && cloth && out && n > 0 && c > 0 && gh > 0 && gw > 0 && h > 0 && w > 0, "warp_grid_sample: bad extent");
  LADI_CHECK(out_pitch >= c_off + c, "warp_grid_sample: channel window outside the output pitch");
  LADI_CHECK((float)gh / h <= 5.f && (float)gw / w <= 5.f, "warp_grid_sample: grid down-scale above 5 not supported");
  LADI_CUDA(ladi_launch(warp_sample_kernel<bf16>, dim3(grid_for((long long)n * h * w)), dim3(256), 0, STREAM, low_grid, gh, gw, cloth, n, c, h,
                        w, ResampleOut<bf16>{(bf16*)out, out_pitch, c_off}));
  return LADI_OK;
}

extern "C" int ladi_warp_grid_sample_f32(const float* low_grid, int gh, int gw, const float* cloth, int n, int c, int h, int w, float* out,
                                         void* stream) {
  LADI_CHECK(low_grid && cloth && out && n > 0 && c > 0 && gh > 0 && gw > 0 && h > 0 && w > 0, "warp_grid_sample_f32: bad extent");
  LADI_CHECK((float)gh / h <= 5.f && (float)gw / w <= 5.f, "warp_grid_sample_f32: grid down-scale above 5 not supported");
  LADI_CUDA(ladi_launch(warp_sample_kernel<float>, dim3(grid_for((long long)n * h * w)), dim3(256), 0, STREAM, low_grid, gh, gw, cloth, n, c, h,
                        w, ResampleOut<float>{out}));
  return LADI_OK;
}

extern "C" int ladi_maxpool2_nhwc(const void* x, int n, int h, int w, int c, void* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && h % 2 == 0 && w % 2 == 0 && c % 8 == 0, "maxpool2: even H, W and C %% 8 == 0");
  LADI_CHECK(aligned16(x), "maxpool2: x %p must be 16-byte aligned", x);
  LADI_CHECK(aligned16(out), "maxpool2: out %p must be 16-byte aligned", out);
  LADI_CUDA(ladi_launch(maxpool2_kernel, dim3(grid_for((long long)n * (h / 2) * (w / 2) * (c / 8))), dim3(256), 0, STREAM, (const bf16*)x, n, h, w,
                        c, (bf16*)out));
  return LADI_OK;
}

extern "C" int ladi_upsample2x_bilinear_ac(const void* x, int n, int h, int w, int c, void* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && h > 0 && w > 0 && c % 8 == 0, "upsample2x_bilinear_ac: C %% 8 == 0");
  LADI_CHECK(aligned16(x), "upsample2x_bilinear_ac: x %p must be 16-byte aligned", x);
  LADI_CHECK(aligned16(out), "upsample2x_bilinear_ac: out %p must be 16-byte aligned", out);
  LADI_CUDA(ladi_launch(upsample2x_ac_kernel, dim3(grid_for((long long)n * 4 * h * w * (c / 8))), dim3(256), 0, STREAM, (const bf16*)x, n, h, w, c,
                        (bf16*)out));
  return LADI_OK;
}

extern "C" int ladi_nhwc_f32_to_nchw_clamp(const float* x, int n, int c, int h, int w, int x_pitch, float lo, float hi, float* out,
                                           void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && x_pitch >= c, "nhwc_f32_to_nchw_clamp: bad extent");
  LADI_CUDA(ladi_launch(nhwc_to_nchw_clamp_kernel, dim3(grid_for((long long)n * c * h * w)), dim3(256), 0, STREAM, x, n, c, h * w, x_pitch, lo, hi,
                        out));
  return LADI_OK;
}

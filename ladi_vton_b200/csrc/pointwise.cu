// HBM-bound kernels of the try-on path: GroupNorm (two-source, NHWC), LayerNorm, row softmax, layout conversion, posterior
// sampling, mask/pose resizing, the fused CFG + DDIM step, image clamp.  All loads/stores are 16-byte vectors on the
// contiguous channel dimension (NHWC) so every warp request is fully coalesced.
#include "common.h"
#include "ptx.cuh"

namespace {

__device__ __forceinline__ void unpack8(const uint4& u, float (&f)[8]) {
  f[0] = ptx::bf16_lo(u.x); f[1] = ptx::bf16_hi(u.x); f[2] = ptx::bf16_lo(u.y); f[3] = ptx::bf16_hi(u.y);
  f[4] = ptx::bf16_lo(u.z); f[5] = ptx::bf16_hi(u.z); f[6] = ptx::bf16_lo(u.w); f[7] = ptx::bf16_hi(u.w);
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  return make_uint4(ptx::pack_bf16(f[0], f[1]), ptx::pack_bf16(f[2], f[3]), ptx::pack_bf16(f[4], f[5]), ptx::pack_bf16(f[6], f[7]));
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float tanh_approx(float x) {
  float y;
  asm("tanh.approx.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

constexpr int GN_MAX_GROUPS = 64;
constexpr int GN_MAX_CHUNKS = 64;

__host__ __device__ inline int gn_chunks(int hw) {
  int c = (hw + 63) / 64;
  return c > GN_MAX_CHUNKS ? GN_MAX_CHUNKS : (c < 1 ? 1 : c);
}

// ---- GroupNorm pass 1: per (image, pixel chunk) partial {sum, sum of squares} per group.  Deterministic: per-thread channel
// partials go to shared memory and are folded in a fixed order (no floating-point atomics), so two runs are bit-identical.
constexpr int GN_SLOTS = 2560;  // >= max(channels, 256 threads * 8 channels)
// grid = (pixel chunks, images, group splits): blockIdx.z owns groups [z*gps, (z+1)*gps) i.e. a contiguous channel range, so the
// low-resolution levels (48..192 pixels, 1280..2560 channels) still spread over the whole GPU.
__global__ void __launch_bounds__(256) gn_stats_kernel(const bf16* __restrict__ x0, int c0, int pitch0, const bf16* __restrict__ x1,
                                                       int c1, int pitch1, int hw, int groups, int chunks, float* __restrict__ ws) {
  ptx::pdl_wait();
  __shared__ float ps[GN_SLOTS], pq[GN_SLOTS];  // [pixel lane][channel of this block's range]
  const int n = blockIdx.y, chunk = blockIdx.x, t = threadIdx.x;
  const int Ctot = c0 + c1, cpg = Ctot / groups;
  const int gps = groups / gridDim.z;            // groups per block
  const int cbeg = blockIdx.z * gps * cpg;       // first channel of this block (multiple of 8 by construction)
  const int C = gps * cpg, nv = C >> 3;
  const int per = (hw + chunks - 1) / chunks;
  const int p0 = chunk * per, p1 = min(hw, p0 + per);
  const int lanes_v = nv < 256 ? nv : 256;
  const int k = 256 / lanes_v;
  // The kernel is instruction-issue bound (ncu: 70 % issue-active, 96 % L2 hits), so the streaming loop is written for few integer
  // instructions: one base pointer per thread advanced by a constant byte stride, full batches of 8 loads without predicates, one
  // predicated batch of 4 for the ragged end.
  if (t < lanes_v * k) {
    const int tv = t % lanes_v, tp = t / lanes_v;
    for (int v = tv; v < nv; v += lanes_v) {
      const int ch = cbeg + v * 8;
      const bf16* base;
      int pitch;
      if (ch < c0) { base = x0 + (size_t)n * hw * pitch0 + ch; pitch = pitch0; }
      else { base = x1 + (size_t)n * hw * pitch1 + (ch - c0); pitch = pitch1; }
      float s[8], q[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) s[i] = q[i] = 0.f;
      const uint4* ptr = reinterpret_cast<const uint4*>(base + (size_t)(p0 + tp) * pitch);
      const size_t stride = (size_t)k * pitch / 8;  // in 16-byte units (pitch % 8 == 0)
      int cnt = p1 - p0 - tp;                       // pixels p0+tp, p0+tp+k, ... < p1
      cnt = cnt > 0 ? (cnt + k - 1) / k : 0;
      for (; cnt >= 8; cnt -= 8, ptr += 8 * stride) {
        uint4 u[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) u[j] = __ldg(ptr + j * stride);
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          float f[8];
          unpack8(u[j], f);
#pragma unroll
          for (int i = 0; i < 8; ++i) { s[i] += f[i]; q[i] = fmaf(f[i], f[i], q[i]); }
        }
      }
      for (; cnt > 0; cnt -= 4, ptr += 4 * stride) {
        uint4 u[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) u[j] = j < cnt ? __ldg(ptr + j * stride) : make_uint4(0u, 0u, 0u, 0u);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float f[8];
          unpack8(u[j], f);
#pragma unroll
          for (int i = 0; i < 8; ++i) { s[i] += f[i]; q[i] = fmaf(f[i], f[i], q[i]); }
        }
      }
#pragma unroll
      for (int i = 0; i < 8; ++i) { ps[tp * C + v * 8 + i] = s[i]; pq[tp * C + v * 8 + i] = q[i]; }
    }
  }
  __syncthreads();
  // fold the k * cpg per-thread partials of every group with 8 lanes per group: lane `part` takes channels part, part+8, ... of the
  // group for every pixel lane (no integer division), then a fixed shuffle tree -- deterministic
  const int part = t & 7;
  for (int base = 0; base < gps; base += 32) {  // uniform trip count: the shuffles below need whole warps
    const int gi = base + (t >> 3);
    float s = 0.f, q = 0.f;
    if (gi < gps) {
      for (int l = 0; l < k; ++l) {
        const float* rs = ps + l * C + gi * cpg;
        const float* rq = pq + l * C + gi * cpg;
        for (int c = part; c < cpg; c += 8) { s += rs[c]; q += rq[c]; }
      }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) { s += __shfl_xor_sync(0xffffffffu, s, o); q += __shfl_xor_sync(0xffffffffu, q, o); }
    if (gi < gps && part == 0) {
      float* dst = ws + (((size_t)n * chunks + chunk) * groups + blockIdx.z * gps + gi) * 2;
      dst[0] = s; dst[1] = q;
    }
  }
}

// ---- GroupNorm pass 2: normalise + affine (+SiLU) (+add), writes the concatenated tensor.  Per-channel scale/shift
// (rstd*gamma, beta - mean*rstd*gamma) are tabulated once per block in shared memory, so the streaming loop is one FMA (+SiLU)
// per element with no integer division; the (pixel, vector) walk advances incrementally.
template <bool HAS_ADD>
__global__ void __launch_bounds__(256, 3) gn_apply_kernel(const bf16* __restrict__ x0, int c0, int pitch0, const bf16* __restrict__ x1,
                                                       int c1, int pitch1, int hw, int groups, int chunks, const float* __restrict__ ws,
                                                       const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                       int silu, const bf16* __restrict__ add, int add_pitch, bf16* __restrict__ out,
                                                       int out_pitch, int px_per_block) {
  ptx::pdl_wait();
  __shared__ float smean[GN_MAX_GROUPS], srstd[GN_MAX_GROUPS];
  __shared__ float reds[8][GN_MAX_GROUPS], redq[8][GN_MAX_GROUPS];
  __shared__ __align__(16) float sa[GN_SLOTS], sb[GN_SLOTS];
  const int n = blockIdx.y, t = threadIdx.x;
  const int C = c0 + c1, nv = C >> 3, cpg = C / groups;
  // ---- streaming walk: element e = t, t+256, ... of this block's (pixel, vector) range; NB independent 16-byte loads in flight per
  // thread; the first batch is issued BEFORE the statistics prologue so its latency overlaps the prologue's.  The kernel is
  // instruction-issue bound (ncu), so addresses are strength-reduced: per-source row pointers advance by constant strides and are
  // corrected on the (pixel, vector) wrap instead of being recomputed with 64-bit multiplies.
  constexpr int NB = 8;
  const int p0 = blockIdx.x * px_per_block, p1 = min(hw, p0 + px_per_block);
  const int total = (p1 - p0) * nv;
  const int dv = 256 % nv, dp = 256 / nv;
  struct Cursor {
    int v;
    const bf16 *r0, *r1, *ra;  // row pointers of the current pixel in source 0 / source 1 (pre-offset by -c0) / the add operand
  };
  Cursor lc;
  {
    const int px = p0 + t / nv;
    lc.v = t % nv;
    lc.r0 = x0 + ((size_t)n * hw + px) * pitch0;
    lc.r1 = c1 > 0 ? x1 + ((size_t)n * hw + px) * pitch1 - c0 : lc.r0;
    lc.ra = HAS_ADD ? add + ((size_t)n * hw + px) * add_pitch : nullptr;
  }
  const int step0 = dp * pitch0, step1 = dp * pitch1, stepa = dp * add_pitch;
  auto advance = [&](Cursor& c) {
    c.v += dv; c.r0 += step0; c.r1 += step1;
    if (HAS_ADD) c.ra += stepa;
    if (c.v >= nv) {
      c.v -= nv; c.r0 += pitch0; c.r1 += pitch1;
      if (HAS_ADD) c.ra += add_pitch;
    }
  };
  uint4 u[NB], ad[HAS_ADD ? NB : 1];
  auto load_batch = [&](int e) {
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      if (e + j * 256 < total) {
        const int ch = lc.v * 8;
        u[j] = __ldg(reinterpret_cast<const uint4*>((ch < c0 ? lc.r0 : lc.r1) + ch));
        if (HAS_ADD) ad[HAS_ADD ? j : 0] = __ldg(reinterpret_cast<const uint4*>(lc.ra + ch));
      }
      advance(lc);
    }
  };
  load_batch(t);
  // ---- prologue: fold the per-chunk partials.  `slices` threads per group take interleaved chunks (independent loads in flight), then
  // one thread per group adds the slices in a fixed order -- deterministic, and ~8x shorter than one thread walking all chunks
  const int slices = min(8, 256 / groups);
  {
    const int g = t % groups, sl = t / groups;
    if (sl < slices) {
      float s = 0.f, q = 0.f;
      const float* src = ws + (size_t)n * chunks * groups * 2 + g * 2;
      for (int c = sl; c < chunks; c += slices) { s += src[(size_t)c * groups * 2]; q += src[(size_t)c * groups * 2 + 1]; }
      reds[sl][g] = s; redq[sl][g] = q;
    }
  }
  __syncthreads();
  if (t < groups) {
    float s = 0.f, q = 0.f;
    for (int sl = 0; sl < slices; ++sl) { s += reds[sl][t]; q += redq[sl][t]; }
    const float cnt = (float)hw * (float)cpg;
    const float mean = s / cnt;
    const float var = fmaxf(q / cnt - mean * mean, 0.f);
    smean[t] = mean;
    srstd[t] = rsqrtf(var + eps);
  }
  __syncthreads();
  for (int c = t; c < C; c += 256) {
    const int g = c / cpg;
    const float a = srstd[g] * __ldg(gamma + c);
    sa[c] = a;
    sb[c] = __ldg(beta + c) - smean[g] * a;
  }
  __syncthreads();
  int v = t % nv;  // process cursor (trails the load cursor by one batch)
  bf16* orow = out + ((size_t)n * hw + p0 + t / nv) * out_pitch;
  const int stepo = dp * out_pitch;
  for (int e = t; e < total; e += NB * 256) {
#pragma unroll
    for (int j = 0; j < NB; ++j) {
      if (e + j * 256 < total) {
        const int ch = v * 8;
        float f[8];
        unpack8(u[j], f);
        const float4 a0 = *reinterpret_cast<const float4*>(sa + ch), a1 = *reinterpret_cast<const float4*>(sa + ch + 4);
        const float4 b0 = *reinterpret_cast<const float4*>(sb + ch), b1 = *reinterpret_cast<const float4*>(sb + ch + 4);
        f[0] = fmaf(f[0], a0.x, b0.x); f[1] = fmaf(f[1], a0.y, b0.y); f[2] = fmaf(f[2], a0.z, b0.z); f[3] = fmaf(f[3], a0.w, b0.w);
        f[4] = fmaf(f[4], a1.x, b1.x); f[5] = fmaf(f[5], a1.y, b1.y); f[6] = fmaf(f[6], a1.z, b1.z); f[7] = fmaf(f[7], a1.w, b1.w);
        if (silu) {
#pragma unroll
          for (int i = 0; i < 8; ++i) {  // x * sigmoid(x) = h * (1 + tanh(h)), h = x / 2: ONE MUFU (tanh.approx, rel. error 2^-11,
            const float h = 0.5f * f[i];  // below the bf16 rounding of the result) instead of ex2 + rcp -- the kernel is MUFU/issue bound
            f[i] = fmaf(h, tanh_approx(h), h);
          }
        }
        if (HAS_ADD) {
          float g8[8];
          unpack8(ad[HAS_ADD ? j : 0], g8);
#pragma unroll
          for (int i = 0; i < 8; ++i) f[i] += g8[i];
        }
        *reinterpret_cast<uint4*>(orow + ch) = pack8(f);
      }
      v += dv; orow += stepo;
      if (v >= nv) { v -= nv; orow += out_pitch; }
    }
    if (e + NB * 256 < total) load_batch(e + NB * 256);
  }
}

// ---- LayerNorm: T lanes per row (T = 32/16/8/4), VPL 16-byte vectors per lane, row cached in registers; several rows per warp
// keep every lane busy for the narrow rows (C = 320: 8 lanes x 5 vectors, 4 rows per warp).
template <int VPL>
__global__ void __launch_bounds__(256) layernorm_kernel(const bf16* __restrict__ x, int x_pitch, int rows, int C, int T,
                                                        const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                                        bf16* __restrict__ out, int out_pitch) {
  ptx::pdl_wait();
  const int rows_per_warp = 32 / T;
  const int warp = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const int sub = lane / T, tl = lane % T;
  const int row = warp * rows_per_warp + sub;
  const bool ok = row < rows;
  float f[VPL][8];
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    if (ok) {
      const uint4 u = __ldg(reinterpret_cast<const uint4*>(x + (size_t)row * x_pitch + (tl + T * j) * 8));
      unpack8(u, f[j]);
    } else {
#pragma unroll
      for (int i = 0; i < 8; ++i) f[j][i] = 0.f;
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) s += f[j][i];
  }
  for (int o = T >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float mean = s / (float)C;
  float q = 0.f;
#pragma unroll
  for (int j = 0; j < VPL; ++j)
#pragma unroll
    for (int i = 0; i < 8; ++i) { const float d = f[j][i] - mean; q += d * d; }
  for (int o = T >> 1; o > 0; o >>= 1) q += __shfl_xor_sync(0xffffffffu, q, o);
  const float rstd = rsqrtf(q / (float)C + eps);
  if (!ok) return;
#pragma unroll
  for (int j = 0; j < VPL; ++j) {
    const int c = (tl + T * j) * 8;
    const float4 g0 = __ldg(reinterpret_cast<const float4*>(gamma + c)), g1 = __ldg(reinterpret_cast<const float4*>(gamma + c + 4));
    const float4 b0 = __ldg(reinterpret_cast<const float4*>(beta + c)), b1 = __ldg(reinterpret_cast<const float4*>(beta + c + 4));
    float y[8];
    y[0] = (f[j][0] - mean) * rstd * g0.x + b0.x; y[1] = (f[j][1] - mean) * rstd * g0.y + b0.y;
    y[2] = (f[j][2] - mean) * rstd * g0.z + b0.z; y[3] = (f[j][3] - mean) * rstd * g0.w + b0.w;
    y[4] = (f[j][4] - mean) * rstd * g1.x + b1.x; y[5] = (f[j][5] - mean) * rstd * g1.y + b1.y;
    y[6] = (f[j][6] - mean) * rstd * g1.z + b1.z; y[7] = (f[j][7] - mean) * rstd * g1.w + b1.w;
    *reinterpret_cast<uint4*>(out + (size_t)row * out_pitch + c) = pack8(y);
  }
}

// ---- row softmax fp32 -> bf16
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ s, int cols, int s_pitch, float scale,
                                                           bf16* __restrict__ out, int out_pitch) {
  ptx::pdl_wait();
  __shared__ float red[8];
  const float* row = s + (size_t)blockIdx.x * s_pitch;
  bf16* orow = out + (size_t)blockIdx.x * out_pitch;
  const int t = threadIdx.x;
  float mx = -INFINITY;
  for (int c = t; c < cols; c += 256) mx = fmaxf(mx, row[c]);
  mx = warp_max(mx);
  if ((t & 31) == 0) red[t >> 5] = mx;
  __syncthreads();
  mx = red[0];
  for (int i = 1; i < 8; ++i) mx = fmaxf(mx, red[i]);
  __syncthreads();
  float sum = 0.f;
  for (int c = t; c < cols; c += 256) sum += __expf((row[c] - mx) * scale);
  sum = warp_sum(sum);
  if ((t & 31) == 0) red[t >> 5] = sum;
  __syncthreads();
  sum = 0.f;
  for (int i = 0; i < 8; ++i) sum += red[i];
  const float inv = 1.f / sum;
  for (int c = t; c < cols; c += 256) orow[c] = __float2bfloat16(__expf((row[c] - mx) * scale) * inv);
}

// ---- CLS-row attention of the inversion adapter's CLIP encoder layer: only token 0 of the layer output is consumed
// (src/models/inversion_adapter.py:26), so the query is the CLS row alone; one block per (head, image).
//   q0 [B, heads*hd] (bias included, unscaled), kv [B, T, 2*heads*hd] (K then V), out [B, heads*hd]
constexpr int CLS_WARPS = 4;  // 128 threads; their reduction slots are the kernel's only static shared memory
__global__ void __launch_bounds__(128) cls_attention_kernel(const bf16* __restrict__ q0, int q_pitch, const bf16* __restrict__ kv,
                                                            int kv_pitch, int T, int heads, int hd, float scale, bf16* __restrict__ out,
                                                            int out_pitch) {
  ptx::pdl_wait();
  extern __shared__ float sm[];  // [hd] query, [T] probabilities
  float* sq = sm;
  float* sp = sm + hd;
  __shared__ float red[CLS_WARPS];
  const int h = blockIdx.x, b = blockIdx.y, t = threadIdx.x;
  const int C = heads * hd;
  for (int d = t; d < hd; d += 128) sq[d] = __bfloat162float(q0[(size_t)b * q_pitch + h * hd + d]) * scale;
  __syncthreads();
  const bf16* kb = kv + (size_t)b * T * kv_pitch + h * hd;
  float mx = -INFINITY;
  for (int tok = t; tok < T; tok += 128) {
    const bf16* kr = kb + (size_t)tok * kv_pitch;
    float s = 0.f;
    for (int d = 0; d < hd; d += 2) {
      const __nv_bfloat162 k2 = *reinterpret_cast<const __nv_bfloat162*>(kr + d);
      s += sq[d] * __low2float(k2) + sq[d + 1] * __high2float(k2);
    }
    sp[tok] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if ((t & 31) == 0) red[t >> 5] = mx;
  __syncthreads();
  mx = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  __syncthreads();
  float sum = 0.f;
  for (int tok = t; tok < T; tok += 128) {
    const float e = __expf(sp[tok] - mx);
    sp[tok] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if ((t & 31) == 0) red[t >> 5] = sum;
  __syncthreads();
  const float inv = 1.f / (red[0] + red[1] + red[2] + red[3]);
  const bf16* vb = kb + C;
  for (int d = t; d < hd; d += 128) {
    float acc = 0.f;
    for (int tok = 0; tok < T; ++tok) acc += sp[tok] * __bfloat162float(vb[(size_t)tok * kv_pitch + d]);
    out[(size_t)b * out_pitch + h * hd + d] = __float2bfloat16(acc * inv);
  }
}

__global__ void add_kernel(const uint4* __restrict__ a, const uint4* __restrict__ b, uint4* __restrict__ o, int64_t nvec) {
  ptx::pdl_wait();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < nvec; i += (int64_t)gridDim.x * blockDim.x) {
    float x[8], y[8];
    unpack8(__ldg(a + i), x);
    unpack8(__ldg(b + i), y);
#pragma unroll
    for (int j = 0; j < 8; ++j) x[j] += y[j];
    o[i] = pack8(x);
  }
}

__global__ void upsample2x_kernel(const uint4* __restrict__ x, int n, int h, int w, int cv, uint4* __restrict__ out) {
  ptx::pdl_wait();
  const int64_t total = (int64_t)n * (2 * h) * (2 * w) * cv;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int v = (int)(i % cv);
    int64_t r = i / cv;
    const int ox = (int)(r % (2 * w)); r /= (2 * w);
    const int oy = (int)(r % (2 * h));
    const int b = (int)(r / (2 * h));
    out[i] = __ldg(x + (((int64_t)b * h + (oy >> 1)) * w + (ox >> 1)) * cv + v);
  }
}

// out[b, y, x, c_off + ch] = src[b, ch, y*f, x*f] * scale * (gate ? (gate[b, 0, y*f, x*f] < 0.5) : 1)
// (f > 1: nearest down-sampling, src index = floor(dst * f); gate: `image * (mask < 0.5)` of prepare_mask_and_masked_image)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ x, int n, int c, int h, int w, int f, float scale,
                                    const float* __restrict__ gate, bf16* __restrict__ out, int out_pitch, int c_off) {
  ptx::pdl_wait();
  const int64_t hw = (int64_t)h * w;
  const int64_t total = (int64_t)n * hw * c;
  const int64_t W = (int64_t)w * f, HW = (int64_t)h * f * W;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % c);
    const int64_t r = i / c;  // r = b*hw + px
    const int64_t b = r / hw, px = r % hw;
    const int64_t sp = (px / w) * f * W + (px % w) * f;
    float v = x[(b * c + ch) * HW + sp] * scale;
    if (gate != nullptr && !(gate[b * HW + sp] < 0.5f)) v = 0.f;
    out[r * out_pitch + c_off + ch] = __float2bfloat16(v);
  }
}

__global__ void nhwc_to_nchw_kernel(const void* __restrict__ x, int is_f32, int n, int c, int hw, int x_pitch, int c_off,
                                    float* __restrict__ out) {
  ptx::pdl_wait();
  const int64_t total = (int64_t)n * c * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t px = i % hw;
    const int64_t r = i / hw;
    const int ch = (int)(r % c);
    const int64_t b = r / c;
    const int64_t src = (b * hw + px) * x_pitch + c_off + ch;
    out[i] = is_f32 ? reinterpret_cast<const float*>(x)[src] : __bfloat162float(reinterpret_cast<const bf16*>(x)[src]);
  }
}

__global__ void posterior_kernel(const float* __restrict__ mom, int m_pitch, const float* __restrict__ noise, int n, int cz, int hw,
                                 float scale, float* __restrict__ out) {
  ptx::pdl_wait();
  const int64_t total = (int64_t)n * cz * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t px = i % hw;
    const int64_t r = i / hw;
    const int ch = (int)(r % cz);
    const int64_t b = r / cz;
    const float* m = mom + (b * hw + px) * m_pitch;
    const float mean = m[ch];
    const float logvar = ptx::clamp_keep_nan(m[cz + ch], -30.f, 20.f);  // torch.clamp(logvar, -30, 20): a NaN logvar stays NaN
    out[i] = (mean + expf(0.5f * logvar) * noise[i]) * scale;
  }
}

__global__ void inv_mask_kernel(const float* __restrict__ mask, int n, int H, int W, int f, float* __restrict__ out) {
  ptx::pdl_wait();
  const int h = H / f, w = W / f;
  const int64_t total = (int64_t)n * h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % w);
    const int64_t r = i / w;
    const int y = (int)(r % h);
    const int64_t b = r / h;
    out[i] = 1.f - mask[(b * H + (int64_t)y * f) * W + (int64_t)x * f];  // nearest: src index = floor(dst * f)
  }
}

// F.interpolate(mode="bilinear", align_corners=False), exact /8: src = (dst+0.5)*8-0.5 = 8*dst+3.5 -> taps 8d+3, 8d+4 at 0.5
__global__ void bilinear8_kernel(const float* __restrict__ x, int nc, int H, int W, float* __restrict__ out) {
  ptx::pdl_wait();
  const int h = H / 8, w = W / 8;
  const int64_t total = (int64_t)nc * h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ox = (int)(i % w);
    const int64_t r = i / w;
    const int oy = (int)(r % h);
    const int64_t p = r / h;
    const float* s = x + (p * H + (int64_t)oy * 8 + 3) * W + (int64_t)ox * 8 + 3;
    // same association order as ATen's upsample_bilinear2d: lerp in x on both rows, then lerp in y (weights 0.5/0.5)
    const float top = 0.5f * s[0] + 0.5f * s[1];
    const float bot = 0.5f * s[W] + 0.5f * s[W + 1];
    out[i] = 0.5f * top + 0.5f * bot;
  }
}

__global__ void ddim_cfg_kernel(const float* __restrict__ eps, int eps_pitch, float* __restrict__ lat, bf16* __restrict__ uin,
                                int in_pitch, int B, int hw, int cfg, float guidance, const float* __restrict__ coef, int* step_ptr,
                                int advance, const float* __restrict__ noise) {
  ptx::pdl_wait();
  const int s = step_ptr ? step_ptr[0] : 0;
  const float inv_sa = coef[8 * s], s1a = coef[8 * s + 1], sap = coef[8 * s + 2], s1ap = coef[8 * s + 3], sigma = coef[8 * s + 4];
  const int64_t total = (int64_t)B * 4 * hw;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t px = i % hw;
    const int64_t r = i / hw;
    const int ch = (int)(r % 4);
    const int64_t b = r / 4;
    float e = eps[(b * hw + px) * eps_pitch + ch];
    if (cfg) {
      const float et = eps[((B + b) * hw + px) * eps_pitch + ch];
      e = e + guidance * (et - e);
    }
    const float x = lat[i];
    const float x0 = (x - s1a * e) * inv_sa;
    float xn = sap * x0 + s1ap * e;
    if (noise != nullptr) xn += sigma * noise[i];  // eta > 0: DDIMScheduler.step's variance noise
    lat[i] = xn;
    const bf16 hb = __float2bfloat16(xn);
    uin[(b * hw + px) * in_pitch + ch] = hb;
    if (cfg) uin[((B + b) * hw + px) * in_pitch + ch] = hb;
  }
  if (advance && step_ptr) {
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
      const int ticket = atomicAdd(step_ptr + 1, 1);
      if (ticket == (int)gridDim.x - 1) {
        step_ptr[1] = 0;
        step_ptr[0] = s + 1;
      }
    }
  }
}

// prepare_mask_and_masked_image's range checks and in-place mask binarisation (tryon_pipe.py:630) without a host round trip: the two
// flags are OR-ed into device memory and read by the pipeline together with the result.  NaN compares false, like the reference's
// `x.min() < lo or x.max() > hi`.
__global__ void check_binarise_kernel(const float* __restrict__ image, int64_t n_image, float* __restrict__ mask, int64_t n_mask,
                                      int* __restrict__ flags) {
  ptx::pdl_wait();
  bool bad_i = false, bad_m = false;
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_image; i += stride) {
    const float v = image[i];
    bad_i |= (v < -1.f) | (v > 1.f);
  }
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < n_mask; i += stride) {
    const float v = mask[i];
    bad_m |= (v < 0.f) | (v > 1.f);
    mask[i] = v < 0.5f ? 0.f : (v >= 0.5f ? 1.f : v);  // mask[mask < 0.5] = 0; mask[mask >= 0.5] = 1 (NaN stays)
  }
  if (__any_sync(0xffffffffu, bad_i) && (threadIdx.x & 31) == 0) atomicOr(flags, 1);
  if (__any_sync(0xffffffffu, bad_m) && (threadIdx.x & 31) == 0) atomicOr(flags + 1, 1);
}

__global__ void image_out_kernel(const void* __restrict__ x, int is_f32, int64_t npx, int x_pitch, float* __restrict__ out) {
  ptx::pdl_wait();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npx * 3; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t px = i / 3;
    const int ch = (int)(i % 3);
    const float v = is_f32 ? reinterpret_cast<const float*>(x)[px * x_pitch + ch]
                           : __bfloat162float(reinterpret_cast<const bf16*>(x)[px * x_pitch + ch]);
    out[i] = ptx::clamp_keep_nan(v * 0.5f + 0.5f, 0.f, 1.f);  // (image / 2 + 0.5).clamp(0, 1) keeps NaN
  }
}

// numpy_to_pil of the reference pipeline base class (called at tryon_pipe.py:760): (x * 255).round().astype(uint8) of the clamped
// image, on the device -- the D2H copy shrinks 4x and the host only wraps the bytes in PIL images.  rintf = round-half-to-even = numpy.
// NaN becomes 0 here (numpy's NaN -> uint8 cast is undefined; fmaxf picks the 0).
__global__ void image_out_u8_kernel(const void* __restrict__ x, int is_f32, int64_t npx, int x_pitch, uint8_t* __restrict__ out) {
  ptx::pdl_wait();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npx * 3; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t px = i / 3;
    const int ch = (int)(i % 3);
    const float v = is_f32 ? reinterpret_cast<const float*>(x)[px * x_pitch + ch]
                           : __bfloat162float(reinterpret_cast<const bf16*>(x)[px * x_pitch + ch]);
    const float c = fminf(fmaxf(v * 0.5f + 0.5f, 0.f), 1.f);
    out[i] = (uint8_t)rintf(c * 255.f);
  }
}

// The EMASC trainer's image writer (src/utils/image_from_pipe.py:252-258): `(x + 1) / 2`, then torchvision.utils.save_image's
// `mul(255).add_(0.5).clamp_(0, 255).to(uint8)`.  Each step is its own fp32 rounding, as torch runs them: `(x + 1) * 0.5` equals the
// division by 2 exactly, and __fmul_rn / __fadd_rn keep nvcc from contracting `t * 255 + 0.5` into one FMA, which rounds once and gives
// another byte at near-ties.  The cast truncates.  NaN gives 0 (fmaxf picks the 0), as in image_out_u8_kernel.
__global__ void image_save_u8_kernel(const float* __restrict__ x, int64_t npx, int x_pitch, uint8_t* __restrict__ out) {
  ptx::pdl_wait();
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < npx * 3; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t px = i / 3;
    const int ch = (int)(i % 3);
    const float t = __fmul_rn(__fadd_rn(x[px * x_pitch + ch], 1.f), 0.5f);
    const float u = fminf(fmaxf(__fadd_rn(__fmul_rn(t, 255.f), 0.5f), 0.f), 255.f);
    out[i] = (uint8_t)__float2uint_rz(u);
  }
}

// src/utils/posemap.py:6-35 kpoint_to_heatmap for all key-points of a batch: out[b,k,y,x] = exp(-((x-kx)^2 + (y-ky)^2) / sigma^2) / (max + eps)
// when any coordinate of the key-point is > 0, else 0.  The maximum over the integer grid is attained at the grid point nearest to the
// key-point (clamped into the map), so it has a closed form and the map is written in one pass.
__global__ void pose_heatmap_kernel(const float* __restrict__ kpts, int n_maps, int h, int w, float inv_sigma2, float* __restrict__ out) {
  ptx::pdl_wait();
  const int64_t total = (int64_t)n_maps * h * w;
  for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % w), y = (int)((i / w) % h);
    const int m = (int)(i / ((int64_t)w * h));
    const float kx = __ldg(kpts + 2 * m), ky = __ldg(kpts + 2 * m + 1);
    float v = 0.f;
    if (kx > 0.f || ky > 0.f) {
      const float nx = fminf(fmaxf(rintf(kx), 0.f), (float)(w - 1)), ny = fminf(fmaxf(rintf(ky), 0.f), (float)(h - 1));
      const float dmin = (nx - kx) * (nx - kx) + (ny - ky) * (ny - ky);
      const float d = ((float)x - kx) * ((float)x - kx) + ((float)y - ky) * ((float)y - ky);
      v = expf(-d * inv_sigma2) / (expf(-dmin * inv_sigma2) + 1.1920929e-07f);
    }
    out[i] = v;
  }
}

// diffusers get_timestep_embedding(flip_sin_to_cos=True, downscale_freq_shift=0) -- the input of UNet2DConditionModel.time_embedding (SURVEY App. A.2):
// emb[s, :] = [cos(t_s * f_i), sin(t_s * f_i)], f_i = exp(-ln(10000) * i / half).  Written as a (hi, lo) pair of bf16 columns (hi = bf16(e), lo = bf16(e - hi)) so
// the first linear of the time MLP reads it through the bf16 GEMM with 2^-17 input error: out [n, 2 * kp], hi at [0, c0), lo at [kp, kp + c0), zeros elsewhere.
__global__ void timestep_embed_kernel(const float* __restrict__ timesteps, int n, int c0, int kp, bf16* __restrict__ out) {
  ptx::pdl_wait();
  const int half = c0 / 2;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n * kp; i += gridDim.x * blockDim.x) {
    const int s = i / kp, j = i - s * kp;
    float e = 0.f;
    if (j < c0) {
      const int k = j < half ? j : j - half;
      const float arg = timesteps[s] * expf(-9.210340371976184f * (float)k / (float)half);
      e = j < half ? cosf(arg) : sinf(arg);
    }
    const bf16 hi = __float2bfloat16(e);
    out[(size_t)s * 2 * kp + j] = hi;
    out[(size_t)s * 2 * kp + kp + j] = __float2bfloat16(e - __bfloat162float(hi));
  }
}

inline int grid_for(int64_t total, int block = 256) {
  int64_t g = (total + block - 1) / block;
  const int64_t cap = (int64_t)ladi_num_sms() * 16;
  return (int)(g < 1 ? 1 : (g > cap ? cap : g));
}

}  // namespace

#define STREAM reinterpret_cast<cudaStream_t>(stream)

extern "C" int ladi_groupnorm_chunks(int hw) { return gn_chunks(hw); }

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// Everything the two GroupNorm launches decide, from their arguments and the SM count alone (no pointer is dereferenced, nothing touches
// a device): validation, then the stats grid (pixel chunks x images x group splits) and the apply grid.  ladi_groupnorm_plan reports
// it; ladi_groupnorm_stats / ladi_groupnorm_apply launch it.
static int gn_plan_stats(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups,
                         const void* ws, int sms, ladi_gn_plan& pl) {
  LADI_CHECK(x0 != nullptr && c0 > 0 && c0 % 8 == 0 && pitch0 % 8 == 0 && pitch0 >= c0,
             "groupnorm x0: need non-null, c0 > 0 and a multiple of 8, pitch0 a multiple of 8 and >= c0 (c0 %d, pitch0 %d)", c0, pitch0);
  LADI_CHECK(aligned16(x0), "groupnorm x0 %p must be 16-byte aligned", x0);
  LADI_CHECK(c1 >= 0 && ((x1 == nullptr && c1 == 0) || (x1 != nullptr && c1 % 8 == 0 && pitch1 % 8 == 0 && pitch1 >= c1)),
             "groupnorm x1: need c1 >= 0 (0 when x1 is null) and a multiple of 8, pitch1 a multiple of 8 and >= c1 (c1 %d, pitch1 %d)",
             c1, pitch1);
  LADI_CHECK(c1 == 0 || aligned16(x1), "groupnorm x1 %p must be 16-byte aligned", x1);
  LADI_CHECK(n > 0 && hw > 0, "groupnorm: need n > 0 and hw > 0 (n %d, hw %d)", n, hw);
  LADI_CHECK(ws != nullptr, "groupnorm ws is null");
  LADI_CHECK(groups > 0 && groups <= GN_MAX_GROUPS && (c0 + c1) % groups == 0, "groupnorm: C %% groups != 0 or groups > 64");
  LADI_CHECK(c0 + c1 <= GN_SLOTS, "groupnorm: more than %d channels", GN_SLOTS);
  const int C = c0 + c1;
  pl.chunks = gn_chunks(hw);
  // split the groups over blockIdx.z until the grid covers the GPU twice; each split must own whole groups and whole 16-byte vectors
  int gsplit = 1;
  while (gsplit < 16 && (long)pl.chunks * n * gsplit < 2L * sms && groups % (gsplit * 2) == 0 && (C / (gsplit * 2)) % 8 == 0) gsplit *= 2;
  pl.gsplit = gsplit;
  pl.block_channels = C / gsplit;  // gn_stats_kernel: C = gps * cpg, nv = C / 8, lanes_v, k, per
  pl.lanes_v = pl.block_channels / 8 < 256 ? pl.block_channels / 8 : 256;
  pl.k = 256 / pl.lanes_v;
  pl.px_per_chunk = (hw + pl.chunks - 1) / pl.chunks;
  return LADI_OK;
}

static int gn_plan_apply(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups, const void* ws,
                         const float* gamma, const float* beta, const void* add, int add_pitch, const void* out, int out_pitch, int sms,
                         ladi_gn_plan& pl) {
  if (int e = gn_plan_stats(x0, c0, pitch0, x1, c1, pitch1, n, hw, groups, ws, sms, pl)) return e;
  const int C = c0 + c1;
  LADI_CHECK(gamma != nullptr && beta != nullptr, "groupnorm gamma / beta is null");
  LADI_CHECK(out != nullptr && aligned16(out), "groupnorm out %p must be non-null and 16-byte aligned", out);
  LADI_CHECK(out_pitch % 8 == 0 && out_pitch >= C, "groupnorm out_pitch %d must be a multiple of 8 and >= C (%d)", out_pitch, C);
  LADI_CHECK(add == nullptr || aligned16(add), "groupnorm add %p must be 16-byte aligned", add);
  LADI_CHECK(add == nullptr || (add_pitch % 8 == 0 && add_pitch >= C), "groupnorm add_pitch %d must be a multiple of 8 and >= C (%d)",
             add_pitch, C);
  const int nv = C / 8;
  int ppb = (256 * 16) / nv;  // >= 16 vectors per thread, and few enough blocks that the per-block channel table amortises
  const int target_blocks = (sms * 3 + n - 1) / n;  // 3 resident blocks per SM (launch bounds): the whole grid is one wave
  const int ppb2 = (hw + target_blocks - 1) / target_blocks;
  if (ppb2 > ppb) ppb = ppb2;
  if (ppb < 1) ppb = 1;
  pl.px_per_block = ppb;
  pl.apply_blocks = (hw + ppb - 1) / ppb;
  pl.dv = 256 % nv;  // gn_apply_kernel's cursor step: dp pixels and dv vectors per 256 elements
  pl.dp = 256 / nv;
  pl.slices = 256 / groups < 8 ? 256 / groups : 8;
  return LADI_OK;
}

extern "C" int ladi_groupnorm_plan(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups,
                                   const float* ws, const float* gamma, const float* beta, float eps, int silu, const void* add,
                                   int add_pitch, const void* out, int out_pitch, int sms, ladi_gn_plan* plan) {
  (void)eps; (void)silu;
  LADI_CHECK(plan != nullptr, "plan output is null");
  return gn_plan_apply(x0, c0, pitch0, x1, c1, pitch1, n, hw, groups, ws, gamma, beta, add, add_pitch, out, out_pitch,
                       sms > 0 ? sms : ladi_num_sms(), *plan);
}

extern "C" int ladi_groupnorm_stats(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups,
                                    float* ws, void* stream) {
  ladi_gn_plan pl;
  if (int e = gn_plan_stats(x0, c0, pitch0, x1, c1, pitch1, n, hw, groups, ws, ladi_num_sms(), pl)) return e;
  LADI_CUDA(ladi_launch(gn_stats_kernel, dim3(dim3(pl.chunks, n, pl.gsplit)), dim3(256), 0, STREAM, (const bf16*)x0, c0, pitch0, (const bf16*)x1, c1, pitch1, hw, groups, pl.chunks, ws));
  return LADI_OK;
}

extern "C" int ladi_groupnorm_apply(const void* x0, int c0, int pitch0, const void* x1, int c1, int pitch1, int n, int hw, int groups,
                                    const float* ws, const float* gamma, const float* beta, float eps, int silu, const void* add,
                                    int add_pitch, void* out, int out_pitch, void* stream) {
  ladi_gn_plan pl;
  if (int e = gn_plan_apply(x0, c0, pitch0, x1, c1, pitch1, n, hw, groups, ws, gamma, beta, add, add_pitch, out, out_pitch, ladi_num_sms(), pl))
    return e;
  const int ppb = pl.px_per_block, blocks = pl.apply_blocks, chunks = pl.chunks;
  if (add != nullptr)
    LADI_CUDA(ladi_launch(gn_apply_kernel<true>, dim3(dim3(blocks, n)), dim3(256), 0, STREAM, (const bf16*)x0, c0, pitch0, (const bf16*)x1, c1, pitch1, hw, groups, chunks, ws,
                          gamma, beta, eps, silu, (const bf16*)add, add_pitch, (bf16*)out, out_pitch, ppb));
  else
    LADI_CUDA(ladi_launch(gn_apply_kernel<false>, dim3(dim3(blocks, n)), dim3(256), 0, STREAM, (const bf16*)x0, c0, pitch0, (const bf16*)x1, c1, pitch1, hw, groups, chunks, ws,
                          gamma, beta, eps, silu, (const bf16*)add, add_pitch, (bf16*)out, out_pitch, ppb));
  return LADI_OK;
}

// The LayerNorm launch's validation and shape: the smallest lane group T whose per-lane vector count VPL fits the register cache.
static int ln_plan(const void* x, int x_pitch, int rows, int c, const float* gamma, const float* beta, const void* out, int out_pitch,
                   ladi_ln_plan& pl) {
  LADI_CHECK(c % 8 == 0 && c <= 2048, "layernorm: C %d must be a multiple of 8 and <= 2048", c);
  LADI_CHECK(rows > 0, "layernorm: rows %d must be > 0", rows);
  LADI_CHECK(x_pitch % 8 == 0 && x_pitch >= c, "layernorm x_pitch %d must be a multiple of 8 and >= C (%d)", x_pitch, c);
  LADI_CHECK(out_pitch % 8 == 0 && out_pitch >= c, "layernorm out_pitch %d must be a multiple of 8 and >= C (%d)", out_pitch, c);
  LADI_CHECK(x != nullptr && aligned16(x), "layernorm x %p must be non-null and 16-byte aligned", x);
  LADI_CHECK(out != nullptr && aligned16(out), "layernorm out %p must be non-null and 16-byte aligned", out);
  LADI_CHECK(gamma != nullptr && aligned16(gamma), "layernorm gamma %p must be non-null and 16-byte aligned", gamma);
  LADI_CHECK(beta != nullptr && aligned16(beta), "layernorm beta %p must be non-null and 16-byte aligned", beta);
  const int nv = c / 8;
  pl.T = pl.vpl = 0;
  for (int t = 4; t <= 32; t *= 2)
    if (nv % t == 0 && nv / t <= 8) { pl.T = t; pl.vpl = nv / t; break; }
  LADI_CHECK(pl.T != 0, "layernorm: unsupported width %d (need C/8 = T * v with T in {4,8,16,32}, v <= 8)", c);
  pl.rows_per_block = 8 * (32 / pl.T);
  pl.blocks = (rows + pl.rows_per_block - 1) / pl.rows_per_block;
  return LADI_OK;
}

extern "C" int ladi_layernorm_plan(const void* x, int x_pitch, int rows, int c, const float* gamma, const float* beta, float eps,
                                   const void* out, int out_pitch, int sms, ladi_ln_plan* plan) {
  (void)eps; (void)sms;
  LADI_CHECK(plan != nullptr, "plan output is null");
  return ln_plan(x, x_pitch, rows, c, gamma, beta, out, out_pitch, *plan);
}

extern "C" int ladi_layernorm(const void* x, int x_pitch, int rows, int c, const float* gamma, const float* beta, float eps, void* out,
                              int out_pitch, void* stream) {
  ladi_ln_plan pl;
  if (int e = ln_plan(x, x_pitch, rows, c, gamma, beta, out, out_pitch, pl)) return e;
  const int T = pl.T, blocks = pl.blocks;
#define LN_CASE(V) \
  case V: LADI_CUDA(ladi_launch(layernorm_kernel<V>, dim3(blocks), dim3(256), 0, STREAM, (const bf16*)x, x_pitch, rows, c, T, gamma, beta, eps, (bf16*)out, out_pitch)); break;
  switch (pl.vpl) {
    LN_CASE(1) LN_CASE(2) LN_CASE(3) LN_CASE(4) LN_CASE(5) LN_CASE(6) LN_CASE(7) LN_CASE(8)
    default: LADI_CHECK(false, "layernorm: bad vectors per lane %d", pl.vpl);
  }
#undef LN_CASE
  return LADI_OK;
}

extern "C" int ladi_softmax_rows(const float* s, int rows, int cols, int s_pitch, float scale, void* out, int out_pitch, void* stream) {
  LADI_CHECK(rows > 0 && cols > 0, "softmax: empty");
  LADI_CUDA(ladi_launch(softmax_rows_kernel, dim3(rows), dim3(256), 0, STREAM, s, cols, s_pitch, scale, (bf16*)out, out_pitch));
  return LADI_OK;
}

// ladi_cls_attention's validation and launch size, shared with ladi_cls_attention_plan: one block per (head, image) for the one CLS
// row, dynamic shared memory for the query and the token probabilities.  The kernel reads K as bf16 pairs and everything else as
// scalars.  Without an opt-in, static and dynamic shared memory together must fit 48 KB.
static int cls_plan(const void* q0, int q_pitch, const void* kv, int kv_pitch, int batch, int tokens, int heads, int head_dim,
                    const void* out, int out_pitch, ladi_sa_plan& pl) {
  LADI_CHECK(q0 && kv && out && batch > 0 && tokens > 0 && heads > 0 && head_dim > 0 && head_dim % 2 == 0, "cls_attention: bad arguments");
  LADI_CHECK(kv_pitch % 2 == 0, "cls_attention kv_pitch %d must be even", kv_pitch);
  LADI_CHECK((reinterpret_cast<uintptr_t>(kv) & 3) == 0, "cls_attention kv %p must be 4-byte aligned", kv);
  const long long width = (long long)heads * head_dim;
  LADI_CHECK(kv_pitch >= 2 * width, "cls_attention kv_pitch %d is below 2*heads*head_dim (%lld)", kv_pitch, 2 * width);
  LADI_CHECK(q_pitch >= width, "cls_attention q_pitch %d is below heads*head_dim (%lld)", q_pitch, width);
  LADI_CHECK(out_pitch >= width, "cls_attention out_pitch %d is below heads*head_dim (%lld)", out_pitch, width);
  const size_t smem = (size_t)(head_dim + tokens) * sizeof(float);
  LADI_CHECK(smem + CLS_WARPS * sizeof(float) <= 48 * 1024, "cls_attention: too many tokens (%zu bytes of shared memory, %d tokens)",
             smem + CLS_WARPS * sizeof(float), tokens);
  pl.chunks = 1;
  pl.rows_per_block = 1;
  pl.smem_bytes = (int)smem;
  pl.smem_optin = 0;
  return LADI_OK;
}

extern "C" int ladi_cls_attention_plan(const void* q0, int q_pitch, const void* kv, int kv_pitch, int batch, int tokens, int heads,
                                       int head_dim, float scale, const void* out, int out_pitch, int sms, ladi_sa_plan* plan) {
  (void)scale; (void)sms;
  LADI_CHECK(plan != nullptr, "plan output is null");
  return cls_plan(q0, q_pitch, kv, kv_pitch, batch, tokens, heads, head_dim, out, out_pitch, *plan);
}

extern "C" int ladi_cls_attention(const void* q0, int q_pitch, const void* kv, int kv_pitch, int batch, int tokens, int heads, int head_dim,
                                  float scale, void* out, int out_pitch, void* stream) {
  ladi_sa_plan pl;
  if (int e = cls_plan(q0, q_pitch, kv, kv_pitch, batch, tokens, heads, head_dim, out, out_pitch, pl)) return e;
  LADI_CUDA(ladi_launch(cls_attention_kernel, dim3(heads, batch), dim3(128), (size_t)pl.smem_bytes, STREAM, (const bf16*)q0, q_pitch,
                        (const bf16*)kv, kv_pitch, tokens, heads, head_dim, scale, (bf16*)out, out_pitch));
  return LADI_OK;
}

extern "C" int ladi_add_bf16(const void* a, const void* b, void* out, int64_t count, void* stream) {
  LADI_CHECK(a && b && out && count >= 0 && count % 8 == 0, "add: null operand, or count not a multiple of 8");
  LADI_CHECK(aligned16(a), "add: a %p must be 16-byte aligned", a);
  LADI_CHECK(aligned16(b), "add: b %p must be 16-byte aligned", b);
  LADI_CHECK(aligned16(out), "add: out %p must be 16-byte aligned", out);
  LADI_CUDA(ladi_launch(add_kernel, dim3(grid_for(count / 8)), dim3(256), 0, STREAM, (const uint4*)a, (const uint4*)b, (uint4*)out, count / 8));
  return LADI_OK;
}

extern "C" int ladi_upsample2x_nhwc(const void* x, int n, int h, int w, int c, void* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && h > 0 && w > 0 && c > 0 && c % 8 == 0, "upsample: bad extent (C must be a multiple of 8)");
  LADI_CHECK(aligned16(x), "upsample: x %p must be 16-byte aligned", x);
  LADI_CHECK(aligned16(out), "upsample: out %p must be 16-byte aligned", out);
  LADI_CUDA(ladi_launch(upsample2x_kernel, dim3(grid_for((int64_t)n * 4 * h * w * (c / 8))), dim3(256), 0, STREAM, (const uint4*)x, n, h, w, c / 8, (uint4*)out));
  return LADI_OK;
}

extern "C" int ladi_nchw_f32_to_nhwc_bf16(const float* x, int n, int c, int h, int w, int f, float scale, const float* gate, void* out,
                                          int out_pitch, int c_off, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h > 0 && w > 0 && f >= 1, "nchw_to_nhwc: bad extent or sampling factor");
  LADI_CHECK(c_off >= 0 && out_pitch >= c_off + c, "nchw_to_nhwc: channel window [%d, %d) outside the output pitch %d", c_off, c_off + c,
             out_pitch);
  LADI_CUDA(ladi_launch(nchw_to_nhwc_kernel, dim3(grid_for((int64_t)n * c * h * w)), dim3(256), 0, STREAM, x, n, c, h, w, f, scale, gate, (bf16*)out, out_pitch, c_off));
  return LADI_OK;
}

extern "C" int ladi_nhwc_to_nchw_f32(const void* x, int x_is_fp32, int n, int c, int h, int w, int x_pitch, int c_off, float* out,
                                     void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && h > 0 && w > 0, "nhwc_to_nchw: bad extent");
  LADI_CHECK(c_off >= 0 && x_pitch >= c_off + c, "nhwc_to_nchw: channel window [%d, %d) outside the input pitch %d", c_off, c_off + c, x_pitch);
  LADI_CUDA(ladi_launch(nhwc_to_nchw_kernel, dim3(grid_for((int64_t)n * c * h * w)), dim3(256), 0, STREAM, x, x_is_fp32, n, c, h * w, x_pitch, c_off, out));
  return LADI_OK;
}

extern "C" int ladi_posterior_sample(const float* moments, int m_pitch, const float* noise_nchw, int n, int cz, int h, int w, float scale,
                                     float* out_nchw, void* stream) {
  LADI_CHECK(moments && noise_nchw && out_nchw && n > 0 && cz > 0 && h > 0 && w > 0, "posterior_sample: bad extent");
  LADI_CHECK(m_pitch >= 2 * cz, "posterior_sample: m_pitch %d is below 2*cz (%d): mean and logvar are read from one row", m_pitch, 2 * cz);
  LADI_CUDA(ladi_launch(posterior_kernel, dim3(grid_for((int64_t)n * cz * h * w)), dim3(256), 0, STREAM, moments, m_pitch, noise_nchw, n, cz, h * w, scale, out_nchw));
  return LADI_OK;
}

extern "C" int ladi_inv_mask_rows(const float* mask, int n, int H, int W, int f, float* out, void* stream) {
  LADI_CHECK(mask && out && n > 0 && H > 0 && W > 0, "inv_mask: null operand or bad extent");
  LADI_CHECK(f >= 1 && H % f == 0 && W % f == 0, "inv_mask: factor must divide H and W");
  LADI_CUDA(ladi_launch(inv_mask_kernel, dim3(grid_for((int64_t)n * (H / f) * (W / f))), dim3(256), 0, STREAM, mask, n, H, W, f, out));
  return LADI_OK;
}

extern "C" int ladi_bilinear_down8(const float* x, int n, int c, int H, int W, float* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && c > 0 && H > 0 && W > 0, "bilinear_down8: null operand or bad extent");
  LADI_CHECK(H % 8 == 0 && W % 8 == 0, "bilinear_down8: H, W must be multiples of 8");
  LADI_CUDA(ladi_launch(bilinear8_kernel, dim3(grid_for((int64_t)n * c * (H / 8) * (W / 8))), dim3(256), 0, STREAM, x, n * c, H, W, out));
  return LADI_OK;
}

extern "C" int ladi_ddim_cfg_step(const float* eps, int eps_pitch, float* latents, void* unet_in, int in_pitch, int B, int h, int w,
                                  int cfg, float guidance, const float* coef, int* step_ptr, int advance, const float* noise, void* stream) {
  LADI_CHECK(eps && latents && unet_in && coef && B > 0 && h > 0 && w > 0, "ddim: null operand or bad extent");
  LADI_CHECK(eps_pitch >= 4, "ddim: eps_pitch %d is below the 4 latent channels", eps_pitch);
  LADI_CHECK(in_pitch >= 4, "ddim: in_pitch %d is below the 4 latent channels", in_pitch);
  LADI_CHECK(!advance || step_ptr, "ddim: advance needs step_ptr (the step counter it advances)");
  LADI_CUDA(ladi_launch(ddim_cfg_kernel, dim3(grid_for((int64_t)B * 4 * h * w)), dim3(256), 0, STREAM, eps, eps_pitch, latents, (bf16*)unet_in, in_pitch, B, h * w, cfg,
                                                                         guidance, coef, step_ptr, advance, noise));
  return LADI_OK;
}

extern "C" int ladi_check_binarise(const float* image, long long n_image, float* mask, long long n_mask, int* flags, void* stream) {
  LADI_CHECK(image && mask && flags && n_image > 0 && n_mask > 0, "check_binarise: bad arguments");
  const long long total = n_image > n_mask ? n_image : n_mask;
  LADI_CUDA(ladi_launch(check_binarise_kernel, dim3(grid_for((total + 3) / 4)), dim3(256), 0, STREAM, image, (int64_t)n_image, mask, (int64_t)n_mask, flags));
  return LADI_OK;
}

extern "C" int ladi_image_out_u8(const void* x, int x_is_fp32, int n, int h, int w, int x_pitch, unsigned char* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && h > 0 && w > 0 && x_pitch >= 3, "image_out_u8: bad extent");
  LADI_CUDA(ladi_launch(image_out_u8_kernel, dim3(grid_for((int64_t)n * h * w * 3)), dim3(256), 0, STREAM, x, x_is_fp32, (int64_t)n * h * w, x_pitch, out));
  return LADI_OK;
}

extern "C" int ladi_image_save_u8(const float* x, int n, int h, int w, int x_pitch, unsigned char* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && h > 0 && w > 0 && x_pitch >= 3, "image_save_u8: bad extent");
  LADI_CUDA(ladi_launch(image_save_u8_kernel, dim3(grid_for((int64_t)n * h * w * 3)), dim3(256), 0, STREAM, x, (int64_t)n * h * w, x_pitch, out));
  return LADI_OK;
}

extern "C" int ladi_pose_heatmaps(const float* keypoints, int n_maps, int h, int w, float sigma, float* out, void* stream) {
  LADI_CHECK(keypoints && out && n_maps > 0 && h > 0 && w > 0 && sigma > 0.f, "pose_heatmaps: bad extent");
  LADI_CUDA(ladi_launch(pose_heatmap_kernel, dim3(grid_for((int64_t)n_maps * h * w)), dim3(256), 0, STREAM, keypoints, n_maps, h, w,
                        1.f / (sigma * sigma), out));
  return LADI_OK;
}

extern "C" int ladi_image_out(const void* x, int x_is_fp32, int n, int h, int w, int x_pitch, float* out, void* stream) {
  LADI_CHECK(x && out && n > 0 && h > 0 && w > 0 && x_pitch >= 3, "image_out: bad extent");
  LADI_CUDA(ladi_launch(image_out_kernel, dim3(grid_for((int64_t)n * h * w * 3)), dim3(256), 0, STREAM, x, x_is_fp32, (int64_t)n * h * w, x_pitch, out));
  return LADI_OK;
}

extern "C" int ladi_timestep_embedding(const float* timesteps, int n, int channels, int k_pad, void* out, void* stream) {
  LADI_CHECK(timesteps && out && n > 0 && channels > 0 && channels % 2 == 0 && k_pad >= channels && k_pad % 8 == 0, "timestep_embedding: bad arguments");
  LADI_CUDA(ladi_launch(timestep_embed_kernel, dim3(grid_for((int64_t)n * k_pad)), dim3(256), 0, STREAM, timesteps, n, channels, k_pad, (bf16*)out));
  return LADI_OK;
}

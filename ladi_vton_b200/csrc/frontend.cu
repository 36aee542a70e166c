// Kernels of the text/vision conditioning front-end (SURVEY.md section 8(f) row 1): the CLIP text transformer of
// src/utils/encode_text_word_embedding.py (77 causal tokens, 16 heads of 64) and the CLIP ViT-H vision tower called at
// src/inference.py:269-273 (257 tokens, 16 heads of 80).  The GEMMs and LayerNorms of both run on the hot-path kernels
// (convgemm.cu, pointwise.cu); this file adds what is specific to the front-end:
//   small_attention_kernel : exact softmax attention for SHORT sequences (<= 1024 keys) and any head width that is a multiple of 8
//                            (80 does not fit the 64-wide wgmma kernel), optional causal mask.  K and V of one (image, head) live in
//                            shared memory, one warp per query row, fp32 scores / probabilities.  ~0.1 TFLOP per call in total, run
//                            once per batch: CUDA-core FMA is the right size for it.
//   clip_embed_kernel      : token-embedding gather with the '$' -> pseudo-word substitution + position embedding.
//   patchify_kernel        : NCHW fp32 pixels -> bf16 im2col rows of the 14x14/14 patch convolution (then one GEMM).
//   vit_assemble_kernel    : [CLS] + patches + position embedding.
#include "common.h"
#include "ptx.cuh"

namespace {

__device__ __forceinline__ float wsum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float wmax(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

constexpr int SA_WARPS = 8;

// grid = (query chunks, heads, images), 256 threads.  Dynamic shared memory:
//   Q  [8 warps][hd] fp32 (pre-multiplied by scale * log2 e),  P [8 warps][nkv_pad] fp32
//   Vw [nkv][hw]     32-bit words = bf16 pairs (lanes read consecutive words of one key)
//   Kw [nkv][hw + 1] words (odd row stride -> lanes reading different keys hit different banks)
__global__ void __launch_bounds__(SA_WARPS * 32) small_attention_kernel(
    const bf16* __restrict__ q, const bf16* __restrict__ k, const bf16* __restrict__ v, bf16* __restrict__ out, int nq, int nkv, int hd,
    int q_pitch, int k_pitch, int v_pitch, int out_pitch, long long q_bs, long long k_bs, long long v_bs, long long out_bs,
    float scale_log2, int causal, int rows_per_block) {
  ptx::pdl_wait();
  extern __shared__ __align__(16) uint32_t sa_smem[];
  const int hw = hd >> 1, kstride = hw + 1, nkv_pad = (nkv + 31) & ~31;
  float* Q = reinterpret_cast<float*>(sa_smem);  // first: rows are read as float4
  float* P = Q + SA_WARPS * hd;
  uint32_t* Vw = reinterpret_cast<uint32_t*>(P + SA_WARPS * nkv_pad);
  uint32_t* Kw = Vw + (size_t)nkv * hw;
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  const int h = blockIdx.y, b = blockIdx.z;
  const int r0 = blockIdx.x * rows_per_block, r1 = min(nq, r0 + rows_per_block);
  const int kv_needed = causal ? min(nkv, r1) : nkv;  // causal: keys beyond the last query row of this block are never read
  {
    const int vpr = hd >> 3;  // 16-byte vectors per row
    const bf16* kb = k + (size_t)b * k_bs + (size_t)h * hd;
    const bf16* vb = v + (size_t)b * v_bs + (size_t)h * hd;
    for (int i = t; i < kv_needed * vpr; i += SA_WARPS * 32) {
      const int row = i / vpr, vec = i - row * vpr;
      const uint4 uk = __ldg(reinterpret_cast<const uint4*>(kb + (size_t)row * k_pitch + vec * 8));
      const uint4 uv = __ldg(reinterpret_cast<const uint4*>(vb + (size_t)row * v_pitch + vec * 8));
      uint32_t* kd = Kw + (size_t)row * kstride + vec * 4;
      kd[0] = uk.x; kd[1] = uk.y; kd[2] = uk.z; kd[3] = uk.w;
      uint32_t* vd = Vw + (size_t)row * hw + vec * 4;
      vd[0] = uv.x; vd[1] = uv.y; vd[2] = uv.z; vd[3] = uv.w;
    }
  }
  __syncthreads();
  float* Pw = P + warp * nkv_pad;
  float* Qw = Q + warp * hd;
  for (int r = r0 + warp; r < r1; r += SA_WARPS) {
    const uint32_t* qrow = reinterpret_cast<const uint32_t*>(q + (size_t)b * q_bs + (size_t)r * q_pitch + (size_t)h * hd);
    for (int w = lane; w < hw; w += 32) {
      const uint32_t u = __ldg(qrow + w);
      Qw[2 * w] = ptx::bf16_lo(u) * scale_log2;
      Qw[2 * w + 1] = ptx::bf16_hi(u) * scale_log2;
    }
    __syncwarp();
    const int kv_end = causal ? min(nkv, r + 1) : nkv;
    float mx = -INFINITY;
    for (int j = lane; j < kv_end; j += 32) {
      const uint32_t* kr = Kw + (size_t)j * kstride;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int w = 0;
      for (; w + 1 < hw; w += 2) {
        const uint32_t u0 = kr[w], u1 = kr[w + 1];
        const float4 qq = *reinterpret_cast<const float4*>(Qw + 2 * w);
        a0 = fmaf(ptx::bf16_lo(u0), qq.x, a0); a1 = fmaf(ptx::bf16_hi(u0), qq.y, a1);
        a2 = fmaf(ptx::bf16_lo(u1), qq.z, a2); a3 = fmaf(ptx::bf16_hi(u1), qq.w, a3);
      }
      const float s = (a0 + a1) + (a2 + a3);  // hw is even (hd % 8 == 0), no tail
      Pw[j] = s;
      mx = fmaxf(mx, s);
    }
    mx = wmax(mx);
    float sum = 0.f;
    for (int j = lane; j < kv_end; j += 32) {
      const float e = exp2f(Pw[j] - mx);
      Pw[j] = e;
      sum += e;
    }
    sum = wsum(sum);
    __syncwarp();
    // O = P V: lane owns bf16 pairs `lane` and `lane + 32` of the head
    const bool own0 = lane < hw, own1 = lane + 32 < hw;
    float o0 = 0.f, o1 = 0.f, o2 = 0.f, o3 = 0.f;
    for (int j = 0; j < kv_end; ++j) {
      const float pj = Pw[j];
      const uint32_t* vr = Vw + (size_t)j * hw;
      if (own0) { const uint32_t u = vr[lane]; o0 = fmaf(pj, ptx::bf16_lo(u), o0); o1 = fmaf(pj, ptx::bf16_hi(u), o1); }
      if (own1) { const uint32_t u = vr[lane + 32]; o2 = fmaf(pj, ptx::bf16_lo(u), o2); o3 = fmaf(pj, ptx::bf16_hi(u), o3); }
    }
    const float inv = 1.f / sum;
    uint32_t* orow = reinterpret_cast<uint32_t*>(out + (size_t)b * out_bs + (size_t)r * out_pitch + (size_t)h * hd);
    if (own0) orow[lane] = ptx::pack_bf16(o0 * inv, o1 * inv);
    if (own1) orow[lane + 32] = ptx::pack_bf16(o2 * inv, o3 * inv);
    __syncwarp();
  }
}

// out[row, :] = (src[row] >= 0 ? tok[src[row]] : word_emb[-src[row] - 1]) + pos[row % seq]   (all bf16, sum in fp32)
__global__ void __launch_bounds__(128) clip_embed_kernel(const int* __restrict__ src, const bf16* __restrict__ tok,
                                                         const bf16* __restrict__ word_emb, const bf16* __restrict__ pos,
                                                         bf16* __restrict__ out, int seq, int c, int out_pitch) {
  ptx::pdl_wait();
  const int row = blockIdx.x;
  const int s = src[row];
  const bf16* e = s >= 0 ? tok + (size_t)s * c : word_emb + (size_t)(-s - 1) * c;
  const bf16* p = pos + (size_t)(row % seq) * c;
  for (int i = threadIdx.x; i < (c >> 3); i += 128) {
    const uint4 a = __ldg(reinterpret_cast<const uint4*>(e) + i), bb = __ldg(reinterpret_cast<const uint4*>(p) + i);
    uint4 o;
    o.x = ptx::pack_bf16(ptx::bf16_lo(a.x) + ptx::bf16_lo(bb.x), ptx::bf16_hi(a.x) + ptx::bf16_hi(bb.x));
    o.y = ptx::pack_bf16(ptx::bf16_lo(a.y) + ptx::bf16_lo(bb.y), ptx::bf16_hi(a.y) + ptx::bf16_hi(bb.y));
    o.z = ptx::pack_bf16(ptx::bf16_lo(a.z) + ptx::bf16_lo(bb.z), ptx::bf16_hi(a.z) + ptx::bf16_hi(bb.z));
    o.w = ptx::pack_bf16(ptx::bf16_lo(a.w) + ptx::bf16_lo(bb.w), ptx::bf16_hi(a.w) + ptx::bf16_hi(bb.w));
    *(reinterpret_cast<uint4*>(out + (size_t)row * out_pitch) + i) = o;
  }
}

// pixels NCHW fp32 [n, ch, h, w] -> rows [n * gh * gw, k_pad] bf16, column = (c * ps + ky) * ps + kx (the flattening of a
// [C_out, ch, ps, ps] convolution weight), zero in the padding columns.
__global__ void __launch_bounds__(256) patchify_kernel(const float* __restrict__ px, bf16* __restrict__ out, int n, int ch, int h, int w,
                                                       int ps, int k_pad) {
  ptx::pdl_wait();
  const int gh = h / ps, gw = w / ps, kk = ch * ps * ps;
  const long long total = (long long)n * gh * gw * k_pad;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < total; i += (long long)gridDim.x * 256) {
    const int col = (int)(i % k_pad);
    const long long row = i / k_pad;
    float val = 0.f;
    if (col < kk) {
      const int kx = col % ps, ky = (col / ps) % ps, c = col / (ps * ps);
      const int gx = (int)(row % gw), gy = (int)((row / gw) % gh), b = (int)(row / ((long long)gw * gh));
      val = __ldg(px + (((size_t)b * ch + c) * h + (gy * ps + ky)) * w + gx * ps + kx);
    }
    out[i] = __float2bfloat16(val);
  }
}

// x[b, 0, :] = cls + pos[0];  x[b, 1 + i, :] = patch[b * np + i, :] + pos[1 + i]
__global__ void __launch_bounds__(128) vit_assemble_kernel(const bf16* __restrict__ patch, int patch_pitch, const bf16* __restrict__ cls,
                                                           const bf16* __restrict__ pos, bf16* __restrict__ out, int np, int c) {
  ptx::pdl_wait();
  const int tkn = blockIdx.x, b = blockIdx.y;
  const bf16* a = tkn == 0 ? cls : patch + ((size_t)b * np + (tkn - 1)) * patch_pitch;
  const bf16* p = pos + (size_t)tkn * c;
  bf16* o = out + ((size_t)b * (np + 1) + tkn) * c;
  for (int i = threadIdx.x; i < (c >> 3); i += 128) {
    const uint4 u = __ldg(reinterpret_cast<const uint4*>(a) + i), bb = __ldg(reinterpret_cast<const uint4*>(p) + i);
    uint4 r;
    r.x = ptx::pack_bf16(ptx::bf16_lo(u.x) + ptx::bf16_lo(bb.x), ptx::bf16_hi(u.x) + ptx::bf16_hi(bb.x));
    r.y = ptx::pack_bf16(ptx::bf16_lo(u.y) + ptx::bf16_lo(bb.y), ptx::bf16_hi(u.y) + ptx::bf16_hi(bb.y));
    r.z = ptx::pack_bf16(ptx::bf16_lo(u.z) + ptx::bf16_lo(bb.z), ptx::bf16_hi(u.z) + ptx::bf16_hi(bb.z));
    r.w = ptx::pack_bf16(ptx::bf16_lo(u.w) + ptx::bf16_lo(bb.w), ptx::bf16_hi(u.w) + ptx::bf16_hi(bb.w));
    *(reinterpret_cast<uint4*>(o) + i) = r;
  }
}

}  // namespace

#define STREAM reinterpret_cast<cudaStream_t>(stream)

static bool aligned_to(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// Everything ladi_attention_small decides, from its arguments and the SM count alone (no pointer is dereferenced, nothing touches a
// device): validation, the dynamic shared memory of one (image, head) and the query-row split.  ladi_attention_small_plan reports it;
// ladi_attention_small launches it.  The kernel reads K and V rows as 16-byte vectors and Q rows / writes O rows as bf16 pairs.
static int sa_plan(const void* q, const void* k, const void* v, const void* out, int batch, int heads, int nq, int nkv, int head_dim,
                   int q_pitch, int k_pitch, int v_pitch, int out_pitch, long long q_batch_stride, long long k_batch_stride,
                   long long v_batch_stride, long long out_batch_stride, int causal, int sms, ladi_sa_plan& pl) {
  LADI_CHECK(q && k && v && out, "attention_small: null pointer");
  LADI_CHECK(batch > 0 && heads > 0 && nq > 0 && nkv > 0 && nkv <= 1024, "attention_small: bad extent (1 <= nkv <= 1024)");
  LADI_CHECK(head_dim >= 8 && head_dim <= 128 && head_dim % 8 == 0, "attention_small: head_dim must be a multiple of 8 in [8,128]");
  LADI_CHECK(q_pitch % 8 == 0 && k_pitch % 8 == 0 && v_pitch % 8 == 0 && out_pitch % 8 == 0 && q_batch_stride % 8 == 0 &&
                 k_batch_stride % 8 == 0 && v_batch_stride % 8 == 0 && out_batch_stride % 8 == 0,
             "attention_small: pitches and batch strides must be multiples of 8 elements");
  LADI_CHECK(aligned_to(k, 16), "attention_small k %p must be 16-byte aligned", k);
  LADI_CHECK(aligned_to(v, 16), "attention_small v %p must be 16-byte aligned", v);
  LADI_CHECK(aligned_to(q, 4), "attention_small q %p must be 4-byte aligned", q);
  LADI_CHECK(aligned_to(out, 4), "attention_small out %p must be 4-byte aligned", out);
  const long long width = (long long)heads * head_dim;
  LADI_CHECK(q_pitch >= width, "attention_small q_pitch %d is below heads*head_dim (%lld)", q_pitch, width);
  LADI_CHECK(k_pitch >= width, "attention_small k_pitch %d is below heads*head_dim (%lld)", k_pitch, width);
  LADI_CHECK(v_pitch >= width, "attention_small v_pitch %d is below heads*head_dim (%lld)", v_pitch, width);
  LADI_CHECK(out_pitch >= width, "attention_small out_pitch %d is below heads*head_dim (%lld)", out_pitch, width);
  LADI_CHECK(batch == 1 || out_batch_stride >= (long long)nq * out_pitch,
             "attention_small out_batch_stride %lld is below nq*out_pitch (%lld): output images would overlap", out_batch_stride,
             (long long)nq * out_pitch);
  LADI_CHECK(!causal || nq == nkv, "attention_small: the causal mask needs nq == nkv");
  const int hw = head_dim / 2, nkv_pad = (nkv + 31) & ~31;
  const size_t smem = ((size_t)nkv * (hw + 1) + (size_t)nkv * hw) * 4 + (size_t)SA_WARPS * nkv_pad * 4 + (size_t)SA_WARPS * head_dim * 4;
  LADI_CHECK(smem <= 200 * 1024, "attention_small: K/V of one head (%zu bytes) do not fit shared memory", smem);
  pl.smem_bytes = (int)smem;
  pl.smem_optin = smem > 48 * 1024;
  // enough blocks to cover the GPU about twice, at least one query row per warp
  int chunks = (2 * sms + batch * heads - 1) / (batch * heads);
  int rpb = (nq + chunks - 1) / chunks;
  if (rpb < SA_WARPS) rpb = SA_WARPS;
  pl.chunks = (nq + rpb - 1) / rpb;
  pl.rows_per_block = rpb;
  return LADI_OK;
}

extern "C" int ladi_attention_small_plan(const void* q, const void* k, const void* v, const void* out, int batch, int heads, int nq,
                                         int nkv, int head_dim, int q_pitch, int k_pitch, int v_pitch, int out_pitch,
                                         long long q_batch_stride, long long k_batch_stride, long long v_batch_stride,
                                         long long out_batch_stride, float scale, int causal, int sms, ladi_sa_plan* plan) {
  (void)scale;
  LADI_CHECK(plan != nullptr, "plan output is null");
  return sa_plan(q, k, v, out, batch, heads, nq, nkv, head_dim, q_pitch, k_pitch, v_pitch, out_pitch, q_batch_stride, k_batch_stride,
                 v_batch_stride, out_batch_stride, causal, sms > 0 ? sms : ladi_num_sms(), *plan);
}

extern "C" int ladi_attention_small(const void* q, const void* k, const void* v, void* out, int batch, int heads, int nq, int nkv,
                                    int head_dim, int q_pitch, int k_pitch, int v_pitch, int out_pitch, long long q_batch_stride,
                                    long long k_batch_stride, long long v_batch_stride, long long out_batch_stride, float scale,
                                    int causal, void* stream) {
  ladi_sa_plan pl;
  if (int e = sa_plan(q, k, v, out, batch, heads, nq, nkv, head_dim, q_pitch, k_pitch, v_pitch, out_pitch, q_batch_stride, k_batch_stride,
                      v_batch_stride, out_batch_stride, causal, ladi_num_sms(), pl))
    return e;
  // the largest size this process has opted the kernel into; a smaller call needs no new attribute
  static size_t configured = 0;
  if ((size_t)pl.smem_bytes > configured) {
    LADI_CUDA(cudaFuncSetAttribute(small_attention_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, pl.smem_bytes));
    configured = pl.smem_bytes;
  }
  LADI_CUDA(ladi_launch(small_attention_kernel, dim3(pl.chunks, heads, batch), dim3(SA_WARPS * 32), (size_t)pl.smem_bytes, STREAM,
                        (const bf16*)q, (const bf16*)k, (const bf16*)v, (bf16*)out, nq, nkv, head_dim, q_pitch, k_pitch, v_pitch, out_pitch,
                        q_batch_stride, k_batch_stride, v_batch_stride, out_batch_stride, scale * 1.4426950408889634f, causal,
                        pl.rows_per_block));
  return LADI_OK;
}

extern "C" int ladi_clip_embed(const int* src, const void* tok, const void* word_emb, const void* pos, void* out, int rows, int seq,
                               int c, int out_pitch, void* stream) {
  LADI_CHECK(src && tok && pos && out && rows > 0 && seq > 0, "clip_embed: bad arguments");
  LADI_CHECK(c % 8 == 0 && out_pitch % 8 == 0 && out_pitch >= c, "clip_embed: width must be a multiple of 8");
  LADI_CHECK(aligned_to(tok, 16), "clip_embed: tok %p must be 16-byte aligned", tok);
  LADI_CHECK(aligned_to(word_emb, 16), "clip_embed: word_emb %p must be 16-byte aligned", word_emb);
  LADI_CHECK(aligned_to(pos, 16), "clip_embed: pos %p must be 16-byte aligned", pos);
  LADI_CHECK(aligned_to(out, 16), "clip_embed: out %p must be 16-byte aligned", out);
  LADI_CUDA(ladi_launch(clip_embed_kernel, dim3(rows), dim3(128), 0, STREAM, src, (const bf16*)tok, (const bf16*)word_emb, (const bf16*)pos,
                        (bf16*)out, seq, c, out_pitch));
  return LADI_OK;
}

extern "C" int ladi_patchify(const float* pixels, void* out, int n, int ch, int h, int w, int patch, int k_pad, void* stream) {
  LADI_CHECK(pixels && out && n > 0 && ch > 0 && patch > 0 && h % patch == 0 && w % patch == 0, "patchify: bad extent");
  LADI_CHECK(k_pad >= ch * patch * patch && k_pad % 8 == 0, "patchify: k_pad too small or not a multiple of 8");
  const long long total = (long long)n * (h / patch) * (w / patch) * k_pad;
  long long g = (total + 255) / 256;
  const long long cap = (long long)ladi_num_sms() * 16;
  if (g > cap) g = cap;
  LADI_CUDA(ladi_launch(patchify_kernel, dim3((unsigned)g), dim3(256), 0, STREAM, pixels, (bf16*)out, n, ch, h, w, patch, k_pad));
  return LADI_OK;
}

extern "C" int ladi_vit_assemble(const void* patch, int patch_pitch, const void* cls, const void* pos, void* out, int n, int n_patches,
                                 int c, void* stream) {
  LADI_CHECK(patch && cls && pos && out && n > 0 && n_patches > 0, "vit_assemble: bad arguments");
  LADI_CHECK(c % 8 == 0 && patch_pitch % 8 == 0, "vit_assemble: width must be a multiple of 8");
  LADI_CHECK(patch_pitch >= c, "vit_assemble: patch_pitch %d is below c (%d)", patch_pitch, c);
  LADI_CHECK(n <= 65535, "vit_assemble: n %d exceeds 65535 images per call (one grid.y slice per image)", n);
  LADI_CHECK(aligned_to(patch, 16), "vit_assemble: patch %p must be 16-byte aligned", patch);
  LADI_CHECK(aligned_to(cls, 16), "vit_assemble: cls %p must be 16-byte aligned", cls);
  LADI_CHECK(aligned_to(pos, 16), "vit_assemble: pos %p must be 16-byte aligned", pos);
  LADI_CHECK(aligned_to(out, 16), "vit_assemble: out %p must be 16-byte aligned", out);
  LADI_CUDA(ladi_launch(vit_assemble_kernel, dim3(n_patches + 1, n), dim3(128), 0, STREAM, (const bf16*)patch, patch_pitch, (const bf16*)cls,
                        (const bf16*)pos, (bf16*)out, n_patches, c));
  return LADI_OK;
}

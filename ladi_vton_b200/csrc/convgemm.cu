// Implicit-GEMM convolution / GEMM for sm_90a: TMA (4-D shifted boxes, zero OOB fill = conv padding) -> 128B-swizzled smem
// -> wgmma (bf16 x bf16 -> fp32 in registers) -> fused epilogue (bias / per-step bias / SiLU / GEGLU / residual / row scale /
// LayerNorm fold / row statistics) -> bf16 or fp32 NHWC.  bf16 rows of whole 16-byte chunks go through a shared-memory staging tile
// and leave as 16-byte stores (staged_epilogue, the epilogue form fixed at compile time); everything else is stored from the
// accumulator fragment.  Persistent CTAs, one per SM; warpgroup 0 = TMA producer, warpgroups 1-2 = MMA + epilogue (64 rows each).
//
// Replaces, on the reference hot path: every nn.Conv2d / nn.Linear executed by UNet2DConditionModel.forward
// (src/vto_pipelines/tryon_pipe.py:732), AutoencoderKL.encode/decode (src/models/vae.py:99-119,183-212) and
// EMASC.forward (src/models/emasc.py:37-40), which the reference runs as cuDNN/cuBLAS library calls.
//
// A GEMM is the degenerate convolution: 1 tap, H=1, W=M.  A 3x3 stride-2 convolution reads the four parity planes of its
// input through tensor maps with doubled strides; a channel concat (UNet skip connections) or a fused 1x1 shortcut is just
// more K segments read through more tensor maps -- the concatenated tensor is never materialised.
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

namespace {

constexpr int BM = 128;   // output pixels (rows) per tile == 2 x wgmma M
constexpr int BK = 64;    // bf16 channels per K block == one 128-byte swizzle row
constexpr int UMMA_K = 16;  // K of one wgmma
constexpr int MAX_SEG = 24;
constexpr int NUM_A_MAPS = 8;
constexpr int MAX_STAGES = 8;
constexpr int A_BYTES = BM * BK * 2;

struct Segment {       // one run of K blocks read from one tensor map with one spatial shift
  int16_t map, dx, dy, chunks;
  int32_t c_begin;
};

struct KParams {
  int n_img, H, W;            // output extent
  int bn, bh, bw;             // M tile = bn x bh x bw pixels (product 128)
  int tiles_x, tiles_y, tiles_b, tiles_m, tiles_n;
  int c_out;
  int nseg, total_kb;
  int stages;                 // smem pipeline depth (runtime: whatever fits beside the staging tiles)
  int splits, kb_per_split;   // split-K: work item = (tile, split); split s reduces K blocks [s*kb_per_split, ...) into fp32 partials
  long long split_stride;     // elements between the partial planes of consecutive splits
  Segment seg[MAX_SEG];
  const float* bias;          // [c_out] fp32 (per column) or [M] (per row) or null
  int bias_per_row;
  int bias_step_stride;       // bias += (*step_ptr) * stride   (per-DDIM-step time-embedding bias table)
  const int* step_ptr;
  const bf16* residual;       // [rows, residual_pitch] or null
  int residual_pitch;
  const float* row_scale;     // [rows] or null (EMASC (1-mask))
  int act;                    // 0 none, 1 SiLU, 2 GEGLU (interleaved value/gate columns -> c_out/2 outputs)
  void* out;
  int out_pitch;
  int out_fp32;
  // LayerNorm folded into the GEMMs on either side of it (BasicTransformerBlock.norm1/2/3):
  float2* rowstat_out;        // producer: per (row, 32-column chunk) {sum, sum of squares} of the values this GEMM stores
  int rowstat_chunks;         //           = c_out / 32
  const float2* ln_stats;     // consumer: the producer's table for this GEMM's A rows; out = rstd*(acc - mean*colsum[c]) + bias[c]
  int ln_chunks;              //           = K / 32 (the normalised width)
  const float* ln_colsum;     //           [c_out] fp32: sum_k of the (gamma-scaled, bf16-rounded) weight row
  float ln_eps;
  // nearest-2x upsample fused into a 3x3 convolution (diffusers Upsample2D): the 4 output parities are 4 groups of M tiles, each a
  // 2x2-tap convolution over the half-resolution input with its own merged weights and a strided output tensor map
  int up2x, tiles_pp;         // tiles_pp = M tiles per parity plane
  // staged epilogue (bf16 out, 16-byte rows; see staged_epilogue): 0 = fragment stores; form = act | residual << 3 | column bias << 4
  int staged, form;
};

struct AMaps {
  CUtensorMap m[NUM_A_MAPS];
};
// x * sigmoid(x) = h * (1 + tanh(h)), h = x / 2: one MUFU op (tanh.approx, relative error 2^-11, below bf16 output resolution)
// instead of ex2 + a guarded division
__device__ __forceinline__ float silu_f(float x) {
  const float h = 0.5f * x;
  float t;
  asm("tanh.approx.f32 %0, %1;" : "=f"(t) : "f"(h));
  return fmaf(h, t, h);
}
// GELU(erf): erf(z) = z * Q(z^2) for |z| <= 3 (degree-8 minimax fit in z^2, clamped to +-1 beyond): |erf error| <= 4.8e-5,
// |gelu error| <= 1e-4 absolute -- below bf16 output resolution -- in 13 FMA-pipe instructions and NO MUFU op.  The GEGLU epilogue
// evaluates it for every element of the widest GEMMs of the UNet, where erff (~30 instr) or an exp-based form made the
// epilogue, not the tensor core, the bottleneck.
__device__ __forceinline__ float gelu_erf(float x) {
  const float z = fminf(fabsf(x) * 0.70710678118654752f, 3.0f);
  const float t = z * z;
  float q = 5.152028155e-08f;
  q = fmaf(q, t, -2.354745293e-06f);
  q = fmaf(q, t, 4.747267050e-05f);
  q = fmaf(q, t, -5.641741965e-04f);
  q = fmaf(q, t, 4.485662883e-03f);
  q = fmaf(q, t, -2.576915092e-02f);
  q = fmaf(q, t, 1.120152109e-01f);
  q = fmaf(q, t, -3.758995125e-01f);
  q = fmaf(q, t, 1.128372696e+00f);
  const float e = fminf(z * q, 1.0f);
  return 0.5f * x * (1.f + copysignf(e, x));
}

// The per-element epilogue, defined here once for the three places that apply it (staged_epilogue, the fragment epilogue of
// convgemm_kernel, splitk_reduce_kernel), which only supply the operands and store the result.  In this order, in fp32:
//   v = acc (after the LayerNorm fold) + bias;  v = act(v);  v += residual;  [row statistics are taken of v here]  v *= row scale;
// then ONE rounding to bf16.  GEGLU instead maps an interleaved (value, gate) column pair to one output and takes no residual.
// ACT as KParams::act: 0 none, 1 SiLU, 3 GELU(erf), 4 ReLU (2 = GEGLU is geglu_f).
template <int ACT>
__device__ __forceinline__ float act_f(float x) {
  if constexpr (ACT == 1) return silu_f(x);
  else if constexpr (ACT == 3) return gelu_erf(x);
  else if constexpr (ACT == 4) return fmaxf(x, 0.f);
  else return x;
}
__device__ __forceinline__ float geglu_f(float value, float gate, float rscale) { return value * gelu_erf(gate) * rscale; }
// act_f of a runtime `act` on every element given: one test per call, not per element.  `act` by reference, so that each test reads
// the kernel parameter where the caller holds it (passing a copy moved the basic blocks of two instantiations around).
template <typename... F>
__device__ __forceinline__ void act_rt(const int& act, F&... v) {
  if (act == 1) ((v = act_f<1>(v)), ...);
  else if (act == 3) ((v = act_f<3>(v)), ...);
  else if (act == 4) ((v = act_f<4>(v)), ...);
}
// the bias row of the current denoising step: bias table [steps][bias_step_stride], *step_ptr advanced on the device
__device__ __forceinline__ const float* step_bias(const float* bias, const int* step_ptr, int bias_step_stride) {
  if (bias != nullptr && step_ptr != nullptr) bias += (size_t)(*step_ptr) * bias_step_stride;
  return bias;
}

struct TileCoord {
  int nt, x0, y0, n0, par;
};
__device__ __forceinline__ TileCoord tile_coord(const KParams& p, int tile) {
  TileCoord t;
  int mt = tile / p.tiles_n;
  t.nt = tile - mt * p.tiles_n;
  t.par = 0;
  if (p.up2x) {
    t.par = mt / p.tiles_pp;
    mt -= t.par * p.tiles_pp;
  }
  const int tb = mt / (p.tiles_y * p.tiles_x);
  const int rem = mt - tb * (p.tiles_y * p.tiles_x);
  const int ty = rem / p.tiles_x, tx = rem - ty * p.tiles_x;
  t.x0 = tx * p.bw; t.y0 = ty * p.bh; t.n0 = tb * p.bn;
  return t;
}

// Row r (0..127) of a tile = pixel (n, y, x) of the bn x bh x bw box.  ok: inside the output extent; grow: its index in the tile grid's
// plane (the row of residual, row_scale, per-row bias and both statistics tables); orow: in the output tensor (differs only with up2x).
struct TileRow { bool ok; size_t grow, orow; };
__device__ __forceinline__ TileRow tile_row(const KParams& p, const TileCoord& tc, int r) {
  const int rn = r / (p.bh * p.bw), rr = r - rn * (p.bh * p.bw);
  const int ry = rr / p.bw, rx = rr - ry * p.bw;
  const int n = tc.n0 + rn, y = tc.y0 + ry, x = tc.x0 + rx;
  TileRow t;
  t.ok = (n < p.n_img) && (y < p.H) && (x < p.W);
  t.grow = ((size_t)n * p.H + y) * p.W + x;
  // up2x: plane pixel (y, x) of output parity par is pixel (2y + py, 2x + px) of the full-resolution output
  t.orow = p.up2x ? ((size_t)n * 2 * p.H + 2 * y + (tc.par >> 1)) * (2 * p.W) + 2 * x + (tc.par & 1) : t.grow;
  return t;
}

// Folded LayerNorm, consumer side: {rstd, -rstd * mean} of A row `row` from the producer's per-chunk partial sums, summed in chunk
// order (deterministic).  {1, 0} without ln_stats.
__device__ __forceinline__ float2 ln_fold_row(const KParams& p, const TileRow& row) {
  if (p.ln_stats == nullptr) return make_float2(1.f, 0.f);
  float s_ = 0.f, q_ = 0.f;
  if (row.ok) {
    const float4* st = reinterpret_cast<const float4*>(p.ln_stats + row.grow * p.ln_chunks);  // ln_chunks is even
    for (int c = 0; c < (p.ln_chunks >> 1); ++c) {
      const float4 u = __ldg(st + c);
      s_ += u.x; q_ += u.y; s_ += u.z; q_ += u.w;
    }
  }
  const float inv_c = 1.f / (32.f * (float)p.ln_chunks);
  const float mean = s_ * inv_c;
  const float var = fmaxf(q_ * inv_c - mean * mean, 0.f);
  const float rstd = rsqrtf(var + p.ln_eps);
  return make_float2(rstd, -rstd * mean);
}

// Staged epilogue: the BM x BN bf16 tile goes through shared memory and leaves as whole 16-byte chunks per output row.
// Staging layout: row r (of the 128 tile rows) is BN * 2 bytes; its 16-byte chunk c sits at chunk c ^ f(r), so that the 8 rows a
// stmatrix / ldmatrix matrix addresses, and the 8 consecutive chunks a quarter-warp drains, hit 8 distinct bank groups.
// BN = 32 (64-byte rows, two per 128-byte bank window) and BN = 160 (320-byte rows: 20 chunks, odd rows start half a bank window in)
// XOR the low 2 bits with the row pair, which keeps a chunk inside its aligned 4-chunk group and so inside the row (c ^ (r & 7) would
// move chunks 16-19 of a 160-wide row past its end).  At BN = 160 the odd rows' half-window offset turns that into 8 distinct bank
// groups for any 8 consecutive rows, and a drain phase that crosses from a row's last 4 chunks into the next row's first 4 finds them
// in opposite halves of the window.  Bank conflicts per 128-row tile at BN = 160 (extra shared-memory wavefronts / access phases):
// stmatrix / ldmatrix 0 / 320, GEGLU b16 stores 0 / 320, residual fill 0 / 320, drain 0 / 320, GEGLU drain (10-chunk rows) 96 / 160.
template <int BN>
__device__ __forceinline__ uint32_t stage_off(int r, int c) {
  const int pc = (BN == 32 || BN == 160) ? (c ^ ((r >> 1) & 3)) : (c ^ (r & 7));
  return (uint32_t)(r * (BN * 2) + pc * 16);
}
constexpr int STAGE_ROWTAB_BYTES = BM * 8;  // per tile row: output pixel index, or -1 past the extent

// One consumer warpgroup's 64 rows, with the epilogue form fixed at compile time (per element as stated at act_f).  ACT as KParams::act;
// COLBIAS: a per-column bias, else the per-row bias (0 without a bias).  No per-element test is left: columns at or past c_out (whole
// 8-column groups, c_out % 8 == 0) and rows past the extent are computed on whatever the staging tile holds and are not stored.
// rowtab holds the output pixel of every tile row (or -1); the caller wrote it and synchronised the warpgroup.
template <int BN, int ACT, bool RES, bool COLBIAS>
__device__ __forceinline__ void staged_epilogue(const KParams& p, const float (&acc)[BN / 2], const float* bias, int acc0, uint32_t sstage,
                                                uint32_t rowtab, int cw, const float (&rscale)[2], const float (&rbias)[2]) {
  constexpr int CPR = BN / 8;                         // 16-byte chunks per staged row
  constexpr int OCPR = ACT == 2 ? CPR / 2 : CPR;      // ... per output row (GEGLU: half width)
  const int tid = threadIdx.x & 127, warp = tid >> 5, lane = tid & 31, q = lane & 3;
  const int r0 = 64 * cw;
  if constexpr (RES) {
    // the residual of this warpgroup's rows, coalesced 16-byte loads into the staging tile.  residual rows are output rows (no up2x).
    // An in-place residual (residual == out) stays correct: these elements are written only by this warpgroup's drain below.
    constexpr int NV = 64 * CPR / 128;
    uint4 v[NV];
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int i = tid + 128 * k, r = r0 + i / CPR, col = acc0 + 8 * (i % CPR);
      const long long o = ptx::ld_shared_s64(rowtab + 8 * r);
      v[k] = (o >= 0 && col < p.c_out) ? __ldg(reinterpret_cast<const uint4*>(p.residual + (size_t)o * p.residual_pitch + col))
                                       : make_uint4(0u, 0u, 0u, 0u);
    }
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      const int i = tid + 128 * k;
      ptx::st_shared_v4(sstage + stage_off<BN>(r0 + i / CPR, i % CPR), v[k]);
    }
    ptx::named_barrier_sync(1 + cw, 128);
  }
  // stmatrix / ldmatrix matrix m = lane / 8 of column groups (j, j+1): rows + 8 * (m & 1), group j + (m >> 1)
  const int wrow = r0 + 16 * (warp & 3);
  const int mrow = wrow + 8 * ((lane >> 3) & 1) + (lane & 7);
#pragma unroll
  for (int j = 0; j < BN / 8; j += 2) {
    float b[2][2];
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int c = acc0 + 8 * (j + jj) + 2 * q;
      float2 bb = make_float2(0.f, 0.f);
      if (COLBIAS && c < p.c_out) bb = __ldg(reinterpret_cast<const float2*>(bias + c));
      b[jj][0] = bb.x; b[jj][1] = bb.y;
    }
    uint32_t res[4];
    const uint32_t maddr = sstage + stage_off<BN>(mrow, j + (lane >> 4));
    if constexpr (RES) ptx::ldmatrix_x4(maddr, res);
    uint32_t packed[4];
#pragma unroll
    for (int m = 0; m < 4; ++m) {
      const int h = m & 1, jj = m >> 1;
      float f0 = acc[4 * (j + jj) + 2 * h], f1 = acc[4 * (j + jj) + 2 * h + 1];
      if constexpr (COLBIAS) { f0 += b[jj][0]; f1 += b[jj][1]; }
      else { f0 += rbias[h]; f1 += rbias[h]; }
      if constexpr (ACT == 2) {  // GEGLU: (value, gate) pair -> output column 4 (j + jj) + q of the half-width tile
        const bf16 g = __float2bfloat16(geglu_f(f0, f1, rscale[h]));
        ptx::st_shared_b16(sstage + stage_off<BN>(wrow + 8 * h + (lane >> 2), (j + jj) >> 1) + 2 * (4 * ((j + jj) & 1) + q),
                           __bfloat16_as_ushort(g));
        continue;
      }
      f0 = act_f<ACT>(f0); f1 = act_f<ACT>(f1);
      if constexpr (RES) { f0 += ptx::bf16_lo(res[m]); f1 += ptx::bf16_hi(res[m]); }
      f0 *= rscale[h]; f1 *= rscale[h];
      packed[m] = ptx::pack_bf16(f0, f1);
    }
    if constexpr (ACT != 2) ptx::stmatrix_x4(maddr, packed);
  }
  ptx::named_barrier_sync(1 + cw, 128);
  // drain: this warpgroup's 64 rows, consecutive threads on consecutive 16-byte chunks of a row
  constexpr int NO = 64 * OCPR / 128;
  const int ocols = ACT == 2 ? p.c_out >> 1 : p.c_out, oc0 = ACT == 2 ? acc0 >> 1 : acc0;
  uint4 v[NO];
#pragma unroll
  for (int k = 0; k < NO; ++k) {
    const int i = tid + 128 * k;
    v[k] = ptx::ld_shared_v4(sstage + stage_off<BN>(r0 + i / OCPR, i % OCPR));
  }
#pragma unroll
  for (int k = 0; k < NO; ++k) {
    const int i = tid + 128 * k, col = oc0 + 8 * (i % OCPR);
    const long long o = ptx::ld_shared_s64(rowtab + 8 * (r0 + i / OCPR));
    if (o >= 0 && col < ocols) *reinterpret_cast<uint4*>(reinterpret_cast<bf16*>(p.out) + (size_t)o * p.out_pitch + col) = v[k];
  }
}

// The staged epilogue body of the launch's form (one branch per tile).
template <int BN>
__device__ __forceinline__ void staged_dispatch(const KParams& p, const float (&acc)[BN / 2], const float* bias, int acc0, uint32_t sstage,
                                                uint32_t rowtab, int cw, const float (&rscale)[2], const float (&rbias)[2]) {
#define LADI_STAGED_FORM(A, R, B) \
  case (A) | ((R) << 3) | ((B) << 4): staged_epilogue<BN, A, R, B>(p, acc, bias, acc0, sstage, rowtab, cw, rscale, rbias); break;
#define LADI_STAGED_ACT(A) LADI_STAGED_FORM(A, 0, 0) LADI_STAGED_FORM(A, 0, 1) LADI_STAGED_FORM(A, 1, 0) LADI_STAGED_FORM(A, 1, 1)
  switch (p.form) {
    LADI_STAGED_ACT(0)
    LADI_STAGED_ACT(1)
    LADI_STAGED_FORM(2, 0, 0)
    LADI_STAGED_FORM(2, 0, 1)
    LADI_STAGED_ACT(3)
    LADI_STAGED_ACT(4)
    default: __trap();
  }
#undef LADI_STAGED_ACT
#undef LADI_STAGED_FORM
}

// One CTA = one 128-row M tile x BN columns at a time, persistent over work items.  Warpgroup 0: TMA producer (one warp issues);
// warpgroups 1 and 2: wgmma consumers, each owning 64 of the 128 rows with its fp32 accumulator in registers, followed by the
// fused epilogue (staged, or straight from the accumulator fragment).  The producer runs ahead into the next work item's K blocks
// while the consumers are in their epilogue.
// PAIR = true: clusters of two CTAs on two M tiles of the same N tile.  Each CTA loads its own A tile and HALF of the B rows,
// multicast into the shared memory of both CTAs, so every B tile crosses L2 -> SM once per pair instead of once per CTA.  A stage
// is refilled only after the consumers of BOTH CTAs have released it.
template <int BN, bool PAIR>
__global__ void __launch_bounds__(384, 1)
convgemm_kernel(const __grid_constant__ AMaps amaps, const __grid_constant__ CUtensorMap tmB, const __grid_constant__ KParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  constexpr int B_BYTES = BN * BK * 2;
  const int STAGES = p.stages;
  constexpr int STAGE_BYTES = BM * BN * 2;
  // [staging tile][row table] only for a staged launch, then the pipeline stages and their barriers
  const uint32_t sstage = ptx::smem_u32(smem), rowtab = sstage + STAGE_BYTES;
  uint8_t* sA = smem + (p.staged ? STAGE_BYTES + STAGE_ROWTAB_BYTES : 0);
  uint8_t* sB = sA + STAGES * A_BYTES;
  uint64_t* bars = reinterpret_cast<uint64_t*>(sB + STAGES * B_BYTES);
  const uint32_t full0 = ptx::smem_u32(bars), empty0 = full0 + 8 * MAX_STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const uint32_t rank = PAIR ? ptx::cluster_ctarank() : 0u;
  const int worker = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x, nworkers = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nseg; ++s) ptx::prefetch_tmap(&amaps.m[p.seg[s].map]);
    ptx::prefetch_tmap(&tmB);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(full0 + 8 * s, 1);
      ptx::mbar_init(empty0 + 8 * s, PAIR ? 4 : 2);  // one arrival per consumer warpgroup (of both CTAs with PAIR)
    }
    ptx::fence_barrier_init();
  }
  if constexpr (PAIR) ptx::cluster_sync();  // the peer's barriers are initialised before anything is signalled across the pair
  else __syncthreads();
  ptx::pdl_wait();  // everything above overlapped the previous kernel's tail; its results are visible from here on

  // work items: single CTA = (tile, K split); pair = (pair of M tiles, N tile), this CTA taking M tile 2*pm + rank (a phantom tile
  // past the end when tiles_m is odd: its loads are zero-filled and its stores masked by row_ok)
  const int num_items = PAIR ? ((p.tiles_m + 1) >> 1) * p.tiles_n : p.tiles_m * p.tiles_n * p.splits;
  auto item_tile = [&](int item) -> int {
    if constexpr (PAIR) {
      const int pm = item / p.tiles_n;
      return (2 * pm + (int)rank) * p.tiles_n + (item - pm * p.tiles_n);
    } else {
      return item / p.splits;
    }
  };

  if (wg == 0) {
    ptx::setmaxnreg_dec<40>();
    if (warp == 0) {
      // ------------------------------------------------------------------ TMA producer (warp-uniform loop, one elected lane issues)
      uint32_t stage = 0, phase = 0;
      // single CTA: blockIdx.x / gridDim.x read where they are used (not `worker` held from the prologue) keep ptxas from spilling the
      // item counter of convgemm_kernel<160, false>
      for (int item = PAIR ? worker : (int)blockIdx.x; item < num_items; item += PAIR ? nworkers : (int)gridDim.x) {
        const int tile = item_tile(item), split = PAIR ? 0 : item - tile * p.splits;
        const int kb0 = split * p.kb_per_split, kb1 = min(p.total_kb, kb0 + p.kb_per_split);
        const TileCoord tc = tile_coord(p, tile);
        int kb = 0;
        for (int s = 0; s < p.nseg && kb < kb1; ++s) {
          const Segment sg = p.seg[s];
          const CUtensorMap* am = &amaps.m[sg.map];
          if (kb + sg.chunks <= kb0) { kb += sg.chunks; continue; }
          for (int c = 0; c < sg.chunks && kb < kb1; ++c, ++kb) {
            if (kb < kb0) continue;
            ptx::mbar_wait(empty0 + 8 * stage, phase ^ 1);
            const uint32_t fb = full0 + 8 * stage;
            if (ptx::elect_one()) {
              ptx::mbar_expect_tx(fb, A_BYTES + B_BYTES);  // with PAIR: own A + own B half + the peer's B half
              ptx::tma_load_4d(am, ptx::smem_u32(sA + stage * A_BYTES), fb, sg.c_begin + c * BK, tc.x0 + sg.dx + (tc.par & 1),
                               tc.y0 + sg.dy + (tc.par >> 1), tc.n0);
              if constexpr (PAIR)
                ptx::tma_load_2d_multicast(&tmB, ptx::smem_u32(sB + stage * B_BYTES + rank * (B_BYTES / 2)), fb, kb * BK,
                                           tc.par * p.c_out + tc.nt * BN + (int)rank * (BN / 2), (uint16_t)3);
              else
                ptx::tma_load_2d(&tmB, ptx::smem_u32(sB + stage * B_BYTES), fb, kb * BK, tc.par * p.c_out + tc.nt * BN);
            }
            __syncwarp();
            if (++stage == (uint32_t)STAGES) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // -------------------------------------------------------------------- consumers: wgmma over the K blocks, then the epilogue
    const int cw = wg - 1;                                   // rows [64 cw, 64 cw + 64) of the tile
    const bool signaller = (threadIdx.x & 127) == 0;
    const uint32_t empty_peer0 = PAIR ? ptx::mapa(empty0, rank ^ 1u) : 0u;
    auto release = [&](uint32_t st) {
      if (signaller) {
        ptx::mbar_arrive(empty0 + 8 * st);
        if constexpr (PAIR) ptx::mbar_arrive_cluster(empty_peer0 + 8 * st);
      }
    };
    const float* bias = step_bias(p.bias, p.step_ptr, p.bias_step_stride);
    const int q = lane & 3;
    const int rbase = 64 * cw + 16 * (warp & 3) + (lane >> 2);  // this thread's rows: rbase and rbase + 8
    uint32_t stage = 0, phase = 0;
    float acc[BN / 2];
    for (int item = PAIR ? worker : (int)blockIdx.x; item < num_items; item += PAIR ? nworkers : (int)gridDim.x) {
      const int tile = item_tile(item), split = PAIR ? 0 : item - tile * p.splits;
      const int nkb = min(p.total_kb, (split + 1) * p.kb_per_split) - split * p.kb_per_split;
      uint32_t prev = 0;
      for (int kb = 0; kb < nkb; ++kb) {
        ptx::mbar_wait(full0 + 8 * stage, phase);
        const uint64_t adesc = ptx::smem_desc_sw128(ptx::smem_u32(sA + stage * A_BYTES + cw * (A_BYTES / 2)));
        const uint64_t bdesc = ptx::smem_desc_sw128(ptx::smem_u32(sB + stage * B_BYTES));
        ptx::wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / UMMA_K; ++k) ptx::Wgmma<BN>::ss(acc, adesc + 2 * k, bdesc + 2 * k, (kb | k) != 0);
        ptx::wgmma_commit();
        if (kb > 0) {
          ptx::wgmma_wait<1>();  // the MMAs of the previous K block have read their stage
          release(prev);
        }
        prev = stage;
        if (++stage == (uint32_t)STAGES) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_wait<0>();
      ptx::reg_fence(acc);
      release(prev);

      // ---------------------------------------------------------------- epilogue, both store paths: this thread's two rows of the tile
      const TileCoord tc = tile_coord(p, tile);
      const int acc0 = tc.nt * BN;                           // first accumulator column of this tile (global)
      TileRow row[2];
      float rscale[2], rbias[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        row[h] = tile_row(p, tc, rbase + 8 * h);
        rscale[h] = (p.row_scale != nullptr && row[h].ok) ? p.row_scale[row[h].grow] : 1.f;
        rbias[h] = (p.bias_per_row && bias != nullptr && row[h].ok) ? bias[row[h].grow] : 0.f;
      }
      // ---------------------------------------------------------------- staged: row table, then the body of the launch's form
      if constexpr (!PAIR && (BN <= 128 || BN == 160)) {
        if (p.staged) {
          ptx::named_barrier_sync(1 + cw, 128);  // the previous tile's drain has read the staging tile and the row table
          if (q == 0) {
#pragma unroll
            for (int h = 0; h < 2; ++h) ptx::st_shared_s64(rowtab + 8 * (rbase + 8 * h), row[h].ok ? (long long)row[h].orow : -1ll);
          }
          ptx::named_barrier_sync(1 + cw, 128);
          staged_dispatch<BN>(p, acc, bias, acc0, sstage, rowtab, cw, rscale, rbias);
          continue;
        }
      }
      // ---------------------------------------------------------------- fragment: stores from the accumulator, forms tested per element
      float2 ln[2];                                  // out = ln.x * acc + ln.y * colsum[c] (+ bias)
#pragma unroll
      for (int h = 0; h < 2; ++h) ln[h] = ln_fold_row(p, row[h]);
      float rs[2] = {0.f, 0.f}, rq[2] = {0.f, 0.f};  // row statistics of the current 32-column chunk (rowstat_out)
      // Columns in groups of 32 (JG column pairs per thread).  A group's bias and residual loads are all issued before any of its
      // arithmetic and stores: each element's branches end a basic block, so loads left inside the element code waited out one
      // memory latency per element pair.
      constexpr int JG = 4;
#pragma unroll
      for (int j0 = 0; j0 < BN / 8; j0 += JG) {
        float bv[JG][2];
        uint32_t rv[JG][2];
#pragma unroll
        for (int jj = 0; jj < JG; ++jj) {
          const int c = acc0 + 8 * (j0 + jj) + 2 * q;
          const bool v0 = c < p.c_out, v1 = c + 1 < p.c_out;
          bv[jj][0] = (bias != nullptr && !p.bias_per_row && v0) ? __ldg(bias + c) : 0.f;
          bv[jj][1] = (bias != nullptr && !p.bias_per_row && v1) ? __ldg(bias + c + 1) : 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            uint32_t u = 0u;
            if (p.residual != nullptr && row[h].ok) {
              const bf16* rr = p.residual + row[h].grow * p.residual_pitch + c;
              if (v1 && (p.residual_pitch & 1) == 0) {
                u = __ldg(reinterpret_cast<const unsigned int*>(rr));
              } else {
                const uint32_t lo = v0 ? (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(rr)) : 0u;
                const uint32_t hi = v1 ? (uint32_t)__ldg(reinterpret_cast<const unsigned short*>(rr) + 1) : 0u;
                u = lo | (hi << 16);
              }
            }
            rv[jj][h] = u;
          }
        }
#pragma unroll
        for (int jj = 0; jj < JG; ++jj) {
          const int j = j0 + jj;
          const int c = acc0 + 8 * j + 2 * q;                  // global accumulator column of this thread's pair
          const bool v0 = c < p.c_out, v1 = c + 1 < p.c_out;
          const float b0 = bv[jj][0], b1 = bv[jj][1];
          float cs0 = 0.f, cs1 = 0.f;
          if (p.ln_stats != nullptr) {
            if (v0) cs0 = __ldg(p.ln_colsum + c);
            if (v1) cs1 = __ldg(p.ln_colsum + c + 1);
          }
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f0 = acc[4 * j + 2 * h], f1 = acc[4 * j + 2 * h + 1];
            if (p.ln_stats != nullptr) { f0 = fmaf(ln[h].y, cs0, ln[h].x * f0); f1 = fmaf(ln[h].y, cs1, ln[h].x * f1); }
            if (p.bias_per_row) { f0 += rbias[h]; f1 += rbias[h]; }
            else { f0 += b0; f1 += b1; }
            if (p.act == 2) {  // GEGLU: interleaved (value, gate) pair -> one output column
              if (row[h].ok && v1)
                reinterpret_cast<bf16*>(p.out)[row[h].orow * p.out_pitch + (c >> 1)] = __float2bfloat16(geglu_f(f0, f1, rscale[h]));
              continue;
            }
            act_rt(p.act, f0, f1);
            // The residual is read through the read-only path (__ldg), preloaded above.  An in-place residual (residual == out) stays
            // correct: each element is read only by the thread that later writes it, and before it writes it.
            if (p.residual != nullptr && row[h].ok) {
              const uint32_t u = rv[jj][h];
              if (v1 && (p.residual_pitch & 1) == 0) {
                f0 += ptx::bf16_lo(u); f1 += ptx::bf16_hi(u);
              } else {
                if (v0) f0 += ptx::bf16_lo(u);
                if (v1) f1 += ptx::bf16_hi(u);
              }
            }
            if (p.rowstat_out != nullptr) {
              rs[h] += f0 + f1;
              rq[h] = fmaf(f0, f0, fmaf(f1, f1, rq[h]));
            }
            f0 *= rscale[h]; f1 *= rscale[h];
            if (!row[h].ok) continue;
            if (p.out_fp32) {
              float* o = reinterpret_cast<float*>(p.out) + (size_t)split * p.split_stride + row[h].orow * p.out_pitch + c;
              if (v1 && (p.out_pitch & 1) == 0) *reinterpret_cast<float2*>(o) = make_float2(f0, f1);
              else { if (v0) o[0] = f0; if (v1) o[1] = f1; }
            } else {
              bf16* o = reinterpret_cast<bf16*>(p.out) + row[h].orow * p.out_pitch + c;
              if (v1 && (p.out_pitch & 1) == 0) *reinterpret_cast<uint32_t*>(o) = ptx::pack_bf16(f0, f1);
              else { if (v0) o[0] = __float2bfloat16(f0); if (v1) o[1] = __float2bfloat16(f1); }
            }
          }
          if (p.rowstat_out != nullptr && (j & 3) == 3) {     // a 32-column chunk is complete: reduce over the 4 lanes of the row
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              float s_ = rs[h], q_ = rq[h];
              s_ += __shfl_xor_sync(0xffffffffu, s_, 1); q_ += __shfl_xor_sync(0xffffffffu, q_, 1);
              s_ += __shfl_xor_sync(0xffffffffu, s_, 2); q_ += __shfl_xor_sync(0xffffffffu, q_, 2);
              const int chunk_col = acc0 + 8 * (j - 3);
              if (q == 0 && row[h].ok && chunk_col < p.c_out) p.rowstat_out[row[h].grow * p.rowstat_chunks + (chunk_col >> 5)] = make_float2(s_, q_);
              rs[h] = 0.f; rq[h] = 0.f;
            }
          }
        }
      }
    }
  }

  ptx::pdl_trigger();
  if constexpr (PAIR) ptx::cluster_sync();  // neither CTA exits while the other may still write its shared memory or barriers
}

// Split-K second pass: out = act(sum_s partial[s] + bias) + residual, bf16.  Partials are summed in split order -> deterministic.
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const float* __restrict__ ws, int splits, long long split_stride, long long rows,
                                                            int c_out, const float* __restrict__ bias, int bias_step_stride,
                                                            const int* __restrict__ step_ptr, int act, const bf16* __restrict__ residual,
                                                            int residual_pitch, bf16* __restrict__ out, int out_pitch) {
  ptx::pdl_wait();
  bias = step_bias(bias, step_ptr, bias_step_stride);
  const int cv = c_out >> 2;
  const long long total = rows * cv;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total; i += (long long)gridDim.x * blockDim.x) {
    const long long row = i / cv;
    const int col = (int)(i - row * cv) * 4;
    float4 acc = *reinterpret_cast<const float4*>(ws + row * c_out + col);
    for (int s = 1; s < splits; ++s) {
      const float4 v = *reinterpret_cast<const float4*>(ws + s * split_stride + row * c_out + col);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
    if (bias != nullptr) {
      const float4 b4 = __ldg(reinterpret_cast<const float4*>(bias + col));
      acc.x += b4.x; acc.y += b4.y; acc.z += b4.z; acc.w += b4.w;
    }
    act_rt(act, acc.x, acc.y, acc.z, acc.w);
    if (residual != nullptr) {
      const uint2 u = __ldg(reinterpret_cast<const uint2*>(residual + row * residual_pitch + col));
      acc.x += ptx::bf16_lo(u.x); acc.y += ptx::bf16_hi(u.x); acc.z += ptx::bf16_lo(u.y); acc.w += ptx::bf16_hi(u.y);
    }
    *reinterpret_cast<uint2*>(out + row * out_pitch + col) = make_uint2(ptx::pack_bf16(acc.x, acc.y), ptx::pack_bf16(acc.z, acc.w));
  }
}

constexpr size_t SMEM_LIMIT = 232448;  // 227 KiB per CTA
constexpr size_t SMEM_TAIL = 2 * MAX_STAGES * 8 + 1024;  // barriers + alignment slack

// Pipeline depth of an N tile and store path: as many (A, B) stages as fit beside the staging tile, at most MAX_STAGES.
int pipeline_stages(int bn, bool staged) {
  const size_t per_stage = A_BYTES + (size_t)bn * BK * 2;
  const size_t staging = staged ? (size_t)BM * bn * 2 + STAGE_ROWTAB_BYTES : 0;
  const int stages = (int)((SMEM_LIMIT - SMEM_TAIL - staging) / per_stage);
  return stages > MAX_STAGES ? MAX_STAGES : stages;
}

// kp.stages is the plan's (pipeline_stages); the launch sizes shared memory and the grid from it and the tile grid.
template <int BN, bool PAIR>
int launch(const AMaps& am, const CUtensorMap& tmB, const KParams& kp, cudaStream_t stream) {
  static bool attr_set = false;
  static int max_clusters = 0;
  if (!attr_set) {
    LADI_CUDA(cudaFuncSetAttribute(convgemm_kernel<BN, PAIR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_LIMIT));
    if (PAIR) {  // how many CTA pairs can be co-resident (one CTA per SM): the persistent grid size
      cudaLaunchConfig_t cfg = {};
      cfg.gridDim = dim3(2 * ladi_num_sms()); cfg.blockDim = dim3(384); cfg.dynamicSmemBytes = SMEM_LIMIT;
      cudaLaunchAttribute at[1];
      at[0].id = cudaLaunchAttributeClusterDimension;
      at[0].val.clusterDim.x = 2; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
      cfg.attrs = at; cfg.numAttrs = 1;
      if (cudaOccupancyMaxActiveClusters(&max_clusters, convgemm_kernel<BN, PAIR>, &cfg) != cudaSuccess || max_clusters <= 0) {
        (void)cudaGetLastError();
        max_clusters = ladi_num_sms() / 2;
      }
    }
    attr_set = true;
  }
  const size_t per_stage = A_BYTES + (size_t)BN * BK * 2;
  const size_t staging = kp.staged ? (size_t)BM * BN * 2 + STAGE_ROWTAB_BYTES : 0;
  const size_t smem = staging + kp.stages * per_stage + SMEM_TAIL;
  if (PAIR) {
    const int items = ((kp.tiles_m + 1) / 2) * kp.tiles_n;
    const int clusters = items < max_clusters ? items : max_clusters;
    LADI_CUDA(ladi_launch_cluster(convgemm_kernel<BN, PAIR>, dim3(2 * clusters), dim3(384), 2u, smem, stream, am, tmB, kp));
    return LADI_OK;
  }
  const int tiles = kp.tiles_m * kp.tiles_n * kp.splits;
  const int grid = tiles < ladi_num_sms() ? tiles : ladi_num_sms();
  LADI_CUDA(ladi_launch(convgemm_kernel<BN, PAIR>, dim3(grid), dim3(384), smem, stream, am, tmB, kp));
  return LADI_OK;
}

int largest_pow2_divisor(int v, int cap) {
  int d = 1;
  while (d * 2 <= cap && v % (d * 2) == 0) d *= 2;
  return d;
}

int validate(const ladi_conv_desc* d) {
  LADI_CHECK(d != nullptr, "conv desc is null");
  LADI_CHECK(d->ksize == 1 || d->ksize == 3, "ksize must be 1 or 3 (got %d)", d->ksize);
  LADI_CHECK(d->stride == 1 || d->stride == 2, "stride must be 1 or 2 (got %d)", d->stride);
  LADI_CHECK(d->n_src >= 1 && d->n_src <= 2 && d->n_sc >= 0 && d->n_sc <= 2, "bad source counts");
  LADI_CHECK(d->n > 0 && d->h_out > 0 && d->w_out > 0 && d->c_out > 0, "bad output extent");
  LADI_CHECK(d->act >= 0 && d->act <= 4, "bad act");
  LADI_CHECK(d->act != 2 || (d->c_out % 2 == 0 && !d->out_fp32 && d->residual == nullptr), "GEGLU needs even c_out, bf16 out");
  LADI_CHECK(d->out != nullptr && d->weight != nullptr, "null out/weight");
  const bool up = d->up2x != 0;
  if (up) {
    LADI_CHECK(d->ksize == 3 && d->stride == 1 && d->n_sc == 0, "up2x: 3x3 stride-1 convolution without fused shortcut only");
    LADI_CHECK(d->h_out % 2 == 0 && d->w_out % 2 == 0, "up2x: output extent must be even");
    LADI_CHECK(d->residual == nullptr && d->row_scale == nullptr && !d->bias_per_row && d->act != 2 && !d->out_fp32,
               "up2x: bf16 output with per-channel bias / SiLU / GELU / ReLU only");
  }
  LADI_CHECK(d->rowstat_out == nullptr || (d->c_out % 32 == 0 && d->act != 2 && d->row_scale == nullptr && !d->out_fp32 && !up),
             "rowstat_out: c_out %% 32 == 0, bf16 out, no GEGLU / row_scale");
  LADI_CHECK(d->ln_stats == nullptr || (d->ln_colsum != nullptr && d->c_out % 32 == 0 && d->ksize == 1 && d->n_src == 1 && d->n_sc == 0 &&
                                        d->src_c[0] % 64 == 0 && !d->out_fp32 && !d->bias_per_row && !up),
             "ln_stats: GEMM over one source of K %% 64 == 0, c_out %% 32 == 0, bf16 out, ln_colsum given");
  // placements no store path can serve (the fragment path stores bf16 pairs as 4 bytes, fp32 pairs as 8, reads residual pairs as 4,
  // writes row statistics as float2 and reads them as float4); the staged and split-K paths need more and are chosen only when it holds
  auto misaligned = [](const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) != 0; };
  LADI_CHECK(!misaligned(d->out, d->out_fp32 ? 8 : 4), "out %p: %s output must be %d-byte aligned", d->out, d->out_fp32 ? "fp32" : "bf16",
             d->out_fp32 ? 8 : 4);
  LADI_CHECK(d->out_pitch >= (d->act == 2 ? d->c_out / 2 : d->c_out), "out_pitch %d below the output width", d->out_pitch);
  LADI_CHECK(d->residual == nullptr || !misaligned(d->residual, 4), "residual %p must be 4-byte aligned", d->residual);
  LADI_CHECK(d->residual == nullptr || d->residual_pitch >= d->c_out, "residual_pitch %d below c_out %d", d->residual_pitch, d->c_out);
  LADI_CHECK(d->rowstat_out == nullptr || !misaligned(d->rowstat_out, 8), "rowstat_out %p must be 8-byte aligned", (void*)d->rowstat_out);
  LADI_CHECK(d->ln_stats == nullptr || !misaligned(d->ln_stats, 16), "ln_stats %p must be 16-byte aligned", (const void*)d->ln_stats);
  return LADI_OK;
}

// The M tile (bn x bh x bw pixels) and the tile grid.  up2x: the grid covers ONE output parity plane (h_out/2 x w_out/2 pixels = the
// input extent); tiles_m counts all four.
void tile_geometry(const ladi_conv_desc* d, KParams& kp) {
  const int up = d->up2x ? 1 : 0;
  const int HO = up ? d->h_out / 2 : d->h_out, WO = up ? d->w_out / 2 : d->w_out;
  kp.n_img = d->n; kp.H = HO; kp.W = WO; kp.c_out = d->c_out;
  kp.bw = largest_pow2_divisor(WO, 128);
  if (d->ksize == 1 && d->h_out == 1 && d->stride == 1) kp.bw = 128;  // plain GEMM: row tail handled by OOB fill
  kp.bh = largest_pow2_divisor(HO, 128 / kp.bw);
  kp.bn = 128 / (kp.bw * kp.bh);
  kp.tiles_x = (WO + kp.bw - 1) / kp.bw;
  kp.tiles_y = (HO + kp.bh - 1) / kp.bh;
  kp.tiles_b = (d->n + kp.bn - 1) / kp.bn;
  kp.tiles_m = kp.tiles_x * kp.tiles_y * kp.tiles_b;
  kp.up2x = up; kp.tiles_pp = kp.tiles_m;
  if (up) kp.tiles_m *= 4;
}

// The input extent the A tensor maps cover (up2x: the half-resolution input = one output parity plane).
int input_h(const ladi_conv_desc* d, const KParams& kp) { return kp.up2x ? kp.H : (d->h_in > 0 ? d->h_in : d->h_out * d->stride); }
int input_w(const ladi_conv_desc* d, const KParams& kp) { return kp.up2x ? kp.W : (d->w_in > 0 ? d->w_in : d->w_out * d->stride); }

// The K segments (host arithmetic only): taps (row-major) x sources, then the shortcut sources; weight K order must match (see packer).
// A tensor maps are numbered as encode_a_maps writes them: the stride x stride parity planes of each source, then one per shortcut.
int walk_segments(const ladi_conv_desc* d, KParams& kp) {
  const int up = kp.up2x, s = d->stride;
  int nmaps = 0, src_map0[2] = {0, 0}, sc_map0[2] = {0, 0};
  for (int i = 0; i < d->n_src; ++i) {
    LADI_CHECK(d->src[i] != nullptr && d->src_c[i] > 0 && d->src_pitch[i] % 8 == 0 && d->src_pitch[i] >= d->src_c[i] &&
                   reinterpret_cast<uintptr_t>(d->src[i]) % 16 == 0,
               "source %d: need non-null and 16-byte aligned, pitch multiple of 8 and >= C", i);
    src_map0[i] = nmaps;
    nmaps += s * s;
  }
  for (int i = 0; i < d->n_sc; ++i) {
    LADI_CHECK(s == 1, "fused 1x1 shortcut requires stride 1");
    LADI_CHECK(d->sc[i] != nullptr && d->sc_c[i] > 0 && d->sc_pitch[i] % 8 == 0 && reinterpret_cast<uintptr_t>(d->sc[i]) % 16 == 0,
               "shortcut source %d invalid", i);
    sc_map0[i] = nmaps++;
  }
  LADI_CHECK(nmaps <= NUM_A_MAPS, "too many tensor maps");

  int nseg = 0, total = 0;
  auto add_seg = [&](int map, int dx, int dy, int channels) -> int {
    LADI_CHECK(nseg < MAX_SEG, "too many K segments");
    Segment& sg = kp.seg[nseg++];
    sg.map = (int16_t)map; sg.dx = (int16_t)dx; sg.dy = (int16_t)dy;
    sg.chunks = (int16_t)((channels + BK - 1) / BK);
    sg.c_begin = 0;
    total += sg.chunks;
    return LADI_OK;
  };
  const int taps = up ? 4 : d->ksize * d->ksize;
  for (int t = 0; t < taps; ++t) {
    const int ky = up ? t / 2 : (d->ksize == 3 ? t / 3 : 0), kx = up ? t % 2 : (d->ksize == 3 ? t % 3 : 0);
    // input coordinate = out*stride + k - pad_lo;  parity plane p = (k - pad_lo) mod s, shift = floor((k - pad_lo) / s)
    // up2x: output pixel 2i+p reads input pixels i+p-1 and i+p (merged taps); the kernel adds the parity p, so the base shift is t-1
    const int oy = up ? ky - 1 : ky - (d->ksize == 3 ? d->pad_lo : 0), ox = up ? kx - 1 : kx - (d->ksize == 3 ? d->pad_lo : 0);
    const int py = ((oy % s) + s) % s, px = ((ox % s) + s) % s;
    for (int i = 0; i < d->n_src; ++i)
      if (const int rc = add_seg(src_map0[i] + py * s + px, (ox - px) / s, (oy - py) / s, d->src_c[i])) return rc;
  }
  for (int i = 0; i < d->n_sc; ++i)
    if (const int rc = add_seg(sc_map0[i], 0, 0, d->sc_c[i])) return rc;
  kp.nseg = nseg; kp.total_kb = total;
  LADI_CHECK(d->k_total == total * BK, "weight K (%d) != %d K-blocks x 64 implied by the sources", d->k_total, total);
  LADI_CHECK(d->weight_pitch % 8 == 0 && d->weight_pitch >= d->k_total, "weight pitch must be a multiple of 8 and >= K");
  return LADI_OK;
}

// The A tensor maps walk_segments numbered: one per (source, parity plane), then one per shortcut source.
int encode_a_maps(const ladi_conv_desc* d, const KParams& kp, AMaps& am) {
  const int s = d->stride, h_in = input_h(d, kp), w_in = input_w(d, kp);
  const uint32_t box[4] = {(uint32_t)BK, (uint32_t)kp.bw, (uint32_t)kp.bh, (uint32_t)kp.bn};
  int nmaps = 0;
  // the st x st parity planes of one NHWC tensor (st = 1: the tensor itself)
  auto add_maps = [&](const void* ptr, int c, int pitch_, int w, int h, int st) -> int {
    for (int py = 0; py < st; ++py)
      for (int px = 0; px < st; ++px) {
        const uint64_t pitch = (uint64_t)pitch_;
        const uint64_t dims[4] = {(uint64_t)c, (uint64_t)((w - px + st - 1) / st), (uint64_t)((h - py + st - 1) / st), (uint64_t)d->n};
        const uint64_t strides[3] = {pitch * 2 * st, pitch * 2 * w * st, pitch * 2 * (uint64_t)w * h};
        const bf16* base = reinterpret_cast<const bf16*>(ptr) + ((size_t)py * w + px) * pitch;
        if (const int rc = ladi_encode_tmap_bf16(&am.m[nmaps++], base, 4, dims, strides, box)) return rc;
      }
    return LADI_OK;
  };
  for (int i = 0; i < d->n_src; ++i)
    if (const int rc = add_maps(d->src[i], d->src_c[i], d->src_pitch[i], w_in, h_in, s)) return rc;
  for (int i = 0; i < d->n_sc; ++i)
    if (const int rc = add_maps(d->sc[i], d->sc_c[i], d->sc_pitch[i], d->w_out, d->h_out, 1)) return rc;
  for (int i = nmaps; i < NUM_A_MAPS; ++i) am.m[i] = am.m[0];
  return LADI_OK;
}

// The path one descriptor takes: the ONLY place that decides it.  Reads nothing but its arguments.
struct Plan {
  int bn, splits, kb_per_split;  // N tile; split-K (splits > 1: fp32 partials, splitk_reduce_kernel runs the epilogue), as in KParams
  bool pair, staged;             // CTA pairs; staged epilogue (else fragment stores)
  int form;                      // KParams::form
};
Plan choose_plan(const ladi_conv_desc* d, int tiles_m, int total_kb, int sms) {
  const bool up = d->up2x != 0;
  Plan pl = {0, 1, total_kb, false, false, 0};
  // ---- N tile.  1. the caller's (force_bn, which also rules out split-K)
  if (d->force_bn > 0) pl.bn = d->force_bn;
  // 2. split-K: few output tiles but a long reduction (the 8x6 / 16x12 UNet levels): spread K over otherwise idle SMs, fp32 partial
  // planes in the caller's workspace, summed (in split order) by splitk_reduce_kernel.  Its N tile is the widest that c_out fills.
  // The reduce moves 4 columns at a time (float4 workspace and bias loads, 8-byte residual loads and output stores): a placement
  // without that alignment runs unsplit.
  const auto aligned = [](const void* p, uintptr_t a) { return (reinterpret_cast<uintptr_t>(p) & (a - 1)) == 0; };
  if (d->splitk_ws != nullptr && d->force_bn == 0 && !d->out_fp32 && d->act != 2 && d->row_scale == nullptr && !d->bias_per_row && !up &&
      d->rowstat_out == nullptr && d->ln_stats == nullptr &&
      d->c_out % 4 == 0 && d->out_pitch % 4 == 0 && (d->residual == nullptr || d->residual_pitch % 4 == 0) && total_kb >= 32 &&
      aligned(d->out, 8) && aligned(d->residual, 8) && aligned(d->splitk_ws, 16) &&
      (d->bias == nullptr || (aligned(d->bias, 16) && d->bias_step_stride % 4 == 0))) {
    const int bn_s = d->c_out >= 256 ? 256 : (d->c_out >= 128 ? 128 : 64);
    const long tiles_s = (long)tiles_m * ((d->c_out + bn_s - 1) / bn_s);
    if (tiles_s * 2 <= sms) {
      int S = (int)(sms / tiles_s);
      if (S > total_kb / 8) S = total_kb / 8;
      if (S > 16) S = 16;
      if (S >= 2) {
        const int per = (total_kb + S - 1) / S;
        S = (total_kb + per - 1) / per;
        if (S >= 2 && (long long)S * d->n * d->h_out * d->w_out * d->c_out * 4 <= d->splitk_ws_bytes) {
          pl.bn = bn_s; pl.splits = S; pl.kb_per_split = per;
        }
      }
    }
  }
  // ---- store path, as far as the descriptor decides it: bf16 rows of whole, aligned 16-byte chunks can be staged through shared memory
  // (16-byte stores); fp32 / split-K partials, the LayerNorm fold, row statistics and odd widths take fragment stores
  const int out_cols = d->act == 2 ? d->c_out / 2 : d->c_out;
  const bool col_bias = d->bias != nullptr && !d->bias_per_row;
  const bool stageable = !d->out_fp32 && d->rowstat_out == nullptr && d->ln_stats == nullptr &&
                         out_cols % 8 == 0 && d->c_out % 8 == 0 && d->out_pitch % 8 == 0 && reinterpret_cast<uintptr_t>(d->out) % 16 == 0 &&
                         (d->residual == nullptr || (d->residual_pitch % 8 == 0 && reinterpret_cast<uintptr_t>(d->residual) % 16 == 0)) &&
                         (!col_bias || (reinterpret_cast<uintptr_t>(d->bias) % 8 == 0 && d->bias_step_stride % 2 == 0));
  const bool pairs = d->pair_mode == 1 || (d->pair_mode == 0 && ladi_conv_pair_default());
  // 3. else minimise (waves x per-tile cost), per-tile cost ~ BN + fixed A-operand cost for 128 / 64 / 32.  160 is a candidate only for
  // a long reduction (total_kb > 8) that takes the staged epilogue: short reductions keep the full-width 128 tile (below), and 160 with
  // fragment stores made the default workload slower (2602 vs 2455 ms per call, 512x384, batch 8, CFG, H100 at 400 W; measured before
  // the staged epilogue existed, when every launch stored from the fragment).  Its per-tile cost, 240, is 1.25 x the 128 tile's: what
  // tools/sweep_conv_tiles.py measured for long-K launches of the UNet step whose waves 160 does not cut (H100 80GB HBM3, 700 W).  So 160
  // wins where it removes a padded tile (c_out 320) or enough waves (c_out 640 at 96 M tiles: 4 -> 3); a tie keeps the old tile, which
  // leaves alone the launches the sweep showed no better or slower at 160 (c_out 1920, 3840, 5120 and 10240 at 24 or 96 M tiles).
  // 192 / 256 stay available through force_bn.
  if (pl.bn == 0) {
    static const int cand[4] = {128, 64, 32, 160};  // 160 last: a tie keeps the narrower tile
    long best = -1;
    for (int i = 0; i < 4; ++i) {
      if (d->pair_mode == 1 && cand[i] < 128) continue;  // forced CTA pairs need a tile they can split
      if (total_kb <= 8 && d->c_out >= 128 && cand[i] < 128) continue;  // short reductions (K <= 512): the full-width tile
      if (cand[i] == 160 && !(total_kb > 8 && d->c_out >= 160 && stageable && !pairs)) continue;
      const long tiles = (long)tiles_m * ((d->c_out + cand[i] - 1) / cand[i]);
      const long cost = ((tiles + sms - 1) / sms) * (cand[i] == 160 ? 240 : cand[i] + 64);
      if (best < 0 || cost < best) { best = cost; pl.bn = cand[i]; }
    }
  }
  const bool split = pl.splits > 1;
  // ---- CTA pairs (2-CTA clusters sharing the B tile by TMA multicast): two M tiles per cluster share one N tile; needs >= 2 M tiles,
  // no split-K, and a B half of whole 8-row swizzle groups.  pair_mode: 0 = library default (off: measured slower than single CTAs on
  // H100 for the UNet's shapes; env LADI_CONV_2CTA=1 turns it on), 1 = force, 2 = never.  up2x: a pair shares one parity's weights, so
  // the M tiles of a parity plane (tiles_m / 4) must pair up.
  if (!split && tiles_m >= 2 && pl.bn >= 128 && pl.bn % 16 == 0 && (!up || (tiles_m / 4) % 2 == 0)) {
    if (d->pair_mode == 1) pl.pair = true;
    // default: pair whenever there are enough M tiles that the phantom tile of an odd count is noise
    else if (d->pair_mode == 0 && ladi_conv_pair_default()) pl.pair = tiles_m >= 4 && (tiles_m % 2 == 0 || tiles_m >= 16);
  }
  // ---- epilogue: staged for the tiles staged_dispatch is instantiated for (160 only past the short-reduction rule); CTA pairs and split-K
  // partials store from the fragment
  pl.staged = stageable && !pl.pair && !split && (pl.bn <= 128 || (pl.bn == 160 && total_kb > 8));
  pl.form = d->act | (d->residual != nullptr ? 1 << 3 : 0) | (col_bias ? 1 << 4 : 0);
  return pl;
}

int encode_b_map(const ladi_conv_desc* d, const Plan& pl, CUtensorMap* tmB) {
  const uint64_t dims[2] = {(uint64_t)d->k_total, (uint64_t)d->c_out * (d->up2x ? 4 : 1)};  // up2x: the four parities' merged weights, stacked
  const uint64_t strides[1] = {(uint64_t)d->weight_pitch * 2};
  const uint32_t bbox[2] = {(uint32_t)BK, (uint32_t)(pl.pair ? pl.bn / 2 : pl.bn)};
  return ladi_encode_tmap_bf16(tmB, d->weight, 2, dims, strides, bbox) ? LADI_ERR_CUDA : LADI_OK;
}

// The kernel of the plan's (BN, pair), then the split-K second pass with the descriptor's own epilogue operands.
int launch_plan(const ladi_conv_desc* d, const Plan& pl, const AMaps& am, const CUtensorMap& tmB, const KParams& kp, cudaStream_t stream) {
  using Launch = int (*)(const AMaps&, const CUtensorMap&, const KParams&, cudaStream_t);
  static const struct { int bn; Launch single, pair; } table[6] = {  // every instantiation there is; tiles below 128 do not pair
      {256, launch<256, false>, launch<256, true>}, {192, launch<192, false>, launch<192, true>},
      {160, launch<160, false>, launch<160, true>}, {128, launch<128, false>, launch<128, true>},
      {64, launch<64, false>, nullptr},             {32, launch<32, false>, nullptr}};
  Launch fn = nullptr;
  for (const auto& e : table)
    if (e.bn == pl.bn) fn = pl.pair ? e.pair : e.single;
  LADI_CHECK(fn != nullptr, "unsupported BN %d", pl.bn);
  const int rc = fn(am, tmB, kp, stream);
  if (rc != LADI_OK || pl.splits == 1) return rc;
  const long long rows = (long long)d->n * d->h_out * d->w_out, vecs = rows * (d->c_out / 4);
  long long blocks = (vecs + 255) / 256;
  if (blocks > (long long)ladi_num_sms() * 8) blocks = (long long)ladi_num_sms() * 8;
  LADI_CUDA(ladi_launch(splitk_reduce_kernel, dim3((unsigned)blocks), dim3(256), 0, stream, (const float*)d->splitk_ws, kp.splits,
                        kp.split_stride, rows, d->c_out, d->bias, d->bias_step_stride, d->step_ptr, d->act,
                        reinterpret_cast<const bf16*>(d->residual), d->residual_pitch, reinterpret_cast<bf16*>(d->out), d->out_pitch));
  return LADI_OK;
}

// Everything a launch decides, from the descriptor and the SM count alone (no pointer is dereferenced, nothing touches a device):
// validation, tile grid, K segments, the plan (choose_plan) and the pipeline depth.  ladi_conv2d_plan reports it; ladi_conv2d_bf16
// launches it.
int plan_conv(const ladi_conv_desc* d, int sms, KParams& kp, Plan& pl) {
  if (const int rc = validate(d)) return rc;
  memset(&kp, 0, sizeof(kp));
  tile_geometry(d, kp);
  if (const int rc = walk_segments(d, kp)) return rc;
  pl = choose_plan(d, kp.tiles_m, kp.total_kb, sms);
  LADI_CHECK(d->pair_mode != 1 || pl.pair, "pair_mode=1 needs >= 2 M tiles, BN >= 128 and no split-K (BN=%d, tiles_m=%d)", pl.bn, kp.tiles_m);
  kp.tiles_n = (d->c_out + pl.bn - 1) / pl.bn;
  kp.splits = pl.splits; kp.kb_per_split = pl.kb_per_split; kp.staged = pl.staged; kp.form = pl.form;
  kp.stages = pipeline_stages(pl.bn, pl.staged);
  LADI_CHECK(kp.stages >= 2, "not enough shared memory for a 2-stage pipeline");
  return LADI_OK;
}

}  // namespace

extern "C" int ladi_conv2d_plan(const ladi_conv_desc* d, int sms, ladi_conv_plan* out) {
  LADI_CHECK(out != nullptr, "plan output is null");
  KParams kp;
  Plan pl;
  if (const int rc = plan_conv(d, sms > 0 ? sms : ladi_num_sms(), kp, pl)) return rc;
  out->bn = pl.bn; out->splits = pl.splits; out->kb_per_split = pl.kb_per_split; out->pair = pl.pair; out->staged = pl.staged;
  out->stages = kp.stages; out->tiles_m = kp.tiles_m; out->tiles_n = kp.tiles_n; out->total_kb = kp.total_kb;
  return LADI_OK;
}

extern "C" int ladi_conv2d_bf16(const ladi_conv_desc* d, void* stream_) {
  KParams kp;
  Plan pl;
  if (const int rc = plan_conv(d, ladi_num_sms(), kp, pl)) return rc;

  // ---- the descriptor's epilogue operands -> kernel parameters
  kp.bias = d->bias; kp.bias_per_row = d->bias_per_row; kp.bias_step_stride = d->bias_step_stride; kp.step_ptr = d->step_ptr;
  kp.residual = reinterpret_cast<const bf16*>(d->residual); kp.residual_pitch = d->residual_pitch;
  kp.row_scale = d->row_scale; kp.act = d->act; kp.out = d->out; kp.out_pitch = d->out_pitch; kp.out_fp32 = d->out_fp32;
  kp.rowstat_out = reinterpret_cast<float2*>(d->rowstat_out); kp.rowstat_chunks = d->c_out / 32;
  kp.ln_stats = reinterpret_cast<const float2*>(d->ln_stats); kp.ln_chunks = d->src_c[0] / 32; kp.ln_colsum = d->ln_colsum; kp.ln_eps = d->ln_eps;
  if (pl.splits > 1) {  // fp32 partial planes to the workspace; bias, activation and residual move to splitk_reduce_kernel
    kp.split_stride = (long long)d->n * d->h_out * d->w_out * d->c_out;
    kp.out = d->splitk_ws; kp.out_pitch = d->c_out; kp.out_fp32 = 1;
    kp.bias = nullptr; kp.step_ptr = nullptr; kp.act = 0; kp.residual = nullptr;
  }
  AMaps am;
  if (const int rc = encode_a_maps(d, kp, am)) return rc;
  CUtensorMap tmB;
  if (const int rc = encode_b_map(d, pl, &tmB)) return rc;
  return launch_plan(d, pl, am, tmB, kp, reinterpret_cast<cudaStream_t>(stream_));
}

// Flash-style fused attention for sm_90a, bf16 in / bf16 out, fp32 softmax state; the score matrix never reaches memory.
//   S = Q K^T  : wgmma (M = 64 queries per warpgroup, N = BKV keys, both operands from 128B-swizzled shared memory) into registers;
//   softmax    : online max / sum in the exp2 domain on the accumulator fragment (a query row lives in the 4 lanes of a quad);
//   O += P V   : wgmma with P as the register A operand (the S fragment packed to bf16 is exactly the A fragment layout) and V
//                read MN-major straight from the TMA-loaded [keys][64] tile; O accumulates in registers.
// Q/K/V tiles arrive by TMA through 3-D tensor maps over [batch][tokens][row pitch], so per-head slices of the fused QKV
// projection output are read in place (no head split / transposes); out-of-range tokens are zero-filled and masked.
//
// Warpgroup 0 of a CTA is the TMA producer; every other warpgroup owns 64 query rows.
//   D = 64  (UNet attn1 / attn2, attention_d64_kernel): 192-row query tiles (three consumer warpgroups), BKV = 128 keys per tile,
//            the whole 64-wide value / output per CTA.  QK^T of the next key tile is issued before the softmax of the current one,
//            and the consumers take turns issuing MMAs, so softmax and tensor-core work overlap.
//   D = 512 (VAE mid-block, one head) and 256 (reduced-width test models, attention_kernel<D>): 128-row query tiles (two consumer
//            warpgroups), BKV = 64, and each CTA computes a 128-column slice of the output (blockIdx.y), which keeps the fp32 O
//            fragment at 64 registers per thread; S is recomputed per slice.  Each consumer issues QK^T, waits, runs the softmax,
//            then issues PV and waits.
//
// Replaces diffusers CrossAttention (attn1/attn2 of BasicTransformerBlock) inside UNet2DConditionModel.forward, which the
// reference runs through torch SDPA or xformers (src/inference.py:143-147; call-site tryon_pipe.py:732), and the VAE
// AttentionBlock (src/models/vae.py:81-90,112,142-150,187: baddbmm + softmax + bmm over the N x N matrix per sample).
#include "common.h"
#include "ptx.cuh"
#include "wgmma.cuh"

#include <algorithm>

namespace {

constexpr int BQ = 128;

struct AttnParams {
  int nq, nkv, n_kv_tiles;
  bf16* out;
  int out_pitch;
  int64_t out_batch_stride;
  float scale_log2;  // scale * log2(e)
  int n_q_tiles, heads, n_items;  // attention_d64_kernel: work items = n_q_tiles x heads x batch
};

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}

// ================================================================================================ D = 64 (UNet attn1 / attn2)
// 192 query rows per CTA: 192 divides every UNet level's token count at 512x384 (3072, 768, 192), and the third consumer warpgroup
// measured faster than 128 rows with two (DESIGN.md section 8).
struct Attn64 {
  static constexpr int NWG = 3;              // consumer warpgroups, 64 query rows each
  static constexpr int BQ = 64 * NWG;        // query rows per CTA
  static constexpr int BKV = 128;            // keys per K / V tile
  static constexpr int TILE = BKV * 128;     // bytes of one [BKV keys][64] tile
  static constexpr int STAGES = 4;           // K / V tiles in flight
  static constexpr int THREADS = 128 * (NWG + 1);
  static constexpr int REG_PRODUCER = 24, REG_CONSUMER = 160;  // setmaxnreg split of the 65536-register file
  static constexpr size_t SMEM = 2 * (size_t)BQ * 128 + 2 * (size_t)STAGES * TILE + (4 + 4 * STAGES) * 8 + 1024;
  static_assert(SMEM <= 232448, "over the 227 KiB per-CTA shared-memory limit");
  static_assert(REG_PRODUCER * 128 + REG_CONSUMER * 128 * NWG <= 65536, "register file over-committed");
};

// Online softmax of one [64 queries][BKV keys] S fragment in place (S -> unnormalised P in fp32): s[4 jj + 2 h + e] = row g + 8 h, key
// key0 + 8 jj + e.  Updates the running max m (scaled, exp2 domain) and this thread's partial row sum l; returns the rescale factor of O.
__device__ __forceinline__ void softmax_tile64(float (&s)[64], float (&m)[2], float (&l)[2], float (&alpha)[2], int key0, int key_end,
                                               int nkv, float scale_log2) {
  if (key_end > nkv) {
#pragma unroll
    for (int jj = 0; jj < 16; ++jj)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        if (key0 + 8 * jj + e >= nkv) { s[4 * jj + e] = -INFINITY; s[4 * jj + 2 + e] = -INFINITY; }
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float mx = -INFINITY;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
    mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
    const float m_new = fmaxf(m[h], mx * scale_log2);  // finite: every tile holds at least one valid key
    alpha[h] = ex2(m[h] - m_new);                     // 0 on the first tile (m = -inf)
    m[h] = m_new;
    float sum = 0.f;
#pragma unroll
    for (int jj = 0; jj < 16; ++jj) {
      const float p0 = ex2(fmaf(s[4 * jj + 2 * h], scale_log2, -m_new));
      const float p1 = ex2(fmaf(s[4 * jj + 2 * h + 1], scale_log2, -m_new));
      s[4 * jj + 2 * h] = p0; s[4 * jj + 2 * h + 1] = p1;
      sum += p0 + p1;
    }
    l[h] = l[h] * alpha[h] + sum;
  }
}

// Persistent: grid.x = min(work items, SMs); CTA c processes items c, c + gridDim.x, ...  An item is one (BQ-row query tile, head,
// image), numbered query tile fastest so that concurrently running CTAs share K / V in L2.  Warpgroup 0 is the TMA producer: per item
// it loads Q into one of two buffers, then K_j and V_j into a ring of STAGES K / V tile pairs, running ahead into the next item while
// the consumers finish the current one (its last tiles, the O / l epilogue).  Consumer warpgroup w owns query rows 64 w .. 64 w + 63
// of the tile.  Each consumer keeps one MMA group in flight while it works on the softmax:
//   S_0 = Q K_0^T; softmax_0
//   for j: issue S_{j+1} = Q K_{j+1}^T, then O += P_j V_j; wait S_{j+1} (PV_j still running) and release K_{j+1}; softmax_{j+1};
//          wait PV_j and release V_j; O *= alpha_{j+1}; pack P_{j+1}
// The consumers take turns issuing (ping-pong through named barriers 1 .. NWG, in warpgroup order, continued across items), so one
// warpgroup's softmax runs while another's MMAs occupy the tensor cores.  Per element the arithmetic and its order are those of the
// wide kernel below.
__global__ void __launch_bounds__(Attn64::THREADS, 1)
attention_d64_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                   const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnParams p) {
  using C = Attn64;
  constexpr int NWG = C::NWG, BQ64 = C::BQ, BKV = C::BKV, TILE = C::TILE, STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                        // 2 x [BQ rows][64]
  uint8_t* sK = sQ + 2 * BQ64 * 128;         // STAGES x [BKV keys][64]
  uint8_t* sV = sK + STAGES * TILE;          // STAGES x [BKV keys][64]
  uint64_t* bars = reinterpret_cast<uint64_t*>(sV + STAGES * TILE);
  const uint32_t q_full0 = ptx::smem_u32(bars), q_empty0 = q_full0 + 16, k_full0 = q_empty0 + 16, v_full0 = k_full0 + 8 * STAGES,
                 k_empty0 = v_full0 + 8 * STAGES, v_empty0 = k_empty0 + 8 * STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int n_tiles = p.n_kv_tiles;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ); ptx::prefetch_tmap(&tmK); ptx::prefetch_tmap(&tmV);
    for (int i = 0; i < 2; ++i) {
      ptx::mbar_init(q_full0 + 8 * i, 1);
      ptx::mbar_init(q_empty0 + 8 * i, NWG);
    }
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(k_full0 + 8 * s, 1);
      ptx::mbar_init(v_full0 + 8 * s, 1);
      ptx::mbar_init(k_empty0 + 8 * s, NWG);  // every consumer warpgroup reads every tile
      ptx::mbar_init(v_empty0 + 8 * s, NWG);
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::pdl_wait();

  if (wg == 0) {
    ptx::setmaxnreg_dec<C::REG_PRODUCER>();
    if (warp == 0) {
      int t = 0;  // K / V tiles loaded so far: ring stage t % STAGES, phase (t / STAGES) & 1
      for (int item = blockIdx.x, it = 0; item < p.n_items; item += gridDim.x, ++it) {
        const int qt = item % p.n_q_tiles, hb = item / p.n_q_tiles, col = 64 * (hb % p.heads), b = hb / p.heads;
        const uint32_t qf = q_full0 + 8 * (it & 1);
        ptx::mbar_wait(q_empty0 + 8 * (it & 1), ((it >> 1) & 1) ^ 1);
        if (ptx::elect_one()) {
          ptx::mbar_expect_tx(qf, BQ64 * 128);
          ptx::tma_load_3d(&tmQ, ptx::smem_u32(sQ + (it & 1) * BQ64 * 128), qf, col, qt * BQ64, b);
        }
        __syncwarp();
        for (int j = 0; j < n_tiles; ++j, ++t) {
          const int s = t % STAGES;
          const uint32_t ph = (t / STAGES) & 1;
          ptx::mbar_wait(k_empty0 + 8 * s, ph ^ 1);
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx(k_full0 + 8 * s, TILE);
            ptx::tma_load_3d(&tmK, ptx::smem_u32(sK + s * TILE), k_full0 + 8 * s, col, j * BKV, b);
          }
          __syncwarp();
          ptx::mbar_wait(v_empty0 + 8 * s, ph ^ 1);
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx(v_full0 + 8 * s, TILE);
            ptx::tma_load_3d(&tmV, ptx::smem_u32(sV + s * TILE), v_full0 + 8 * s, col, j * BKV, b);
          }
          __syncwarp();
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<C::REG_CONSUMER>();
    const int cw = wg - 1, q = lane & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    // ping-pong: this warpgroup issues after bar.sync on its barrier, which the previous warpgroup's bar.arrive completes (256 threads:
    // the 128 that wait and the 128 that arrive)
    const uint32_t my_turn = 1 + cw, next_turn = 1 + (cw + 1) % NWG;
    if (cw == NWG - 1) ptx::named_barrier_arrive(1, 256);  // warpgroup 0 issues first
    float o[32];
    float m[2], l[2];  // rows g and g + 8; l is this thread's partial row sum
    float s[BKV / 2], alpha[2];
    uint32_t pa[BKV / 16][4];  // P as bf16 A fragments, one per 16 keys
    uint64_t qd;
    auto issue_s = [&](int t) {
      const uint64_t kd = ptx::smem_desc_sw128(ptx::smem_u32(sK + (t % STAGES) * TILE));
#pragma unroll
      for (int k = 0; k < 4; ++k) ptx::Wgmma<BKV>::ss(s, qd + 2 * k, kd + 2 * k, k != 0);
      ptx::wgmma_commit();
    };
    auto issue_pv = [&](int t) {
      const uint64_t vd = ptx::smem_desc_sw128(ptx::smem_u32(sV + (t % STAGES) * TILE));
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk) ptx::Wgmma<64>::rs_bmn(o, pa[kk], vd + 128 * kk, 1);
      ptx::wgmma_commit();
    };
    auto pack_p = [&]() {
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk) {
        pa[kk][0] = ptx::pack_bf16(s[8 * kk], s[8 * kk + 1]);
        pa[kk][1] = ptx::pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
        pa[kk][2] = ptx::pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
        pa[kk][3] = ptx::pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
      }
    };
    auto rescale_o = [&]() {
#pragma unroll
      for (int jj = 0; jj < 8; ++jj) {
        o[4 * jj] *= alpha[0]; o[4 * jj + 1] *= alpha[0];
        o[4 * jj + 2] *= alpha[1]; o[4 * jj + 3] *= alpha[1];
      }
    };

    int t = 0;  // first K / V tile of the current item
    for (int item = blockIdx.x, it = 0; item < p.n_items; item += gridDim.x, ++it, t += n_tiles) {
      const int qt = item % p.n_q_tiles, hb = item / p.n_q_tiles, col = 64 * (hb % p.heads), b = hb / p.heads;
      const bool last_item = item + (int)gridDim.x >= p.n_items;
      const uint32_t q_empty = q_empty0 + 8 * (it & 1);
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = 0.f;
      m[0] = m[1] = -INFINITY;
      l[0] = l[1] = 0.f;
      qd = ptx::smem_desc_sw128(ptx::smem_u32(sQ + (it & 1) * BQ64 * 128) + cw * 64 * 128);
      ptx::mbar_wait(q_full0 + 8 * (it & 1), (it >> 1) & 1);

      // ---- prologue: S_0, softmax_0
      ptx::mbar_wait(k_full0 + 8 * (t % STAGES), (t / STAGES) & 1);
      ptx::named_barrier_sync(my_turn, 256);
      ptx::wgmma_fence();
      issue_s(t);
      ptx::named_barrier_arrive(next_turn, 256);
      ptx::wgmma_wait<0>();
      ptx::reg_fence(s);
      if (signaller) {
        ptx::mbar_arrive(k_empty0 + 8 * (t % STAGES));
        if (n_tiles == 1) ptx::mbar_arrive(q_empty);  // the item's last read of Q has completed
      }
      softmax_tile64(s, m, l, alpha, 2 * q, BKV, p.nkv, p.scale_log2);
      rescale_o();
      pack_p();

      for (int j = 0; j + 1 < n_tiles; ++j) {
        const int tv = t + j, tk = tv + 1;
        ptx::mbar_wait(k_full0 + 8 * (tk % STAGES), (tk / STAGES) & 1);
        ptx::mbar_wait(v_full0 + 8 * (tv % STAGES), (tv / STAGES) & 1);
        ptx::named_barrier_sync(my_turn, 256);
        ptx::wgmma_fence();
        issue_s(tk);
        issue_pv(tv);
        ptx::named_barrier_arrive(next_turn, 256);
        ptx::wgmma_wait<1>();
        ptx::reg_fence(s);
        if (signaller) {
          ptx::mbar_arrive(k_empty0 + 8 * (tk % STAGES));
          if (j + 2 == n_tiles) ptx::mbar_arrive(q_empty);
        }
        softmax_tile64(s, m, l, alpha, (j + 1) * BKV + 2 * q, (j + 2) * BKV, p.nkv, p.scale_log2);
        ptx::wgmma_wait<0>();
        ptx::reg_fence(o);
        if (signaller) ptx::mbar_arrive(v_empty0 + 8 * (tv % STAGES));
        rescale_o();
        pack_p();
      }
      // ---- last tile: PV only
      {
        const int tv = t + n_tiles - 1;
        ptx::mbar_wait(v_full0 + 8 * (tv % STAGES), (tv / STAGES) & 1);
        ptx::named_barrier_sync(my_turn, 256);
        ptx::wgmma_fence();
        issue_pv(tv);
        // the last turn of the last warpgroup hands over to no one
        if (!last_item || cw != NWG - 1) ptx::named_barrier_arrive(next_turn, 256);
        ptx::wgmma_wait<0>();
        ptx::reg_fence(o);
        if (signaller) ptx::mbar_arrive(v_empty0 + 8 * (tv % STAGES));
      }

      // ---- output: O / l
      const int g = 64 * cw + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float lt = l[h];
        lt += __shfl_xor_sync(0xffffffffu, lt, 1);
        lt += __shfl_xor_sync(0xffffffffu, lt, 2);
        const float inv = 1.f / lt;
        const int qi = qt * BQ64 + g + 8 * h;
        if (qi < p.nq) {
          bf16* orow = p.out + (size_t)b * p.out_batch_stride + (size_t)qi * p.out_pitch + col + 2 * q;
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
            *reinterpret_cast<uint32_t*>(orow + 8 * jj) = ptx::pack_bf16(o[4 * jj + 2 * h] * inv, o[4 * jj + 2 * h + 1] * inv);
        }
      }
    }
  }
  ptx::pdl_trigger();
}

// ================================================================================================ D = 512 / 256 (VAE mid-block)
template <int D> struct AttnCfg {
  static constexpr int BKV = 64;                          // keys per K/V tile
  static constexpr int VW = 128;                          // value / output columns per CTA
  static constexpr int KCH = D / 64, VCH = VW / 64;       // 64-column chunks of a K tile / of the value slice
  static constexpr int CHUNK = BKV * 128;                 // bytes of one [BKV keys][64] chunk
  static constexpr int STAGES = 10;                       // ring depth (>= KCH: S needs all K chunks of a tile at once)
  static constexpr size_t SMEM = (size_t)KCH * BQ * 128 + (size_t)STAGES * CHUNK + (1 + 2 * STAGES) * 8 + 1024;
  static_assert(STAGES >= KCH && STAGES >= VCH, "ring too shallow");
  static_assert(SMEM <= 232448, "over the 227 KiB per-CTA shared-memory limit");
};

// grid: (query tiles, 128-column output slices, batch)
template <int D>
__global__ void __launch_bounds__(384, 1)
attention_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                 const __grid_constant__ CUtensorMap tmV, const __grid_constant__ AttnParams p) {
  using C = AttnCfg<D>;
  constexpr int BKV = C::BKV, KCH = C::KCH, VCH = C::VCH, CHUNK = C::CHUNK, STAGES = C::STAGES;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~uintptr_t(1023));
  uint8_t* sQ = smem;                        // KCH chunks [128 rows][64]
  uint8_t* sR = sQ + KCH * BQ * 128;         // ring of [BKV keys][64] chunks
  uint64_t* bars = reinterpret_cast<uint64_t*>(sR + STAGES * CHUNK);
  const uint32_t q_full = ptx::smem_u32(bars), full0 = q_full + 8, empty0 = full0 + 8 * STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7;
  const int qt = blockIdx.x, b = blockIdx.z;
  // one head; blockIdx.y = 128-column slice of V and out
  const int col_qk = 0;
  const int col_v = C::VW * blockIdx.y;
  const int n_tiles = p.n_kv_tiles;

  if (threadIdx.x == 0) {
    ptx::prefetch_tmap(&tmQ); ptx::prefetch_tmap(&tmK); ptx::prefetch_tmap(&tmV);
    ptx::mbar_init(q_full, 1);
    for (int s = 0; s < STAGES; ++s) {
      ptx::mbar_init(full0 + 8 * s, 1);
      ptx::mbar_init(empty0 + 8 * s, 2);  // both consumer warpgroups read every chunk
    }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  ptx::pdl_wait();

  if (wg == 0) {
    ptx::setmaxnreg_dec<40>();
    if (warp == 0) {
      // ---------------------------------------------------------------- TMA producer: Q once, then per tile K chunks, V chunks
      if (ptx::elect_one()) {
        ptx::mbar_expect_tx(q_full, KCH * BQ * 128);
        for (int c = 0; c < KCH; ++c) ptx::tma_load_3d(&tmQ, ptx::smem_u32(sQ + c * BQ * 128), q_full, col_qk + 64 * c, qt * BQ, b);
      }
      __syncwarp();
      uint32_t stage = 0, phase = 0;
      for (int j = 0; j < n_tiles; ++j) {
        for (int c = 0; c < KCH + VCH; ++c) {
          ptx::mbar_wait(empty0 + 8 * stage, phase ^ 1);
          const uint32_t fb = full0 + 8 * stage;
          if (ptx::elect_one()) {
            ptx::mbar_expect_tx(fb, CHUNK);
            if (c < KCH) ptx::tma_load_3d(&tmK, ptx::smem_u32(sR + stage * CHUNK), fb, col_qk + 64 * c, j * BKV, b);
            else ptx::tma_load_3d(&tmV, ptx::smem_u32(sR + stage * CHUNK), fb, col_v + 64 * (c - KCH), j * BKV, b);
          }
          __syncwarp();
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<232>();
    // ------------------------------------------------------------------ consumers: 64 query rows per warpgroup
    const int cw = wg - 1, q = lane & 3;
    const bool signaller = (threadIdx.x & 127) == 0;
    float o[VCH][32];
#pragma unroll
    for (int c = 0; c < VCH; ++c)
#pragma unroll
      for (int i = 0; i < 32; ++i) o[c][i] = 0.f;
    float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};  // rows g and g + 8; l is this thread's partial row sum
    uint32_t stage = 0, phase = 0;
    ptx::mbar_wait(q_full, 0);
    const uint32_t q_base = ptx::smem_u32(sQ) + cw * 64 * 128;
    for (int j = 0; j < n_tiles; ++j) {
      // ---- S = Q K^T over the KCH d-chunks
      float s[BKV / 2];
      uint32_t kst[KCH];
      ptx::wgmma_fence();
#pragma unroll
      for (int c = 0; c < KCH; ++c) {
        ptx::mbar_wait(full0 + 8 * stage, phase);
        kst[c] = stage;
        const uint64_t qd = ptx::smem_desc_sw128(q_base + c * BQ * 128);
        const uint64_t kd = ptx::smem_desc_sw128(ptx::smem_u32(sR + stage * CHUNK));
#pragma unroll
        for (int k = 0; k < 4; ++k) ptx::Wgmma<BKV>::ss(s, qd + 2 * k, kd + 2 * k, (c | k) != 0);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
      ptx::reg_fence(s);
      if (signaller)
#pragma unroll
        for (int c = 0; c < KCH; ++c) ptx::mbar_arrive(empty0 + 8 * kst[c]);

      // ---- online softmax on the fragment: s[4 jj + 2 h + e] = row g + 8 h, key j*BKV + 8 jj + 2 q + e
      const int key0 = j * BKV + 2 * q;
      if (j * BKV + BKV > p.nkv) {
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj)
#pragma unroll
          for (int e = 0; e < 2; ++e)
            if (key0 + 8 * jj + e >= p.nkv) { s[4 * jj + e] = -INFINITY; s[4 * jj + 2 + e] = -INFINITY; }
      }
      float alpha[2];
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float mx = -INFINITY;
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj) mx = fmaxf(mx, fmaxf(s[4 * jj + 2 * h], s[4 * jj + 2 * h + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        const float m_new = fmaxf(m[h], mx * p.scale_log2);  // finite: every tile holds at least one valid key
        alpha[h] = ex2(m[h] - m_new);                       // 0 on the first tile (m = -inf)
        m[h] = m_new;
        float sum = 0.f;
#pragma unroll
        for (int jj = 0; jj < BKV / 8; ++jj) {
          const float p0 = ex2(fmaf(s[4 * jj + 2 * h], p.scale_log2, -m_new));
          const float p1 = ex2(fmaf(s[4 * jj + 2 * h + 1], p.scale_log2, -m_new));
          s[4 * jj + 2 * h] = p0; s[4 * jj + 2 * h + 1] = p1;
          sum += p0 + p1;
        }
        l[h] = l[h] * alpha[h] + sum;
      }
#pragma unroll
      for (int c = 0; c < VCH; ++c)
#pragma unroll
        for (int jj = 0; jj < 8; ++jj) {
          o[c][4 * jj] *= alpha[0]; o[c][4 * jj + 1] *= alpha[0];
          o[c][4 * jj + 2] *= alpha[1]; o[c][4 * jj + 3] *= alpha[1];
        }
      // P as bf16 A fragments, one per 16 keys
      uint32_t pa[BKV / 16][4];
#pragma unroll
      for (int kk = 0; kk < BKV / 16; ++kk) {
        pa[kk][0] = ptx::pack_bf16(s[8 * kk], s[8 * kk + 1]);
        pa[kk][1] = ptx::pack_bf16(s[8 * kk + 2], s[8 * kk + 3]);
        pa[kk][2] = ptx::pack_bf16(s[8 * kk + 4], s[8 * kk + 5]);
        pa[kk][3] = ptx::pack_bf16(s[8 * kk + 6], s[8 * kk + 7]);
      }

      // ---- O += P V over the value chunks
      uint32_t vst[VCH];
      ptx::wgmma_fence();
#pragma unroll
      for (int c = 0; c < VCH; ++c) {
        ptx::mbar_wait(full0 + 8 * stage, phase);
        vst[c] = stage;
        const uint64_t vd = ptx::smem_desc_sw128(ptx::smem_u32(sR + stage * CHUNK));
#pragma unroll
        for (int kk = 0; kk < BKV / 16; ++kk) ptx::Wgmma<64>::rs_bmn(o[c], pa[kk], vd + 128 * kk, 1);
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>();
#pragma unroll
      for (int c = 0; c < VCH; ++c) ptx::reg_fence(o[c]);
      if (signaller)
#pragma unroll
        for (int c = 0; c < VCH; ++c) ptx::mbar_arrive(empty0 + 8 * vst[c]);
    }

    // ---- output: O / l
    const int g = 64 * cw + 16 * (warp & 3) + (lane >> 2);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float lt = l[h];
      lt += __shfl_xor_sync(0xffffffffu, lt, 1);
      lt += __shfl_xor_sync(0xffffffffu, lt, 2);
      const float inv = 1.f / lt;
      const int qi = qt * BQ + g + 8 * h;
      if (qi < p.nq) {
        bf16* orow = p.out + (size_t)b * p.out_batch_stride + (size_t)qi * p.out_pitch + col_v + 2 * q;
#pragma unroll
        for (int c = 0; c < VCH; ++c)
#pragma unroll
          for (int jj = 0; jj < 8; ++jj)
            *reinterpret_cast<uint32_t*>(orow + 64 * c + 8 * jj) = ptx::pack_bf16(o[c][4 * jj + 2 * h] * inv, o[c][4 * jj + 2 * h + 1] * inv);
      }
    }
  }
  ptx::pdl_trigger();
}

int make_map(CUtensorMap* m, const void* ptr, int cols, int tokens, int batch, int pitch, int64_t batch_stride, int box_rows) {
  const uint64_t dims[3] = {(uint64_t)cols, (uint64_t)tokens, (uint64_t)batch};
  const uint64_t strides[2] = {(uint64_t)pitch * 2, (uint64_t)batch_stride * 2};
  const uint32_t box[3] = {64u, (uint32_t)box_rows, 1u};
  return ladi_encode_tmap_bf16(m, ptr, 3, dims, strides, box);
}

template <int D>
int launch(const ladi_attn_desc* d, const ladi_attn_plan& pl, cudaStream_t stream) {
  using C = AttnCfg<D>;
  static bool attr_set = false;
  if (!attr_set) {
    LADI_CUDA(cudaFuncSetAttribute(attention_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    attr_set = true;
  }
  CUtensorMap tq, tk, tv;
  if (make_map(&tq, d->q, D, d->nq, d->batch, d->q_pitch, d->q_batch_stride, BQ)) return LADI_ERR_CUDA;
  if (make_map(&tk, d->k, D, d->nkv, d->batch, d->k_pitch, d->k_batch_stride, C::BKV)) return LADI_ERR_CUDA;
  if (make_map(&tv, d->v, D, d->nkv, d->batch, d->v_pitch, d->v_batch_stride, C::BKV)) return LADI_ERR_CUDA;
  AttnParams p;
  p.nq = d->nq; p.nkv = d->nkv; p.n_kv_tiles = pl.n_kv_tiles;
  p.out = reinterpret_cast<bf16*>(d->out); p.out_pitch = d->out_pitch; p.out_batch_stride = d->out_batch_stride;
  p.scale_log2 = d->scale * 1.4426950408889634f;
  LADI_CUDA(ladi_launch(attention_kernel<D>, dim3(pl.grid_x, pl.grid_y, pl.grid_z), dim3(384), C::SMEM, stream, tq, tk, tv, p));
  return LADI_OK;
}

bool aligned_to(const void* p, uintptr_t bytes) { return (reinterpret_cast<uintptr_t>(p) & (bytes - 1)) == 0; }

// Everything the two attention launches decide from the descriptor and the SM count alone (no pointer is dereferenced, nothing touches
// a device): validation, the kernel's tile constants and its grid.  ladi_attention_plan reports it; ladi_attention_bf16 (wide = 0) and
// ladi_attention_d512_bf16 (wide = 1) launch it.  Q, K and V are read by TMA (16-byte aligned base, strides multiples of 16 bytes); both
// kernels store the output as bf16 pairs (4 bytes): out must be 4-byte aligned and every batch's rows start on a pair.
int attn_plan(const ladi_attn_desc* d, int wide, int sms, ladi_attn_plan& pl) {
  LADI_CHECK(d != nullptr && d->q && d->k && d->v && d->out, "null attention operand");
  if (wide) {
    LADI_CHECK(d->batch > 0 && d->heads == 1 && d->nq > 0 && d->nkv > 0, "d512 attention: one head, non-empty extents");
  } else {
    LADI_CHECK(d->batch > 0 && d->heads > 0 && d->nq > 0 && d->nkv > 0, "bad attention extent");
  }
  LADI_CHECK(d->q_pitch % 8 == 0 && d->k_pitch % 8 == 0 && d->v_pitch % 8 == 0 && d->out_pitch % 8 == 0, "pitches must be multiples of 8");
  const int D = wide ? (d->head_dim == 0 ? 512 : d->head_dim) : 64;
  if (wide) {
    LADI_CHECK(D == 512 || D == 256, "wide attention: head_dim must be 512 (or 256), got %d", D);
    LADI_CHECK(d->q_pitch >= D && d->k_pitch >= D && d->v_pitch >= D && d->out_pitch >= D, "pitch < head_dim");
  } else {
    LADI_CHECK(d->q_pitch >= d->heads * 64 && d->k_pitch >= d->heads * 64 && d->v_pitch >= d->heads * 64 && d->out_pitch >= d->heads * 64,
               "pitch < heads*64");
  }
  LADI_CHECK(aligned_to(d->q, 16), "q %p must be 16-byte aligned (TMA)", d->q);
  LADI_CHECK(aligned_to(d->k, 16), "k %p must be 16-byte aligned (TMA)", d->k);
  LADI_CHECK(aligned_to(d->v, 16), "v %p must be 16-byte aligned (TMA)", d->v);
  LADI_CHECK(d->q_batch_stride % 8 == 0, "q_batch_stride %lld must be a multiple of 8 (TMA)", (long long)d->q_batch_stride);
  LADI_CHECK(d->k_batch_stride % 8 == 0, "k_batch_stride %lld must be a multiple of 8 (TMA)", (long long)d->k_batch_stride);
  LADI_CHECK(d->v_batch_stride % 8 == 0, "v_batch_stride %lld must be a multiple of 8 (TMA)", (long long)d->v_batch_stride);
  LADI_CHECK(aligned_to(d->out, 4), "out %p must be 4-byte aligned", d->out);
  LADI_CHECK(d->out_batch_stride % 2 == 0, "out_batch_stride %lld must be even", (long long)d->out_batch_stride);
  if (!wide)
    LADI_CHECK(d->variant == 0 || d->variant == 1 || d->variant == 2 || d->variant == 4 || d->variant == 5 || d->variant == 6 ||
                   (d->variant == 8 && d->nkv <= 128),
               "bad attention variant %d", d->variant);
  pl.head_dim = D;
  if (wide) {
    pl.q_tile = BQ; pl.kv_tile = 64; pl.consumers = 2;
    pl.stages = D == 512 ? AttnCfg<512>::STAGES : AttnCfg<256>::STAGES;
    pl.smem_bytes = (int)(D == 512 ? AttnCfg<512>::SMEM : AttnCfg<256>::SMEM);
  } else {
    pl.q_tile = Attn64::BQ; pl.kv_tile = Attn64::BKV; pl.consumers = Attn64::NWG; pl.stages = Attn64::STAGES;
    pl.smem_bytes = (int)Attn64::SMEM;
  }
  pl.n_q_tiles = (d->nq + pl.q_tile - 1) / pl.q_tile;
  pl.n_kv_tiles = (d->nkv + pl.kv_tile - 1) / pl.kv_tile;
  const int last_rows = d->nq - (pl.n_q_tiles - 1) * pl.q_tile;
  pl.idle_consumers_last_q_tile = pl.consumers - (last_rows + 63) / 64;
  if (wide) {
    pl.grid_x = pl.n_q_tiles; pl.grid_y = D / 128; pl.grid_z = d->batch;
    pl.n_items = pl.grid_x * pl.grid_y * pl.grid_z;
    pl.items_min = pl.items_max = 1;
  } else {
    // persistent: at most one CTA per SM (the kernel's registers and shared memory allow no second one)
    pl.n_items = pl.n_q_tiles * d->heads * d->batch;
    pl.grid_x = std::min(pl.n_items, sms); pl.grid_y = pl.grid_z = 1;
    pl.items_min = pl.n_items / pl.grid_x;
    pl.items_max = (pl.n_items + pl.grid_x - 1) / pl.grid_x;
  }
  return LADI_OK;
}

}  // namespace

extern "C" int ladi_attention_plan(const ladi_attn_desc* d, int wide, int sms, ladi_attn_plan* out) {
  LADI_CHECK(out != nullptr, "plan output is null");
  return attn_plan(d, wide, sms > 0 ? sms : ladi_num_sms(), *out);
}

extern "C" int ladi_attention_bf16(const ladi_attn_desc* d, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ladi_attn_plan pl;
  if (const int rc = attn_plan(d, 0, ladi_num_sms(), pl)) return rc;
  using C = Attn64;
  static bool attr_set = false;
  if (!attr_set) {
    LADI_CUDA(cudaFuncSetAttribute(attention_d64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)C::SMEM));
    attr_set = true;
  }
  const int cols = d->heads * 64;
  CUtensorMap tq, tk, tv;
  if (make_map(&tq, d->q, cols, d->nq, d->batch, d->q_pitch, d->q_batch_stride, C::BQ)) return LADI_ERR_CUDA;
  if (make_map(&tk, d->k, cols, d->nkv, d->batch, d->k_pitch, d->k_batch_stride, C::BKV)) return LADI_ERR_CUDA;
  if (make_map(&tv, d->v, cols, d->nkv, d->batch, d->v_pitch, d->v_batch_stride, C::BKV)) return LADI_ERR_CUDA;
  AttnParams p;
  p.nq = d->nq; p.nkv = d->nkv; p.n_kv_tiles = pl.n_kv_tiles;
  p.out = reinterpret_cast<bf16*>(d->out); p.out_pitch = d->out_pitch; p.out_batch_stride = d->out_batch_stride;
  p.scale_log2 = d->scale * 1.4426950408889634f;
  p.n_q_tiles = pl.n_q_tiles; p.heads = d->heads; p.n_items = pl.n_items;
  LADI_CUDA(ladi_launch(attention_d64_kernel, dim3(pl.grid_x, pl.grid_y, pl.grid_z), dim3(C::THREADS), C::SMEM, stream, tq, tk, tv, p));
  return LADI_OK;
}

extern "C" int ladi_attention_d512_bf16(const ladi_attn_desc* d, void* stream_) {
  cudaStream_t stream = reinterpret_cast<cudaStream_t>(stream_);
  ladi_attn_plan pl;
  if (const int rc = attn_plan(d, 1, ladi_num_sms(), pl)) return rc;
  return pl.head_dim == 512 ? launch<512>(d, pl, stream) : launch<256>(d, pl, stream);
}

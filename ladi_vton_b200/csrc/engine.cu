// Module-level C ABI (SURVEY.md section 8(b), "what the .so must export"): an opaque per-device engine handle built from packed
// weights + a static architecture config, and one entry point per module of the try-on path -- UNet forward, VAE encode, VAE decode
// with the EMASC skips, EMASC, inversion adapter, the denoise loop -- each taking caller-owned device pointers, explicit shapes, a
// caller-supplied workspace (size query: ladi_workspace_bytes) and an explicit stream.  Nothing here allocates, synchronises or uses
// an implicit stream (the two scratch buffers every call shares -- split-K partials, GroupNorm statistics -- are allocated once in
// ladi_engine_create), so every call is CUDA-graph capturable; errors come back as codes + ladi_last_error().
//
// The launch sequences are the reference's module forwards re-expressed over the kernels of this library:
//   UNet2DConditionModel.forward (diffusers 0.14, built hubconf.py:30-37, called tryon_pipe.py:732)       -> unet_forward
//   Encoder.forward / AutoencoderKL.encode (src/models/vae.py:99-119, AutoencoderKL.py:145-157)             -> vae_encode
//   Decoder.forward / AutoencoderKL.decode with intermediate features (vae.py:183-212, AutoencoderKL.py:159-188) -> vae_decode
//   EMASC.forward + mask_features (src/models/emasc.py:37-40, src/utils/data_utils.py:4-16)                 -> emasc_forward
//   InversionAdapter.forward (src/models/inversion_adapter.py:22-28)                                        -> adapter_forward
// Every module body is written ONCE against a small `Ctx` that either launches (run mode) or only walks the allocator (plan mode:
// workspace sizing, and an op trace the CPU test-suite compares with the Python sequencing in ladi_vton_b200/{unet,vae,adapter}.py).
#include <stdarg.h>
#include <string.h>

#include <map>
#include <string>
#include <unordered_map>
#include <vector>

#include "common.h"

namespace {

// ------------------------------------------------------------------------------------------------------------------ allocator
// Offsets inside the caller's workspace; best-fit free list with coalescing.  The module bodies allocate and free in a fixed order, so
// the layout (and the high-water mark reported by ladi_workspace_bytes) is a pure function of (module, shape).
struct Arena {
  uint8_t* base = nullptr;
  size_t cap = 0, high = 0;
  std::map<size_t, size_t> free_;                 // offset -> size
  std::unordered_map<size_t, size_t> live_;       // offset -> size
  void reset(void* b, size_t c) {
    base = reinterpret_cast<uint8_t*>(b); cap = c; high = 0;
    free_.clear(); live_.clear();
    free_[0] = c;
  }
  void* alloc(size_t bytes) {
    bytes = (bytes + 255) & ~size_t(255);
    if (bytes == 0) bytes = 256;
    auto best = free_.end();
    for (auto it = free_.begin(); it != free_.end(); ++it)
      if (it->second >= bytes && (best == free_.end() || it->second < best->second)) best = it;
    if (best == free_.end()) return nullptr;
    const size_t off = best->first, sz = best->second;
    free_.erase(best);
    if (sz > bytes) free_[off + bytes] = sz - bytes;
    live_[off] = bytes;
    if (off + bytes > high) high = off + bytes;
    return base + off;
  }
  void release(const void* p) {
    if (p == nullptr) return;
    const size_t off = reinterpret_cast<const uint8_t*>(p) - base;
    auto it = live_.find(off);
    if (it == live_.end()) return;
    size_t o = off, sz = it->second;
    live_.erase(it);
    auto nx = free_.lower_bound(o);
    if (nx != free_.end() && o + sz == nx->first) { sz += nx->second; nx = free_.erase(nx); }
    if (nx != free_.begin()) {
      auto pv = std::prev(nx);
      if (pv->first + pv->second == o) { o = pv->first; sz += pv->second; free_.erase(pv); }
    }
    free_[o] = sz;
  }
};

struct Weight {
  const void* p = nullptr;
  int rows = 0, cols = 0;  // bf16 matrices: [rows][cols] (cols = K = row pitch); fp32 vectors: rows = 1
};

// NHWC bf16 (or fp32) activation view: pixel (n, y, x) at p + ((n*h + y)*w + x) * pitch elements
struct T {
  void* p = nullptr;
  int n = 0, h = 0, w = 0, c = 0, pitch = 0;
  bool f32 = false, owned = false;
  size_t rows() const { return (size_t)n * h * w; }
  T slice(int c0, int cn) const {
    T t = *this;
    t.p = reinterpret_cast<uint8_t*>(p) + (size_t)c0 * (f32 ? 4 : 2);
    t.c = cn; t.owned = false;
    return t;
  }
  T as_rows() const {  // [1, 1, rows, c]
    T t = *this;
    t.w = (int)rows(); t.n = 1; t.h = 1;
    return t;
  }
  T as_image(int n_, int h_, int w_) const {
    T t = *this;
    t.n = n_; t.h = h_; t.w = w_;
    return t;
  }
};

struct Engine {
  ladi_engine_config cfg;
  std::unordered_map<std::string, Weight> w;
  std::vector<std::pair<std::string, int>> resnets, transformers;  // (prefix, width) in forward order
  std::unordered_map<std::string, int> temb_off, kv_off;
  int temb_total = 0, kv_total = 0, in_pitch = 0;
  void* splitk_ws = nullptr;
  size_t splitk_bytes = 0;
  float* gn_ws = nullptr;
  size_t gn_floats = 0;
  std::string trace;  // last plan-mode op trace (ladi_engine_trace)
};

struct ConvOpt {
  int ksize = 3, stride = 1, pad_lo = 1;
  const float* bias = nullptr;
  int bias_per_row = 0, bias_step_stride = 0;
  const int* step_ptr = nullptr;
  const T* residual = nullptr;
  const float* row_scale = nullptr;
  int act = 0;
  bool out_fp32 = false, up2x = false;
  const T* out = nullptr;  // write into this view instead of allocating
  const T* sc0 = nullptr;  // fused 1x1 shortcut sources
  const T* sc1 = nullptr;
};

struct Ctx {
  Engine* e;
  Arena arena;
  cudaStream_t st;
  bool plan;
  int rc = LADI_OK;
  std::string* trace = nullptr;
  bool ok() const { return rc == LADI_OK; }
  void fail(const char* fmt, ...) {
    if (rc != LADI_OK) return;
    char buf[384];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    ladi_set_error("%s", buf);
    rc = LADI_ERR_INVALID;
  }
  void rec(const char* fmt, ...) {
    if (trace == nullptr) return;
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    trace->append(buf);
    trace->push_back('\n');
  }
  // traces print raw addresses; the test-suite renames them by order of first appearance before comparing with the Python sequencing
  static unsigned long long A(const void* p) { return (unsigned long long)reinterpret_cast<uintptr_t>(p); }
  const Weight& W(const std::string& name) {
    static Weight none;
    auto it = e->w.find(name);
    if (it == e->w.end()) {
      fail("engine: weight '%s' not in the table", name.c_str());
      return none;
    }
    return it->second;
  }
  const float* F(const std::string& name) { return reinterpret_cast<const float*>(W(name).p); }
  T make(int n, int h, int w, int c, bool f32 = false) {
    T t;
    t.n = n; t.h = h; t.w = w; t.c = c; t.f32 = f32;
    t.pitch = (f32 || c % 8 == 0) ? c : (c + 7) / 8 * 8;
    t.p = arena.alloc(t.rows() * t.pitch * (f32 ? 4 : 2));
    t.owned = true;
    if (t.p == nullptr) fail("engine: workspace too small (need more than %zu bytes; query ladi_workspace_bytes)", arena.cap);
    return t;
  }
  void drop(T& t) {
    if (t.owned) arena.release(t.p);
    t.p = nullptr; t.owned = false;
  }

  // ---------------------------------------------------------------------------------------------------------------- ops
  T conv(const T* s0, const T* s1, const Weight& wt, int c_out, const ConvOpt& o) {
    T out;
    if (!ok()) return out;
    const int n = s0->n, h_in = s0->h, w_in = s0->w;
    int h_out = h_in, w_out = w_in;
    if (o.up2x) { h_out = 2 * h_in; w_out = 2 * w_in; }
    else if (o.ksize == 3 && o.stride == 2) {
      h_out = (h_in + (o.pad_lo == 1 ? 2 : 1) - 3) / 2 + 1;
      w_out = (w_in + (o.pad_lo == 1 ? 2 : 1) - 3) / 2 + 1;
    }
    const int c_eff = o.act == LADI_ACT_GEGLU ? c_out / 2 : c_out;
    if (o.out != nullptr) out = *o.out, out.owned = false;
    else out = make(n, h_out, w_out, c_eff, o.out_fp32);
    if (!ok()) return out;
    ladi_conv_desc d;
    memset(&d, 0, sizeof(d));
    d.n = n; d.h_out = h_out; d.w_out = w_out; d.c_out = c_out; d.h_in = h_in; d.w_in = w_in;
    d.ksize = o.ksize; d.stride = o.stride; d.pad_lo = o.pad_lo; d.up2x = o.up2x ? 1 : 0;
    d.n_src = s1 != nullptr ? 2 : 1;
    d.src[0] = s0->p; d.src_c[0] = s0->c; d.src_pitch[0] = s0->pitch;
    if (s1 != nullptr) { d.src[1] = s1->p; d.src_c[1] = s1->c; d.src_pitch[1] = s1->pitch; }
    if (o.sc0 != nullptr) { d.sc[d.n_sc] = o.sc0->p; d.sc_c[d.n_sc] = o.sc0->c; d.sc_pitch[d.n_sc] = o.sc0->pitch; ++d.n_sc; }
    if (o.sc1 != nullptr) { d.sc[d.n_sc] = o.sc1->p; d.sc_c[d.n_sc] = o.sc1->c; d.sc_pitch[d.n_sc] = o.sc1->pitch; ++d.n_sc; }
    d.weight = wt.p; d.k_total = wt.cols; d.weight_pitch = wt.cols;
    d.bias = o.bias; d.bias_per_row = o.bias_per_row; d.bias_step_stride = o.bias_step_stride; d.step_ptr = o.step_ptr;
    if (o.residual != nullptr) { d.residual = o.residual->p; d.residual_pitch = o.residual->pitch; }
    d.row_scale = o.row_scale; d.act = o.act;
    d.out = out.p; d.out_pitch = out.pitch; d.out_fp32 = o.out_fp32 ? 1 : 0;
    d.splitk_ws = e->splitk_ws; d.splitk_ws_bytes = (int64_t)e->splitk_bytes;
    rec("conv k=%d s=%d p=%d up=%d n=%d h=%d w=%d hin=%d win=%d cout=%d nsrc=%d src0=@%llx c0=%d p0=%d src1=@%llx c1=%d p1=%d nsc=%d sc0=@%llx sc0c=%d sc0p=%d sc1=@%llx sc1c=%d sc1p=%d "
        "wt=@%llx K=%d wp=%d bias=@%llx bpr=%d bss=%d step=@%llx res=@%llx rp=%d rs=@%llx act=%d out=@%llx op=%d f32=%d",
        d.ksize, d.stride, d.pad_lo, d.up2x, d.n, d.h_out, d.w_out, d.h_in, d.w_in, d.c_out, d.n_src, A(d.src[0]), d.src_c[0], d.src_pitch[0], A(d.src[1]), d.src_c[1],
        d.src_pitch[1], d.n_sc, A(d.sc[0]), d.sc_c[0], d.sc_pitch[0], A(d.sc[1]), d.sc_c[1], d.sc_pitch[1], A(d.weight), d.k_total, d.weight_pitch, A(d.bias),
        d.bias_per_row, d.bias_step_stride, A(d.step_ptr), A(d.residual), d.residual_pitch, A(d.row_scale), d.act, A(d.out), d.out_pitch, d.out_fp32);
    if (!plan) {
      const int r = ladi_conv2d_bf16(&d, st);
      if (r != LADI_OK) rc = r;
    }
    return out;
  }
  T gemm(const T& a, const Weight& wt, int n_out, ConvOpt o = ConvOpt()) {
    o.ksize = 1; o.stride = 1;
    const T a4 = a.as_rows();
    T out4, res4;
    if (o.out != nullptr) { out4 = o.out->as_rows(); o.out = &out4; }
    if (o.residual != nullptr) { res4 = o.residual->as_rows(); o.residual = &res4; }
    return conv(&a4, nullptr, wt, n_out, o);
  }
  T groupnorm(const T* s0, const T* s1, const std::string& name, float eps, bool silu, const T* add = nullptr) {
    T out;
    if (!ok()) return out;
    const int n = s0->n, hw = s0->h * s0->w, groups = e->cfg.norm_groups;
    const int c1 = s1 != nullptr ? s1->c : 0;
    out = make(n, s0->h, s0->w, s0->c + c1);
    if (!ok()) return out;
    const size_t need = (size_t)n * ladi_groupnorm_chunks(hw) * groups * 2;
    if (need > e->gn_floats) { fail("engine: GroupNorm statistics workspace too small for batch %d", n); return out; }
    const float* gamma = F(name + ".0");
    const float* beta = F(name + ".1");
    rec("gn_stats x0=@%llx c0=%d p0=%d x1=@%llx c1=%d p1=%d n=%d hw=%d groups=%d", A(s0->p), s0->c, s0->pitch, A(s1 ? s1->p : nullptr), c1, s1 ? s1->pitch : 0, n, hw, groups);
    rec("gn_apply x0=@%llx c0=%d p0=%d x1=@%llx c1=%d p1=%d n=%d hw=%d groups=%d gamma=@%llx beta=@%llx eps=%.3g silu=%d add=@%llx ap=%d out=@%llx op=%d", A(s0->p), s0->c,
        s0->pitch, A(s1 ? s1->p : nullptr), c1, s1 ? s1->pitch : 0, n, hw, groups, A(gamma), A(beta), (double)eps, silu ? 1 : 0, A(add ? add->p : nullptr),
        add ? add->pitch : 0, A(out.p), out.pitch);
    if (!plan && ok()) {
      int r = ladi_groupnorm_stats(s0->p, s0->c, s0->pitch, s1 ? s1->p : nullptr, c1, s1 ? s1->pitch : 0, n, hw, groups, e->gn_ws, st);
      if (r == LADI_OK)
        r = ladi_groupnorm_apply(s0->p, s0->c, s0->pitch, s1 ? s1->p : nullptr, c1, s1 ? s1->pitch : 0, n, hw, groups, e->gn_ws, gamma, beta, eps, silu ? 1 : 0,
                                 add ? add->p : nullptr, add ? add->pitch : 0, out.p, out.pitch, st);
      if (r != LADI_OK) rc = r;
    }
    return out;
  }
  T layernorm(const T& x, const std::string& name, float eps) {
    T out;
    if (!ok()) return out;
    out = make(x.n, x.h, x.w, x.c);
    if (!ok()) return out;
    const float* gamma = F(name + ".0");
    const float* beta = F(name + ".1");
    rec("ln x=@%llx xp=%d rows=%d c=%d gamma=@%llx beta=@%llx eps=%.3g out=@%llx op=%d", A(x.p), x.pitch, (int)x.rows(), x.c, A(gamma), A(beta), (double)eps, A(out.p), out.pitch);
    if (!plan && ok()) {
      const int r = ladi_layernorm(x.p, x.pitch, (int)x.rows(), x.c, gamma, beta, eps, out.p, out.pitch, st);
      if (r != LADI_OK) rc = r;
    }
    return out;
  }
  // q/k/v: token views [B, tokens, >= heads*64] given as T with n = B, h = 1, w = tokens
  T attention(const T& q, const T& k, const T& v, int heads, float scale, int head_dim = 64) {
    T out;
    if (!ok()) return out;
    const int width = head_dim == 64 ? heads * 64 : head_dim;
    out = make(q.n, 1, q.w, width);
    if (!ok()) return out;
    ladi_attn_desc d;
    memset(&d, 0, sizeof(d));
    d.batch = q.n; d.heads = heads; d.nq = q.w; d.nkv = k.w;
    d.q = q.p; d.q_pitch = q.pitch; d.q_batch_stride = (int64_t)q.w * q.pitch;
    d.k = k.p; d.k_pitch = k.pitch; d.k_batch_stride = (int64_t)k.w * k.pitch;
    d.v = v.p; d.v_pitch = v.pitch; d.v_batch_stride = (int64_t)v.w * v.pitch;
    d.out = out.p; d.out_pitch = out.pitch; d.out_batch_stride = (int64_t)out.w * out.pitch;
    d.scale = scale; d.head_dim = head_dim == 64 ? 0 : head_dim;
    rec("attn d=%d batch=%d heads=%d nq=%d nkv=%d q=@%llx qp=%d qbs=%lld k=@%llx kp=%d kbs=%lld v=@%llx vp=%d vbs=%lld out=@%llx op=%d obs=%lld scale=%.6g", head_dim, d.batch,
        d.heads, d.nq, d.nkv, A(d.q), d.q_pitch, (long long)d.q_batch_stride, A(d.k), d.k_pitch, (long long)d.k_batch_stride, A(d.v), d.v_pitch, (long long)d.v_batch_stride,
        A(d.out), d.out_pitch, (long long)d.out_batch_stride, (double)d.scale);
    if (!plan) {
      const int r = head_dim == 64 ? ladi_attention_bf16(&d, st) : ladi_attention_d512_bf16(&d, st);
      if (r != LADI_OK) rc = r;
    }
    return out;
  }
  T add(const T& a, const T& b) {
    T out;
    if (!ok()) return out;
    if (a.pitch != a.c || b.pitch != b.c || a.c != b.c || a.rows() != b.rows()) { fail("engine: add needs dense equal tensors"); return out; }
    out = make(a.n, a.h, a.w, a.c);
    if (!ok()) return out;
    rec("add a=@%llx b=@%llx out=@%llx count=%lld", A(a.p), A(b.p), A(out.p), (long long)(a.rows() * a.c));
    if (!plan) {
      const int r = ladi_add_bf16(a.p, b.p, out.p, (int64_t)(a.rows() * a.c), st);
      if (r != LADI_OK) rc = r;
    }
    return out;
  }
  T upsample2x(const T& x) {
    T out;
    if (!ok()) return out;
    out = make(x.n, 2 * x.h, 2 * x.w, x.c);
    if (!ok()) return out;
    rec("upsample2x x=@%llx n=%d h=%d w=%d c=%d out=@%llx", A(x.p), x.n, x.h, x.w, x.c, A(out.p));
    if (!plan) {
      const int r = ladi_upsample2x_nhwc(x.p, x.n, x.h, x.w, x.c, out.p, st);
      if (r != LADI_OK) rc = r;
    }
    return out;
  }
};

std::string fmt(const char* f, ...) {
  char buf[256];
  va_list ap;
  va_start(ap, f);
  vsnprintf(buf, sizeof(buf), f, ap);
  va_end(ap);
  return buf;
}

// =================================================================================================================== UNet
// ResnetBlock2D (SURVEY App. A.3): GN+SiLU -> conv1 (+ per-step time-embedding bias table) -> GN+SiLU -> conv2 with the skip as an
// epilogue residual, or -- when the width changes -- the 1x1 conv_shortcut as extra K segments of the same accumulation.
T unet_resnet(Ctx& c, const std::string& p, const T* s0, const T* s1, int co, const float* steps, const int* step_ptr) {
  const float eps = c.e->cfg.unet_norm_eps;
  T hn = c.groupnorm(s0, s1, p + ".n1", eps, true);
  ConvOpt o1;
  o1.bias = steps + c.e->temb_off[p]; o1.bias_step_stride = c.e->temb_total; o1.step_ptr = step_ptr;
  T h = c.conv(&hn, nullptr, c.W(p + ".w1"), co, o1);
  c.drop(hn);
  T hn2 = c.groupnorm(&h, nullptr, p + ".n2", eps, true);
  c.drop(h);
  ConvOpt o2;
  o2.bias = c.F(p + ".b2");
  const int ci = s0->c + (s1 ? s1->c : 0);
  if (ci != co) { o2.sc0 = s0; o2.sc1 = s1; }
  else o2.residual = s0;
  T out = c.conv(&hn2, nullptr, c.W(p + ".w2"), co, o2);
  c.drop(hn2);
  return out;
}

// Transformer2DModel with one BasicTransformerBlock (SURVEY App. A.4): GN -> proj_in -> [LN -> QKV -> self-attention -> to_out + x]
// -> [LN -> Q -> cross-attention over the pre-projected text K/V -> to_out + x] -> [LN -> GEGLU -> ff2 + x] -> proj_out + input.
T unet_transformer(Ctx& c, const std::string& p, const T& x, int heads, const T& ctx_kv) {
  const int B = x.n, h = x.h, w = x.w, C = x.c, N = h * w;
  const std::string b = p + ".transformer_blocks.0";
  const float scale = 1.0f / sqrtf((float)(C / heads));
  T hn = c.groupnorm(&x, nullptr, p + ".norm", 1e-6f, false);
  ConvOpt o;
  o.bias = c.F(p + ".proj_in.b");
  T t = c.gemm(hn, c.W(p + ".proj_in.w"), C, o);
  c.drop(hn);
  T l1 = c.layernorm(t, b + ".ln1", 1e-5f);
  T qkv = c.gemm(l1, c.W(b + ".qkv"), 3 * C);
  c.drop(l1);
  const T qkv_t = qkv.as_image(B, 1, N);
  T a = c.attention(qkv_t.slice(0, C), qkv_t.slice(C, C), qkv_t.slice(2 * C, C), heads, scale);
  c.drop(qkv);
  ConvOpt o1;
  o1.bias = c.F(b + ".o1.b"); o1.residual = &t;
  T t2 = c.gemm(a, c.W(b + ".o1.w"), C, o1);
  c.drop(a); c.drop(t);
  T l2 = c.layernorm(t2, b + ".ln2", 1e-5f);
  T q = c.gemm(l2, c.W(b + ".q2"), C);
  c.drop(l2);
  const int off = c.e->kv_off[p];
  T a2 = c.attention(q.as_image(B, 1, N), ctx_kv.slice(off, C), ctx_kv.slice(off + C, C), heads, scale);
  c.drop(q);
  ConvOpt o2;
  o2.bias = c.F(b + ".o2.b"); o2.residual = &t2;
  T t3 = c.gemm(a2, c.W(b + ".o2.w"), C, o2);
  c.drop(a2); c.drop(t2);
  T l3 = c.layernorm(t3, b + ".ln3", 1e-5f);
  ConvOpt of;
  of.bias = c.F(b + ".ff1.b"); of.act = LADI_ACT_GEGLU;
  T ff = c.gemm(l3, c.W(b + ".ff1.w"), 8 * C, of);
  c.drop(l3);
  ConvOpt o3;
  o3.bias = c.F(b + ".ff2.b"); o3.residual = &t3;
  T t4 = c.gemm(ff, c.W(b + ".ff2.w"), C, o3);
  c.drop(ff); c.drop(t3);
  ConvOpt o4;
  o4.bias = c.F(p + ".proj_out.b"); o4.residual = &x;
  T out = c.gemm(t4, c.W(p + ".proj_out.w"), C, o4).as_image(B, h, w);
  c.drop(t4);
  return out;
}

void unet_forward(Ctx& c, const T& x_in, const int* step_ptr, const float* steps, const T& ctx_kv, const T& eps_out) {
  const ladi_engine_config& cf = c.e->cfg;
  const int* ch = cf.unet_channels;
  const int L = cf.unet_layers_per_block;
  std::vector<T> skips;
  ConvOpt oi;
  oi.bias = c.F("conv_in.b");
  const T xin = x_in.slice(0, cf.unet_in_channels);
  T x = c.conv(&xin, nullptr, c.W("conv_in.w"), ch[0], oi);
  skips.push_back(x);
  for (int i = 0; i < 4 && c.ok(); ++i) {
    const int out = ch[i];
    for (int l = 0; l < L; ++l) {
      T y = unet_resnet(c, fmt("down_blocks.%d.resnets.%d", i, l), &x, nullptr, out, steps, step_ptr);
      if (cf.unet_down_attn[i]) {
        T z = unet_transformer(c, fmt("down_blocks.%d.attentions.%d", i, l), y, cf.unet_heads[i], ctx_kv);
        c.drop(y);
        y = z;
      }
      x = y;  // the previous x stays alive: it is a skip connection
      skips.push_back(x);
    }
    if (i < 3) {
      const std::string p = fmt("down_blocks.%d.downsamplers.0.conv", i);
      ConvOpt od;
      od.bias = c.F(p + ".b"); od.stride = 2; od.pad_lo = 1;
      x = c.conv(&x, nullptr, c.W(p + ".w"), out, od);
      skips.push_back(x);
    }
  }
  {
    T y = unet_resnet(c, "mid_block.resnets.0", &x, nullptr, ch[3], steps, step_ptr);
    T z = unet_transformer(c, "mid_block.attentions.0", y, cf.unet_heads[3], ctx_kv);
    c.drop(y);
    x = unet_resnet(c, "mid_block.resnets.1", &z, nullptr, ch[3], steps, step_ptr);
    c.drop(z);
  }
  for (int i = 0; i < 4 && c.ok(); ++i) {
    const int out = ch[3 - i];
    for (int l = 0; l < L + 1; ++l) {
      T skip = skips.back();
      skips.pop_back();
      T y = unet_resnet(c, fmt("up_blocks.%d.resnets.%d", i, l), &x, &skip, out, steps, step_ptr);  // concat [current, skip] stays virtual
      c.drop(x); c.drop(skip);
      if (cf.unet_up_attn[i]) {
        T z = unet_transformer(c, fmt("up_blocks.%d.attentions.%d", i, l), y, cf.unet_heads[3 - i], ctx_kv);
        c.drop(y);
        y = z;
      }
      x = y;
    }
    if (i < 3) {
      const std::string p = fmt("up_blocks.%d.upsamplers.0.conv", i);
      ConvOpt ou;
      ou.bias = c.F(p + ".b");
      T y;
      if (cf.fuse_upsample) {
        ou.up2x = true;
        y = c.conv(&x, nullptr, c.W(p + ".w"), out, ou);
      } else {
        T u = c.upsample2x(x);
        y = c.conv(&u, nullptr, c.W(p + ".w"), out, ou);
        c.drop(u);
      }
      c.drop(x);
      x = y;
    }
  }
  T hn = c.groupnorm(&x, nullptr, "conv_norm_out", cf.unet_norm_eps, true);
  c.drop(x);
  ConvOpt oo;
  oo.bias = c.F("conv_out.b"); oo.out_fp32 = true; oo.out = &eps_out;
  c.conv(&hn, nullptr, c.W("conv_out.w"), cf.unet_out_channels, oo);
  c.drop(hn);
}

// plan_steps (unet.py): sinusoid (hi, lo) table -> linear_1 + SiLU -> linear_2 + SiLU (= silu(emb)) -> all time_emb_proj at once (+ conv1.bias), fp32 out
void unet_plan_steps(Ctx& c, const float* timesteps, int n, const T& steps_out) {
  const Weight& w1 = c.W("te1.w");
  if (!c.ok()) return;
  const int kp = w1.cols / 2, c0 = c.e->cfg.unet_channels[0];
  T pair = c.make(1, 1, n, 2 * kp);
  c.rec("timestep_embedding t=@%llx n=%d c=%d kp=%d out=@%llx", Ctx::A(timesteps), n, c0, kp, Ctx::A(pair.p));
  if (!c.plan && c.ok()) {
    const int r = ladi_timestep_embedding(timesteps, n, c0, kp, pair.p, c.st);
    if (r != LADI_OK) c.rc = r;
  }
  ConvOpt o1;
  o1.bias = c.F("te1.b"); o1.act = LADI_ACT_SILU;
  T e1 = c.gemm(pair, w1, w1.rows, o1);
  c.drop(pair);
  ConvOpt o2;
  o2.bias = c.F("te2.b"); o2.act = LADI_ACT_SILU;
  T e2 = c.gemm(e1, c.W("te2.w"), c.W("te2.w").rows, o2);
  c.drop(e1);
  ConvOpt o3;
  o3.bias = c.F("temb_all.b"); o3.out_fp32 = true; o3.out = &steps_out;
  c.gemm(e2, c.W("temb_all.w"), c.e->temb_total, o3);
  c.drop(e2);
}

// =================================================================================================================== VAE
T vae_resnet(Ctx& c, const std::string& p, const T& x, int co) {
  T hn = c.groupnorm(&x, nullptr, p + ".norm1", 1e-6f, true);
  ConvOpt o1;
  o1.bias = c.F(p + ".b1");
  T h = c.conv(&hn, nullptr, c.W(p + ".w1"), co, o1);
  c.drop(hn);
  T hn2 = c.groupnorm(&h, nullptr, p + ".norm2", 1e-6f, true);
  c.drop(h);
  ConvOpt o2;
  o2.bias = c.F(p + ".b2");
  if (x.c != co) o2.sc0 = &x;
  else o2.residual = &x;
  T out = c.conv(&hn2, nullptr, c.W(p + ".w2"), co, o2);
  c.drop(hn2);
  return out;
}

// diffusers 0.14 AttentionBlock, one head of width C (vae.py:81-90,142-150): GN -> fused Q|K|V GEMM -> wide flash attention -> proj_attn + x
T vae_attn(Ctx& c, const std::string& a, const T& x) {
  const int B = x.n, h = x.h, w = x.w, C = x.c, N = h * w;
  if (C != 512 && C != 256) { c.fail("engine: VAE mid-block attention is built for C = 512 (or 256), got %d", C); return T(); }
  T hn = c.groupnorm(&x, nullptr, a + ".group_norm", 1e-6f, false);
  ConvOpt o;
  o.bias = c.F(a + ".qkv.b");
  T qkv = c.gemm(hn, c.W(a + ".qkv.w"), 3 * C, o);
  c.drop(hn);
  const T t = qkv.as_image(B, 1, N);
  T at = c.attention(t.slice(0, C), t.slice(C, C), t.slice(2 * C, C), 1, 1.0f / sqrtf((float)C), C);
  c.drop(qkv);
  ConvOpt oo;
  oo.bias = c.F(a + ".o.b"); oo.residual = &x;
  T out = c.gemm(at, c.W(a + ".o.w"), C, oo).as_image(B, h, w);
  c.drop(at);
  return out;
}

T vae_mid(Ctx& c, const std::string& p, const T& x) {
  T a = vae_resnet(c, p + ".resnets.0", x, x.c);
  T b = vae_attn(c, p + ".attentions.0", a);
  c.drop(a);
  T out = vae_resnet(c, p + ".resnets.1", b, x.c);
  c.drop(b);
  return out;
}

// x: NHWC bf16 [B, H, W, >= 3]; feats[1..5] = caller buffers for the retained encoder features (vae.py:100-109; entry 0 is the input
// itself and entries 1 and 2 are the same tensor), any of them may be null (-> workspace, not returned); moments NHWC fp32 [B,h,w,2cz]
void vae_encode(Ctx& c, const T& x, const T& moments, T* feats /* [6], in/out */) {
  const ladi_engine_config& cf = c.e->cfg;
  const int* ch = cf.vae_channels;
  const int L = cf.vae_layers_per_block;
  const T xin = x.slice(0, cf.vae_in_channels);
  ConvOpt oi;
  oi.bias = c.F("encoder.conv_in.b");
  if (feats[1].p != nullptr) oi.out = &feats[1];
  T h = c.conv(&xin, nullptr, c.W("encoder.conv_in.w"), ch[0], oi);
  feats[0] = xin; feats[1] = h; feats[2] = h;
  std::vector<T> keep;  // tensors that must outlive their block: the retained features that live in the workspace
  for (int i = 0; i < 4 && c.ok(); ++i) {
    // feats[2 + i] (i >= 1) is the input of down block i = the output of the previous downsampler; set below
    T cur = h;
    for (int l = 0; l < L; ++l) {
      T y = vae_resnet(c, fmt("encoder.down_blocks.%d.resnets.%d", i, l), cur, ch[i]);
      if (!(l == 0)) c.drop(cur);  // the block input is a retained feature; later intermediates are not
      cur = y;
    }
    if (i < 3) {
      const std::string p = fmt("encoder.down_blocks.%d.downsamplers.0.conv", i);
      ConvOpt od;
      od.bias = c.F(p + ".b"); od.stride = 2; od.pad_lo = 0;
      if (feats[3 + i].p != nullptr) od.out = &feats[3 + i];
      T y = c.conv(&cur, nullptr, c.W(p + ".w"), ch[i], od);
      c.drop(cur);
      feats[3 + i] = y;
      h = y;
    } else {
      h = cur;
    }
  }
  T m = vae_mid(c, "encoder.mid_block", h);
  c.drop(h);
  T hn = c.groupnorm(&m, nullptr, "encoder.conv_norm_out", 1e-6f, true);
  c.drop(m);
  ConvOpt oo;
  oo.bias = c.F("enc_out.b"); oo.out_fp32 = true; oo.out = &moments;
  c.conv(&hn, nullptr, c.W("enc_out.w"), 2 * cf.vae_latent_channels, oo);
  c.drop(hn);
}

// zq: NHWC bf16 [B,h,w,8] = post_quant_conv input already laid out by the caller (latents / scaling_factor); feats = EMASC outputs in the
// reference's list order (ascending layer index; vae.py:190 reverses it), n_feats of them, int_layers their layer indices; img NHWC fp32
void vae_decode(Ctx& c, const T& zin, const T* feats, int n_feats, const int* int_layers, const T& img) {
  const ladi_engine_config& cf = c.e->cfg;
  const int* ch = cf.vae_channels;
  const int L = cf.vae_layers_per_block, cz = cf.vae_latent_channels;
  const int B = zin.n, h = zin.h, w = zin.w;
  T zq = c.make(B, h, w, 8);
  {
    const T zr = zin.slice(0, cz).as_rows();
    T zo = zq.slice(0, cz).as_rows();
    zo.owned = false;
    ConvOpt o;
    o.bias = c.F("post_quant.b"); o.out = &zo;
    c.gemm(zr, c.W("post_quant.w"), cz, o);
  }
  ConvOpt oi;
  oi.bias = c.F("decoder.conv_in.b");
  const T zq4 = zq.slice(0, cz);
  T x0 = c.conv(&zq4, nullptr, c.W("decoder.conv_in.w"), ch[3], oi);
  c.drop(zq);
  T x = vae_mid(c, "decoder.mid_block", x0);
  c.drop(x0);
  for (int i = 0; i < 4 && c.ok(); ++i) {
    const int co = ch[3 - i];
    if (i < n_feats) {  // vae.py:193 `sample += int_feat` with the REVERSED list
      T y = c.add(x, feats[n_feats - 1 - i]);
      c.drop(x);
      x = y;
    }
    for (int l = 0; l < L + 1; ++l) {
      T y = vae_resnet(c, fmt("decoder.up_blocks.%d.resnets.%d", i, l), x, co);
      c.drop(x);
      x = y;
    }
    if (i < 3) {
      const std::string p = fmt("decoder.up_blocks.%d.upsamplers.0.conv", i);
      ConvOpt ou;
      ou.bias = c.F(p + ".b");
      T y;
      if (cf.fuse_upsample) {
        ou.up2x = true;
        y = c.conv(&x, nullptr, c.W(p + ".w"), co, ou);
      } else {
        T u = c.upsample2x(x);
        y = c.conv(&u, nullptr, c.W(p + ".w"), co, ou);
        c.drop(u);
      }
      c.drop(x);
      x = y;
    }
  }
  // vae.py:204-210: the level-1 skip is added after norm + SiLU, the level-0 (image-space) skip after conv_out
  const T* last = nullptr;
  const T* res0 = nullptr;
  T res0v;
  for (int k = 0; k < n_feats; ++k) {
    if (int_layers[k] == 1) last = &feats[k];  // reversed index n-1-index(1) of the reversed list == original position k
    if (int_layers[k] == 0) { res0v = feats[k].slice(0, cf.vae_out_channels); res0 = &res0v; }
  }
  T hn = c.groupnorm(&x, nullptr, "decoder.conv_norm_out", 1e-6f, true, last);
  c.drop(x);
  ConvOpt oo;
  oo.bias = c.F("decoder.conv_out.b"); oo.out_fp32 = true; oo.out = &img; oo.residual = res0;
  c.conv(&hn, nullptr, c.W("decoder.conv_out.w"), cf.vae_out_channels, oo);
  c.drop(hn);
}

// EMASC (emasc.py:20-33,37-40): per scale either the nonlinear form conv -> SiLU -> conv, or (no `emasc.%d.w2` in the weight table) the
// linear form, one conv.  mask_features' (1 - mask) is the row scale of the last conv.  The kernel size is read from the packed width of
// `emasc.%d.w1` (taps x 64-padded input channels): 9 taps -> 3x3 with padding 1, 1 tap -> 1x1 with padding 0.
void emasc_forward(Ctx& c, const T* feats, const float* const* inv_masks, int n, const T* outs) {
  for (int i = 0; i < n && c.ok(); ++i) {
    const Weight& w1 = c.W(fmt("emasc.%d.w1", i));
    if (!c.ok()) return;
    const int cin = c.e->cfg.emasc_in[i], kpad = (cin + 63) / 64 * 64;
    const int taps = w1.cols % kpad == 0 ? w1.cols / kpad : 0;
    if (taps != 9 && taps != 1) { c.fail("engine: emasc.%d.w1 is %d wide: not a 3x3 or 1x1 kernel over %d channels", i, w1.cols, cin); return; }
    const int k = taps == 9 ? 3 : 1;
    const bool linear = c.e->w.find(fmt("emasc.%d.w2", i)) == c.e->w.end();
    const float* rs = inv_masks != nullptr ? inv_masks[i] : nullptr;
    ConvOpt o1;
    o1.ksize = k; o1.pad_lo = k / 2; o1.bias = c.F(fmt("emasc.%d.b1", i));
    if (linear) {
      o1.row_scale = rs; o1.out = &outs[i];
      c.conv(&feats[i], nullptr, w1, c.e->cfg.emasc_out[i], o1);
      continue;
    }
    o1.act = LADI_ACT_SILU;
    T t = c.conv(&feats[i], nullptr, w1, cin, o1);
    ConvOpt o2;
    o2.ksize = k; o2.pad_lo = k / 2; o2.bias = c.F(fmt("emasc.%d.b2", i)); o2.row_scale = rs; o2.out = &outs[i];
    const T ts = t.slice(0, cin);
    c.conv(&ts, nullptr, c.W(fmt("emasc.%d.w2", i)), c.e->cfg.emasc_out[i], o2);
    c.drop(t);
  }
}

// One full pre-LN CLIP encoder layer over all tokens (transformers CLIPEncoderLayer; the sequence of clip.py encoder_layer):
// LN1 -> fused QKV GEMM -> ladi_attention_small -> out-proj + residual -> LN2 -> fc1 + GELU -> fc2 + residual.  x [B, 1, T, d].
T adapter_encoder_layer(Ctx& c, const std::string& p, const T& x) {
  const ladi_engine_config& cf = c.e->cfg;
  const int B = x.n, Tk = x.w, d = x.c, heads = cf.adapter_heads, hd = d / heads;
  T y = c.layernorm(x.as_rows(), p + "ln1", 1e-5f);
  ConvOpt oqkv;
  oqkv.bias = c.F(p + "qkv.b");
  T qkv = c.gemm(y, c.W(p + "qkv.w"), 3 * d, oqkv);
  c.drop(y);
  T a = c.make(B, 1, Tk, d);
  if (!c.ok()) return a;
  const long long qbs = (long long)Tk * qkv.pitch, obs = (long long)Tk * a.pitch;
  const float scale = 1.0f / sqrtf((float)hd);
  const uint8_t* q = reinterpret_cast<const uint8_t*>(qkv.p);
  c.rec("attn_small batch=%d heads=%d nq=%d nkv=%d hd=%d q=@%llx qp=%d qbs=%lld k=@%llx kp=%d kbs=%lld v=@%llx vp=%d vbs=%lld out=@%llx op=%d obs=%lld "
        "scale=%.6g causal=0", B, heads, Tk, Tk, hd, Ctx::A(q), qkv.pitch, qbs, Ctx::A(q + 2 * d), qkv.pitch, qbs, Ctx::A(q + 4 * d), qkv.pitch, qbs,
        Ctx::A(a.p), a.pitch, obs, (double)scale);
  if (!c.plan && c.ok()) {
    const int r = ladi_attention_small(q, q + 2 * d, q + 4 * d, a.p, B, heads, Tk, Tk, hd, qkv.pitch, qkv.pitch, qkv.pitch, a.pitch, qbs, qbs, qbs, obs, scale,
                                       0, c.st);
    if (r != LADI_OK) c.rc = r;
  }
  c.drop(qkv);
  ConvOpt oo;
  oo.bias = c.F(p + "o.b"); oo.residual = &x;
  T x1 = c.gemm(a, c.W(p + "o.w"), d, oo);
  c.drop(a);
  T l2 = c.layernorm(x1, p + "ln2", 1e-5f);
  ConvOpt o1;
  o1.bias = c.F(p + "fc1.b"); o1.act = LADI_ACT_GELU;
  T hmid = c.gemm(l2, c.W(p + "fc1.w"), cf.adapter_mlp, o1);
  c.drop(l2);
  ConvOpt o2;
  o2.bias = c.F(p + "fc2.b"); o2.residual = &x1;
  T x2 = c.gemm(hmid, c.W(p + "fc2.w"), d, o2);
  c.drop(hmid); c.drop(x1);
  return x2.as_image(B, 1, Tk);
}

// InversionAdapter.forward (inversion_adapter.py:22-28): L CLIP ViT-H encoder layers, then LayerNorm + Linear-GELU-Linear-GELU-Linear
// on the CLS row.  Layers 0..L-2 (weights `adapter.enc<l>.*`, present only when L > 1) run over all T tokens; of the last layer
// (weights `adapter.ln1`, `adapter.kv.w`, ...) only the CLS row is consumed, so its query, attention, out-projection and MLP run on one
// row per image.  x bf16 [B, T, d]; out bf16 [B, out_dim]
void adapter_forward(Ctx& c, const T& x_in /* n=B, h=1, w=T, c=d */, const T& out) {
  const ladi_engine_config& cf = c.e->cfg;
  T xe = x_in;
  for (int l = 0; c.ok() && c.e->w.count(fmt("adapter.enc%d.ln1.0", l)); ++l) {
    T nx = adapter_encoder_layer(c, fmt("adapter.enc%d.", l), xe);
    c.drop(xe);
    xe = nx;
  }
  if (!c.ok()) return;
  const T& x = xe;
  const int B = x.n, Tk = x.w, d = x.c, heads = cf.adapter_heads, hd = d / heads;
  T y = c.layernorm(x.as_rows(), "adapter.ln1", 1e-5f);
  ConvOpt ok;
  ok.bias = c.F("adapter.kv.b");
  T kv = c.gemm(y, c.W("adapter.kv.w"), 2 * d, ok);
  // CLS rows: row b*T of y (pitch T*d)
  T y0 = y;
  y0.n = 1; y0.h = 1; y0.w = B; y0.pitch = Tk * d; y0.owned = false;
  ConvOpt oq;
  oq.bias = c.F("adapter.q.b");
  T q0 = c.gemm(y0, c.W("adapter.q.w"), d, oq);
  T a = c.make(1, 1, B, d);
  c.rec("cls_attn q=@%llx qp=%d kv=@%llx kvp=%d batch=%d tokens=%d heads=%d hd=%d out=@%llx op=%d", Ctx::A(q0.p), q0.pitch, Ctx::A(kv.p), kv.pitch, B, Tk, heads, hd, Ctx::A(a.p), a.pitch);
  if (!c.plan && c.ok()) {
    const int r = ladi_cls_attention(q0.p, q0.pitch, kv.p, kv.pitch, B, Tk, heads, hd, 1.0f / sqrtf((float)hd), a.p, a.pitch, c.st);
    if (r != LADI_OK) c.rc = r;
  }
  c.drop(q0); c.drop(kv);
  T x0v = x;
  x0v.n = 1; x0v.h = 1; x0v.w = B; x0v.pitch = Tk * d; x0v.owned = false;
  ConvOpt oo;
  oo.bias = c.F("adapter.o.b"); oo.residual = &x0v;
  T x0 = c.gemm(a, c.W("adapter.o.w"), d, oo);
  c.drop(a); c.drop(y); c.drop(xe);
  T l2 = c.layernorm(x0, "adapter.ln2", 1e-5f);
  ConvOpt o1;
  o1.bias = c.F("adapter.fc1.b"); o1.act = LADI_ACT_GELU;
  T hmid = c.gemm(l2, c.W("adapter.fc1.w"), cf.adapter_mlp, o1);
  c.drop(l2);
  ConvOpt o2;
  o2.bias = c.F("adapter.fc2.b"); o2.residual = &x0;
  T x1 = c.gemm(hmid, c.W("adapter.fc2.w"), d, o2);
  c.drop(hmid); c.drop(x0);
  T z = c.layernorm(x1, "adapter.lnp", 1e-5f);
  c.drop(x1);
  ConvOpt g0;
  g0.bias = c.F("adapter.l0.b"); g0.act = LADI_ACT_GELU;
  T z0 = c.gemm(z, c.W("adapter.l0.w"), cf.adapter_hidden, g0);
  c.drop(z);
  ConvOpt g3;
  g3.bias = c.F("adapter.l3.b"); g3.act = LADI_ACT_GELU;
  T z3 = c.gemm(z0, c.W("adapter.l3.w"), cf.adapter_hidden, g3);
  c.drop(z0);
  ConvOpt g6;
  g6.bias = c.F("adapter.l6.b"); g6.out = &out;
  c.gemm(z3, c.W("adapter.l6.w"), cf.adapter_out, g6);
  c.drop(z3);
}

// ------------------------------------------------------------------------------------------------------------- derived tables
void derive(Engine* e) {
  const ladi_engine_config& cf = e->cfg;
  e->resnets.clear(); e->transformers.clear();
  const int* ch = cf.unet_channels;
  const int L = cf.unet_layers_per_block;
  for (int i = 0; i < 4; ++i)
    for (int l = 0; l < L; ++l) {
      e->resnets.push_back({fmt("down_blocks.%d.resnets.%d", i, l), ch[i]});
      if (cf.unet_down_attn[i]) e->transformers.push_back({fmt("down_blocks.%d.attentions.%d", i, l), ch[i]});
    }
  e->resnets.push_back({"mid_block.resnets.0", ch[3]});
  e->transformers.push_back({"mid_block.attentions.0", ch[3]});
  e->resnets.push_back({"mid_block.resnets.1", ch[3]});
  for (int i = 0; i < 4; ++i)
    for (int l = 0; l < L + 1; ++l) {
      e->resnets.push_back({fmt("up_blocks.%d.resnets.%d", i, l), ch[3 - i]});
      if (cf.unet_up_attn[i]) e->transformers.push_back({fmt("up_blocks.%d.attentions.%d", i, l), ch[3 - i]});
    }
  int off = 0;
  for (auto& r : e->resnets) { e->temb_off[r.first] = off; off += r.second; }
  e->temb_total = off;
  off = 0;
  for (auto& t : e->transformers) { e->kv_off[t.first] = off; off += 2 * t.second; }
  e->kv_total = off;
  e->in_pitch = (cf.unet_in_channels + 7) / 8 * 8;
}

T view(const void* p, int n, int h, int w, int c, int pitch, bool f32 = false) {
  T t;
  t.p = const_cast<void*>(p); t.n = n; t.h = h; t.w = w; t.c = c; t.pitch = pitch; t.f32 = f32;
  return t;
}

struct Call {  // one module invocation: run for real, or plan it (workspace high-water mark / op trace)
  Ctx c;
  Call(Engine* e, void* ws, size_t ws_bytes, void* stream, bool plan) {
    c.e = e; c.st = reinterpret_cast<cudaStream_t>(stream); c.plan = plan;
    if (plan) c.arena.reset(reinterpret_cast<void*>(uintptr_t(1) << 40), size_t(1) << 44);  // fake address space, never dereferenced
    else c.arena.reset(ws, ws_bytes);
  }
};

}  // namespace

struct ladi_engine {
  Engine e;
};

#define ENGINE_CHECK(h) LADI_CHECK((h) != nullptr, "engine handle is null")

extern "C" int ladi_engine_create(const ladi_engine_config* cfg, const ladi_weight* table, int n_weights, ladi_engine** out) {
  LADI_CHECK(cfg != nullptr && out != nullptr && (table != nullptr || n_weights == 0), "engine_create: null argument");
  LADI_CHECK(cfg->norm_groups >= 0 && cfg->norm_groups <= 64, "engine_create: norm_groups must be in 1..64 (0 = 32)");
  ladi_engine* h = new ladi_engine();
  h->e.cfg = *cfg;
  if (h->e.cfg.norm_groups == 0) h->e.cfg.norm_groups = 32;
  for (int i = 0; i < n_weights; ++i) {
    if (table[i].name == nullptr || table[i].ptr == nullptr) {
      delete h;
      LADI_CHECK(false, "engine_create: weight %d has a null name or pointer", i);
    }
    Weight w;
    w.p = table[i].ptr; w.rows = table[i].rows; w.cols = table[i].cols;
    h->e.w[table[i].name] = w;
  }
  derive(&h->e);
  if (cfg->plan_only == 0) {  // the two scratch buffers shared by every call (the only allocations this library ever makes)
    h->e.splitk_bytes = size_t(64) << 20;
    h->e.gn_floats = size_t(512) * 64 * 64 * 2;
    if (cudaMalloc(&h->e.splitk_ws, h->e.splitk_bytes) != cudaSuccess || cudaMalloc(reinterpret_cast<void**>(&h->e.gn_ws), h->e.gn_floats * 4) != cudaSuccess) {
      ladi_set_error("engine_create: cudaMalloc of the shared scratch buffers failed: %s", cudaGetErrorString(cudaGetLastError()));
      if (h->e.splitk_ws) cudaFree(h->e.splitk_ws);
      delete h;
      return LADI_ERR_CUDA;
    }
  } else {
    h->e.splitk_ws = reinterpret_cast<void*>(uintptr_t(7) << 40); h->e.splitk_bytes = size_t(64) << 20;
    h->e.gn_ws = reinterpret_cast<float*>(uintptr_t(9) << 40); h->e.gn_floats = size_t(512) * 64 * 64 * 2;
  }
  *out = h;
  return LADI_OK;
}

extern "C" int ladi_engine_destroy(ladi_engine* h) {
  if (h == nullptr) return LADI_OK;
  if (h->e.cfg.plan_only == 0) {
    if (h->e.splitk_ws) cudaFree(h->e.splitk_ws);
    if (h->e.gn_ws) cudaFree(h->e.gn_ws);
  }
  delete h;
  return LADI_OK;
}

extern "C" int ladi_engine_query(const ladi_engine* h, int what) {
  if (h == nullptr) return -1;
  switch (what) {
    case LADI_Q_TEMB_TOTAL: return h->e.temb_total;
    case LADI_Q_KV_TOTAL: return h->e.kv_total;
    case LADI_Q_IN_PITCH: return h->e.in_pitch;
    default: return -1;
  }
}

// ---- the module bodies behind one dispatcher (run / plan) --------------------------------------------------------------------
static int run_unet(ladi_engine* h, bool plan, std::string* trace, const void* x_in, const int* step_ptr, const float* steps, const void* ctx_kv, int B, int hh, int ww,
                    int ctx_tokens, void* eps_out, void* ws, size_t ws_bytes, void* stream, size_t* high) {
  Call k(&h->e, ws, ws_bytes, stream, plan);
  k.c.trace = trace;
  const T xin = view(x_in, B, hh, ww, h->e.in_pitch, h->e.in_pitch);
  const T kv = view(ctx_kv, B, 1, ctx_tokens, h->e.kv_total, h->e.kv_total);
  const T eps = view(eps_out, B, hh, ww, 4, 4, true);
  unet_forward(k.c, xin, step_ptr, steps, kv, eps);
  if (high) *high = k.c.arena.high;
  return k.c.rc;
}

extern "C" int ladi_unet_forward(ladi_engine* h, const void* x_in, const int* step_ptr, const float* steps, const void* ctx_kv, int batch, int lat_h, int lat_w,
                                 int ctx_tokens, void* eps_out, void* workspace, int64_t workspace_bytes, void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(x_in && step_ptr && steps && ctx_kv && eps_out && workspace, "unet_forward: null operand");
  LADI_CHECK(batch > 0 && lat_h > 0 && lat_w > 0 && ctx_tokens > 0, "unet_forward: bad extent");
  return run_unet(h, false, nullptr, x_in, step_ptr, steps, ctx_kv, batch, lat_h, lat_w, ctx_tokens, eps_out, workspace, (size_t)workspace_bytes, stream, nullptr);
}

static int run_plan_steps(ladi_engine* h, bool plan, std::string* trace, const float* timesteps, int n, void* steps_out, void* ws, size_t ws_bytes, void* stream,
                          size_t* high) {
  Call k(&h->e, ws, ws_bytes, stream, plan);
  k.c.trace = trace;
  const T out = view(steps_out, 1, 1, n, h->e.temb_total, h->e.temb_total, true);
  unet_plan_steps(k.c, timesteps, n, out);
  if (high) *high = k.c.arena.high;
  return k.c.rc;
}

extern "C" int ladi_unet_plan_steps(ladi_engine* h, const float* timesteps, int n, float* steps_out, void* workspace, int64_t workspace_bytes, void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(timesteps && steps_out && workspace && n > 0, "unet_plan_steps: bad arguments");
  return run_plan_steps(h, false, nullptr, timesteps, n, steps_out, workspace, (size_t)workspace_bytes, stream, nullptr);
}

extern "C" int ladi_unet_plan_context(ladi_engine* h, const void* ctx, int rows, int ctx_dim, void* ctx_kv_out, void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(ctx && ctx_kv_out && rows > 0 && ctx_dim > 0 && ctx_dim % 8 == 0, "unet_plan_context: bad arguments");
  Call k(&h->e, nullptr, 0, stream, false);
  const T c = view(ctx, 1, 1, rows, ctx_dim, ctx_dim);
  const T out = view(ctx_kv_out, 1, 1, rows, h->e.kv_total, h->e.kv_total);
  ConvOpt o;
  o.out = &out;
  k.c.gemm(c, k.c.W("kv_all.w"), h->e.kv_total, o);
  return k.c.rc;
}

static int run_encode(ladi_engine* h, bool plan, std::string* trace, const void* x, int B, int H, int W, void* moments, void* const* skips, void* ws, size_t ws_bytes,
                      void* stream, size_t* high) {
  Call k(&h->e, ws, ws_bytes, stream, plan);
  k.c.trace = trace;
  const ladi_engine_config& cf = h->e.cfg;
  const T xin = view(x, B, H, W, 8, 8);
  const T mom = view(moments, B, H / 8, W / 8, 2 * cf.vae_latent_channels, 2 * cf.vae_latent_channels, true);
  T feats[6];
  // retained features (vae.py:100-109): [1] = [2] = conv_in output (C0, full res); [3], [4], [5] = downsampler outputs
  const int fc[6] = {0, cf.vae_channels[0], cf.vae_channels[0], cf.vae_channels[0], cf.vae_channels[1], cf.vae_channels[2]};
  const int fs[6] = {1, 1, 1, 2, 4, 8};
  for (int i = 1; i < 6; ++i)
    if (skips != nullptr && skips[i] != nullptr) feats[i] = view(skips[i], B, H / fs[i], W / fs[i], fc[i], fc[i]);
  vae_encode(k.c, xin, mom, feats);
  if (high) *high = k.c.arena.high;
  return k.c.rc;
}

extern "C" int ladi_vae_encode(ladi_engine* h, const void* x_nhwc8, int batch, int height, int width, float* moments, void* const* skips, void* workspace,
                               int64_t workspace_bytes, void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(x_nhwc8 && moments && workspace, "vae_encode: null operand");
  LADI_CHECK(batch > 0 && height % 8 == 0 && width % 8 == 0 && height > 0 && width > 0, "vae_encode: height / width must be positive multiples of 8");
  return run_encode(h, false, nullptr, x_nhwc8, batch, height, width, moments, skips, workspace, (size_t)workspace_bytes, stream, nullptr);
}

static int run_decode(ladi_engine* h, bool plan, std::string* trace, const void* z, int B, int hh, int ww, const void* const* feats, int n_feats, const int* int_layers,
                      void* img, void* ws, size_t ws_bytes, void* stream, size_t* high) {
  Call k(&h->e, ws, ws_bytes, stream, plan);
  k.c.trace = trace;
  const ladi_engine_config& cf = h->e.cfg;
  const T zin = view(z, B, hh, ww, 8, 8);
  const T out = view(img, B, hh * 8, ww * 8, 4, 4, true);
  T f[8];
  for (int i = 0; i < n_feats; ++i) {
    const int layer = int_layers[i];
    // channels / resolution of the EMASC output for encoder layer `layer` (hubconf.py:41-42): 0: image, 1: C0, 2: C1@1, 3: C2@/2, 4: C3@/4, 5: C3@/8
    const int c_ = layer == 0 ? cf.vae_out_channels : layer == 1 ? cf.vae_channels[0] : layer == 2 ? cf.vae_channels[1] : layer == 3 ? cf.vae_channels[2] : cf.vae_channels[3];
    const int s_ = layer <= 2 ? 1 : layer == 3 ? 2 : layer == 4 ? 4 : 8;
    f[i] = view(feats[i], B, hh * 8 / s_, ww * 8 / s_, c_, (c_ + 7) / 8 * 8);
  }
  vae_decode(k.c, zin, f, n_feats, int_layers, out);
  if (high) *high = k.c.arena.high;
  return k.c.rc;
}

extern "C" int ladi_vae_decode_emasc(ladi_engine* h, const void* z_nhwc8, int batch, int lat_h, int lat_w, const void* const* feats, int n_feats,
                                     const int* int_layers, float* image_out, void* workspace, int64_t workspace_bytes, void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(z_nhwc8 && image_out && workspace, "vae_decode: null operand");
  LADI_CHECK(n_feats >= 0 && n_feats <= 6 && (n_feats == 0 || (feats != nullptr && int_layers != nullptr)), "vae_decode: bad feature list");
  return run_decode(h, false, nullptr, z_nhwc8, batch, lat_h, lat_w, feats, n_feats, int_layers, image_out, workspace, (size_t)workspace_bytes, stream, nullptr);
}

static int run_emasc(ladi_engine* h, bool plan, std::string* trace, const void* const* feats, const float* const* inv, int B, int H, int W, void* const* outs, void* ws,
                     size_t ws_bytes, void* stream, size_t* high) {
  Call k(&h->e, ws, ws_bytes, stream, plan);
  k.c.trace = trace;
  const ladi_engine_config& cf = h->e.cfg;
  T f[8], o[8];
  for (int i = 0; i < cf.emasc_scales; ++i) {
    const int s_ = cf.emasc_stride[i];
    f[i] = view(feats[i], B, H / s_, W / s_, cf.emasc_in[i], (cf.emasc_in[i] + 7) / 8 * 8);
    o[i] = view(outs[i], B, H / s_, W / s_, cf.emasc_out[i], (cf.emasc_out[i] + 7) / 8 * 8);
  }
  emasc_forward(k.c, f, inv, cf.emasc_scales, o);
  if (high) *high = k.c.arena.high;
  return k.c.rc;
}

extern "C" int ladi_emasc_forward(ladi_engine* h, const void* const* feats, const float* const* inv_masks, int batch, int height, int width, void* const* outs,
                                  void* workspace, int64_t workspace_bytes, void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(feats && outs && workspace, "emasc_forward: null operand");
  return run_emasc(h, false, nullptr, feats, inv_masks, batch, height, width, outs, workspace, (size_t)workspace_bytes, stream, nullptr);
}

static int run_adapter(ladi_engine* h, bool plan, std::string* trace, const void* x, int B, int tokens, void* out, void* ws, size_t ws_bytes, void* stream, size_t* high) {
  Call k(&h->e, ws, ws_bytes, stream, plan);
  k.c.trace = trace;
  const ladi_engine_config& cf = h->e.cfg;
  const T xin = view(x, B, 1, tokens, cf.adapter_dim, cf.adapter_dim);
  const T o = view(out, 1, 1, B, cf.adapter_out, cf.adapter_out);
  adapter_forward(k.c, xin, o);
  if (high) *high = k.c.arena.high;
  return k.c.rc;
}

extern "C" int ladi_inversion_adapter_forward(ladi_engine* h, const void* feats, int batch, int tokens, void* out, void* workspace, int64_t workspace_bytes,
                                              void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(feats && out && workspace && batch > 0 && tokens > 0, "inversion_adapter_forward: bad arguments");
  return run_adapter(h, false, nullptr, feats, batch, tokens, out, workspace, (size_t)workspace_bytes, stream, nullptr);
}

// N x (UNet forward + CFG + DDIM update + rewrite of the 4 dynamic UNet input channels), enqueued on `stream` (tryon_pipe.py:713-747).
// A caller with CUDA graphs captures ONE step (ladi_unet_forward + ladi_ddim_cfg_step) and replays it; this is the same loop for callers
// without.  The device-side step counter `step_ptr` (int32[2], zeroed by the caller) advances on the device: no host sync in the loop.
extern "C" int ladi_denoise_loop(ladi_engine* h, void* unet_in, float* latents, int* step_ptr, const float* steps, const float* coef, const void* ctx_kv, int batch,
                                 int lat_h, int lat_w, int ctx_tokens, int cfg, float guidance, int n_steps, float* eps_scratch, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  ENGINE_CHECK(h);
  LADI_CHECK(unet_in && latents && step_ptr && steps && coef && ctx_kv && eps_scratch && workspace && n_steps > 0, "denoise_loop: bad arguments");
  const int Bp = cfg ? 2 * batch : batch;
  for (int i = 0; i < n_steps; ++i) {
    int r = run_unet(h, false, nullptr, unet_in, step_ptr, steps, ctx_kv, Bp, lat_h, lat_w, ctx_tokens, eps_scratch, workspace, (size_t)workspace_bytes, stream, nullptr);
    if (r != LADI_OK) return r;
    r = ladi_ddim_cfg_step(eps_scratch, 4, latents, unet_in, h->e.in_pitch, batch, lat_h, lat_w, cfg, guidance, coef, step_ptr, 1, nullptr, stream);
    if (r != LADI_OK) return r;
  }
  return LADI_OK;
}

// Workspace bytes of one module call (plan-mode walk of the same body); also leaves the op trace of that walk in the handle.
extern "C" int64_t ladi_workspace_bytes(ladi_engine* h, int module, int batch, int height, int width) {
  if (h == nullptr) return -1;
  size_t high = 0;
  h->e.trace.clear();
  int rc = LADI_OK;
  static const int dummy_layers[6] = {1, 2, 3, 4, 5, 0};
  const void* fake[8];
  for (int i = 0; i < 8; ++i) fake[i] = reinterpret_cast<const void*>((uintptr_t(2) << 40) + (uintptr_t(i) << 34));
  void* fake_out[8];
  for (int i = 0; i < 8; ++i) fake_out[i] = reinterpret_cast<void*>((uintptr_t(3) << 40) + (uintptr_t(i) << 34));
  const void* X = reinterpret_cast<const void*>(uintptr_t(4) << 40);
  void* Y = reinterpret_cast<void*>(uintptr_t(5) << 40);
  switch (module) {
    case LADI_MODULE_UNET:
      rc = run_unet(h, true, &h->e.trace, X, reinterpret_cast<const int*>(fake[0]), reinterpret_cast<const float*>(fake[1]), fake[2], batch, height, width, 77, Y, nullptr, 0,
                    nullptr, &high);
      break;
    case LADI_MODULE_VAE_ENCODE:
      rc = run_encode(h, true, &h->e.trace, X, batch, height, width, Y, fake_out, nullptr, 0, nullptr, &high);
      break;
    case LADI_MODULE_VAE_DECODE:
      rc = run_decode(h, true, &h->e.trace, X, batch, height, width, fake, h->e.cfg.emasc_scales, dummy_layers, Y, nullptr, 0, nullptr, &high);
      break;
    case LADI_MODULE_EMASC:
      rc = run_emasc(h, true, &h->e.trace, fake, nullptr, batch, height, width, fake_out, nullptr, 0, nullptr, &high);
      break;
    case LADI_MODULE_ADAPTER:
      rc = run_adapter(h, true, &h->e.trace, X, batch, height /* tokens */, Y, nullptr, 0, nullptr, &high);
      break;
    case LADI_MODULE_UNET_PLAN:
      rc = run_plan_steps(h, true, &h->e.trace, reinterpret_cast<const float*>(X), batch, Y, nullptr, 0, nullptr, &high);
      break;
    default:
      ladi_set_error("workspace_bytes: unknown module %d", module);
      return -1;
  }
  if (rc != LADI_OK) return -1;
  return (int64_t)high;
}

extern "C" const char* ladi_engine_trace(const ladi_engine* h) { return h != nullptr ? h->e.trace.c_str() : ""; }

// C ABI of libsvc_b200.so: model handle, workspace arena and the stage pipelines.
// Entry points and the reference code each one replaces are documented in include/svcb.h.
#include <algorithm>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"

namespace svcb {

static thread_local std::string g_err;
static thread_local int64_t g_launches = 0;
void set_error(const std::string& msg) { g_err = msg; }
void count_launch() { ++g_launches; }

int device_sm_count() {
  static std::atomic<int> cache[kMaxDevices];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 0;
  const bool cached = dev >= 0 && dev < kMaxDevices;
  int n = cached ? cache[dev].load(std::memory_order_relaxed) : 0;
  if (n > 0) return n;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return 0;
  if (cached) cache[dev].store(n, std::memory_order_relaxed);
  return n;
}

// ----------------------------------------------------------------------------- kernel timing
struct TimedLaunch { std::string name; cudaEvent_t e0, e1; double flops, bytes, aux; };
static bool g_timing = false;
static std::vector<TimedLaunch> g_timed;
static std::string g_report;

KernelScope::KernelScope(const char* name, cudaStream_t s, double flops, double bytes, double aux)
    : slot(-1), stream(s) {
  if (!g_timing) return;
  TimedLaunch t;
  t.name = name; t.flops = flops; t.bytes = bytes; t.aux = aux;
  if (cudaEventCreate(&t.e0) != cudaSuccess || cudaEventCreate(&t.e1) != cudaSuccess) return;
  cudaEventRecord(t.e0, s);
  g_timed.push_back(t);
  slot = (int)g_timed.size() - 1;
}
KernelScope::~KernelScope() {
  if (slot >= 0) cudaEventRecord(g_timed[slot].e1, stream);
}

struct ConvW {
  const float* w = nullptr;
  const float* b = nullptr;
  int cin = 0, cout = 0, cout_pad = 0, k = 1;
  const uint8_t* tc = nullptr;  // tensor-core tile image (pack.py:pack_conv_tc_general) or null
  int cin_pad = 0, bn = 0, ntiles = 0;
};

// must match pack.py:tc_tiling
static void tc_tiling(ConvW& w) {
  w.cin_pad = (w.cin + kConvTcKch - 1) / kConvTcKch * kConvTcKch;
  const int cp16 = (w.cout + 15) / 16 * 16;
  w.ntiles = (cp16 + 255) / 256;
  w.bn = ((cp16 + w.ntiles - 1) / w.ntiles + 15) / 16 * 16;
}
struct SnakeW {
  const float *ea = nullptr, *ib = nullptr, *fu = nullptr, *fd = nullptr;
  SnakeTapsV taps = {};   // the 12 + 12 alias-filter taps by value (read back once at model creation)
};

struct EncLayer {
  ConvW qkv, o, ffn1, ffn2;
  const float *ek, *ev, *ln1g, *ln1b, *ln2g, *ln2b;
};
struct FlowLayer {
  ConvW pre, post;
  std::vector<ConvW> in, rs;
  const float *snac_w, *snac_b;
};
// Which kernels run each generator stage.  They depend only on the config, the precision and the blob's images,
// so resolve() chooses them once at model creation.
enum UpsForm { UPS_POLYPHASE, UPS_COMB, UPS_FUSED };      // `rate` phase convs + ups_finalize | `comb` | ups_fused
enum NoiseForm { NOISE_IN_UPS, NOISE_TC, NOISE_CONV1D };  // inside the upsampler's kernel | `noise_tc` | conv1d
enum AmpForm { AMP_S2D, AMP_BLOCK_FUSED, AMP_TC, AMP_FP32 };

struct UpStage {
  std::vector<ConvW> phase;  // one sub-convolution per output phase
  const float* bias;
  ConvW noise;
  ConvW noise_tc;            // long noise filter as a 2-tap conv over the space-to-depth source
  int comb_cin1 = 0, comb_cin2 = 0;   // comb's input channels: [0, comb_cin1) the stage input (zero padded), then windows of the source
  ConvW comb;                // all phases as ONE conv with rate * Cout channels, taps + 1 taps (pack.py:ups_combined) or tc == null
  int rate, k, pad, taps;
  int sf = 1;                // source samples per output sample: the product of the later stages' rates
  UpsForm form = UPS_POLYPHASE;
  std::vector<bool> phase_tc;   // UPS_POLYPHASE: phase r runs as conv_tc, else conv1d
  std::vector<int> q0;          // UPS_POLYPHASE: phase r's first output (independent of L)
  NoiseForm noise_form = NOISE_IN_UPS;
  bool ragged = false;          // stops each ragged item at its end: comb and ups_fused read it, and tensor-core phases over the
                                // zero tail + NOISE_TC read nothing past it (SRCP is cut there)
};
struct ResBlock {
  ConvW c1[3], c2[3];
  const uint8_t *c1_tc[3], *c2_tc[3];  // bf16 hi/lo tensor-core images of the same weights
  // narrow stages (C * r = 160, r = s2d_r): block-Toeplitz matrices of the same convs (pack.py:pack_conv_s2d_slots)
  const uint8_t *c1_s2d[3] = {nullptr, nullptr, nullptr}, *c2_s2d[3] = {nullptr, nullptr, nullptr};
  int s2d_r = 0;
  S2dPlan s2d1[3], s2d2[3];             // c1's fold, taps and the columns each reaches (s2d_tap_plan); c2's (fold 1)
  SnakeW act[6];
  int k, dil[3];
  AmpForm form = AMP_FP32;
  AmpForm fallback = AMP_FP32;   // the form at a length the S2D links do not fit (= form unless that is AMP_S2D)
};

// must match pack.py:s2d_factor
static int s2d_link_factor(int ch) { return ch == 40 ? 4 : ch == 20 ? 8 : ch == 10 ? 16 : 0; }
// The S2D links of factor r run at length L: whole rows of r samples, whole octets of rows.
static bool s2d_fits(long long L, int r) { return L > 0 && r > 0 && L % r == 0 && L % 8 == 0; }

}  // namespace svcb

struct svcb_model {
  svcb_config cfg;
  int hop = 1;
  // cfg.precision as the pipelines use it: the convs' operand split (0 = fp32 CUDA cores, 1, 3), prior attention on wgmma
  int nsplit = 0;
  bool attn_tc = false;
  // resolved views
  svcb::ConvW pre, hub, proj;
  const float* pit_emb = nullptr;
  std::vector<svcb::EncLayer> enc;
  std::vector<svcb::FlowLayer> flow;
  const float *ad_sw, *ad_sb, *ad_bw, *ad_bb;
  svcb::ConvW conv_pre, conv_post;
  const float *merge_w, *merge_b;
  std::vector<svcb::UpStage> ups;
  std::vector<svcb::ResBlock> res;
  svcb::SnakeW post_act;
  std::vector<float> conv_post_h;   // host copy of conv_post's taps [cin][7] (kernel parameters of the fused tail)
};

namespace svcb {

// ----------------------------------------------------------------------------- arena
struct Ctx {
  char* base = nullptr;
  size_t cap = 0, off = 0, peak = 0;
  bool dry = false;
  cudaStream_t stream = nullptr;
  const svcb_taps* taps = nullptr;

  template <class T>
  T* alloc(size_t n) {
    off = align256(off);
    const size_t o = off;
    off += n * sizeof(T);
    if (off > peak) peak = off;
    if (dry) return reinterpret_cast<T*>((uintptr_t)4096 + o);
    if (off > cap) return nullptr;
    return reinterpret_cast<T*>(base + o);
  }
  // after the allocations a step makes and before its launches; a dry run sizes the workspace and checks nothing
  int check() const { return dry ? SVCB_OK : check_workspace(base, cap, peak, "model"); }
};

#define RUN(expr)                    \
  do {                               \
    if (!ctx.dry) SVCB_TRY(expr);    \
  } while (0)

static int tap(Ctx& ctx, int id, const float* src, size_t numel) {
  if (ctx.dry || !ctx.taps || !ctx.taps->ptr[id]) return SVCB_OK;
  SVCB_CUDA_CHECK(cudaMemcpyAsync(ctx.taps->ptr[id], src, numel * sizeof(float),
                                  cudaMemcpyDeviceToDevice, ctx.stream));
  return SVCB_OK;
}

// y[B,cout,T] = conv(x[B,cin,T]) with the standard contiguous layouts.
static ConvParams std_conv(const ConvW& w, const float* x, float* y, int B, int Tin, int Tout,
                           int pad, int dil = 1, int stride = 1) {
  ConvParams p;
  p.x = x; p.sxb = (long long)w.cin * Tin; p.sxc = Tin; p.sxt = 1;
  p.w = w.w; p.cout_pad = w.cout_pad; p.bias = w.b;
  p.y = y; p.syb = (long long)w.cout * Tout; p.syc = Tout; p.syt = 1;
  p.B = B; p.Cin = w.cin; p.Cout = w.cout; p.Tin = Tin;
  p.K = w.k; p.stride = stride; p.dil = dil; p.pad = pad;
  p.q0 = 0; p.nq = Tout;
  return p;
}

// A stride-1 tensor-core convolution of w over x[b, ci, t] = x[b * sxb + ci * sxc + t * sxt] into y[B, Cout, Tout].
static ConvTcParams conv_tc_params(const ConvW& w, const float* x, long long sxb, long long sxc, long long sxt, float* y,
                                   int B, int Tin, int Tout, int dil, int pad, int nsplit) {
  ConvTcParams q;
  q.x = x; q.sxb = sxb; q.sxc = sxc; q.sxt = sxt;
  q.wpk = w.tc; q.bias = w.b; q.y = y;
  q.B = B; q.Cin = w.cin; q.cin_pad = w.cin_pad; q.Cout = w.cout; q.Tin = Tin; q.Tout = Tout;
  q.K = w.k; q.dil = dil; q.pad = pad; q.bn = w.bn; q.ntiles = w.ntiles;
  q.nsplit = nsplit;
  return q;
}

// A conv of the prior encoder, the flow or conv_pre, on the tensor cores unless all convs run on the CUDA cores.  Every
// caller builds p with std_conv from w (a tile image, p.bias, Cin, Cout, K): a stride-1 'same' conv, contiguous y.
static int run_conv(const svcb_model* m, const ConvW& w, const ConvParams& p, cudaStream_t s) {
  if (m->nsplit == 0) return launch_conv1d(p, s);
  ConvTcParams q = conv_tc_params(w, p.x, p.sxb, p.sxc, p.sxt, p.y, p.B, p.Tin, p.nq, p.dil, p.pad, m->nsplit);
  q.res = p.res; q.lengths = p.lengths; q.flags = p.flags; q.act = p.act;
  return launch_conv_tc(q, s);
}

__global__ void mask_mul_kernel(float* __restrict__ x, const long long* __restrict__ lengths, int C,
                                int T) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x, c = blockIdx.y, b = blockIdx.z;
  if (t < T && t >= lengths[b]) x[((long long)b * C + c) * T + t] = 0.f;
}
static int launch_mask_mul(float* x, const long long* lengths, int B, int C, int T, cudaStream_t s) {
  dim3 grid((T + 127) / 128, C, B);
  KernelScope ks("mask_mul", s, 0.0, 4.0 * B * C * (double)T);
  mask_mul_kernel<<<grid, 128, 0, s>>>(x, lengths, C, T);
  SVCB_LAUNCH_CHECK("mask_mul");
  return SVCB_OK;
}

// x[b, c, t] = 0 for lengths[b] <= t < T: the tails of a ragged batch, one thread per element of the longest tail
// (no launch when every item fills T)
__global__ void zero_tail_kernel(float* __restrict__ x, const long long* __restrict__ lengths, int C, int T) {
  const long long t = lengths[blockIdx.z] + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (t < T) x[((long long)blockIdx.z * C + blockIdx.y) * T + t] = 0.f;
}
static int launch_zero_tail(float* x, const long long* lengths, long long min_len, int B, int C, int T, cudaStream_t s) {
  if (min_len >= T) return SVCB_OK;
  dim3 grid((unsigned)((T - min_len + 127) / 128), C, B);
  KernelScope ks("zero_tail", s, 0.0, 4.0 * B * C * (double)(T - min_len));
  zero_tail_kernel<<<grid, 128, 0, s>>>(x, lengths, C, T);
  SVCB_LAUNCH_CHECK("zero_tail");
  return SVCB_OK;
}

// ----------------------------------------------------------------------------- upsampler finalize
// The ConvTranspose1d upsamplers (generator.py:183) run as `rate` polyphase sub-convolutions.  Each
// phase writes its outputs CONTIGUOUSLY into a phase-major scratch (coalesced stores); this kernel
// interleaves the phases back into y[b, co, n], adds the transposed conv's bias and, for the stages
// whose noise conv is short (K <= 8), noise_convs[i](source) + its bias (generator.py:185-186) in
// the same pass — one coalesced write of the stage input instead of `rate` strided ones plus a
// read-modify-write.
struct UpsFinalizeParams {
  const float* tmp[SVCB_MAX_UPS];  // per phase r: [B][C][nq[r]]
  int nq[SVCB_MAX_UPS], q0[SVCB_MAX_UPS];
  const float* bias;               // [C]
  const float* src;                // [B][Ltot] or null (noise handled elsewhere)
  const float* wn;                 // packed [1][Kn][cout_pad]
  const float* bn;                 // [C]
  float* y;                        // [B][C][Ln]
  int C, Ln, rate, pad, Kn, sf, padn, cout_pad;
  long long Ltot;
};

__global__ void __launch_bounds__(256)
ups_finalize_kernel(const UpsFinalizeParams p) {
  const int n = blockIdx.x * 256 + threadIdx.x, co = blockIdx.y, b = blockIdx.z;
  if (n >= p.Ln) return;
  const int r = (n + p.pad) % p.rate, q = (n + p.pad) / p.rate;
  const int qi = q - p.q0[r];
  float v = __ldg(p.bias + co);
  if (qi >= 0 && qi < p.nq[r]) v += p.tmp[r][((long long)b * p.C + co) * p.nq[r] + qi];
  if (p.src) {
    const float* sb = p.src + (long long)b * p.Ltot;
    float a = __ldg(p.bn + co);
    for (int j = 0; j < p.Kn; ++j) {
      const long long si = (long long)n * p.sf + j - p.padn;
      if (si >= 0 && si < p.Ltot) a = fmaf(__ldg(sb + si), __ldg(p.wn + (long long)j * p.cout_pad + co), a);
    }
    v += a;
  }
  p.y[((long long)b * p.C + co) * p.Ln + n] = v;
}

static int launch_ups_finalize(const UpsFinalizeParams& p, int B, cudaStream_t s) {
  dim3 grid((p.Ln + 255) / 256, p.C, B);
  KernelScope ks("ups_finalize", s, 2.0 * B * p.C * (double)p.Ln * (p.src ? p.Kn : 0),
                 8.0 * B * p.C * (double)p.Ln);
  ups_finalize_kernel<<<grid, 256, 0, s>>>(p);
  SVCB_LAUNCH_CHECK("ups_finalize");
  return SVCB_OK;
}

// source [B][Ltot] -> zero-padded copy [B][32 + Ltot + tail] for the space-to-depth noise convs; a ragged item's source
// ends at lens[b] * hop samples
constexpr int SRC_PADF = 32;
__global__ void pad_source_kernel(const float* __restrict__ src, float* __restrict__ dst, long long Ltot,
                                  long long Lpad, const int* __restrict__ lens, int hop) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= Lpad) return;
  const long long si = i - SRC_PADF;
  const long long n = lens ? (long long)lens[b] * hop : Ltot;
  dst[(long long)b * Lpad + i] = (si >= 0 && si < n) ? src[(long long)b * Ltot + si] : 0.f;
}

// ----------------------------------------------------------------------------- prior encoder
// ragged (svcb_infer_ragged): pre / hub also read ppg / vec as zero past each item's length, as a lone call's padding
// (the reference convolves its padded batch unmasked there)
static int run_prior(const svcb_model* m, Ctx& ctx, const float* ppg, const float* vec,
                     const float* pit, const long long* lengths, const float* eps, float* z_p, int B,
                     int T, bool ragged = false) {
  const svcb_config& c = m->cfg;
  const int H = c.hidden_channels, C = c.inter_channels, Fc = c.filter_channels;
  cudaStream_t s = ctx.stream;
  float* x = ctx.alloc<float>((size_t)B * H * T);
  float* y = ctx.alloc<float>((size_t)B * H * T);
  float* qkv = ctx.alloc<float>((size_t)B * 3 * H * T);
  float* att = ctx.alloc<float>((size_t)B * H * T);
  float* hbuf = ctx.alloc<float>((size_t)B * Fc * T);
  float* stats = ctx.alloc<float>((size_t)B * 2 * C * T);
  const size_t attn_ws_bytes = m->attn_tc ? rel_attention_ws_bytes(B, c.enc_heads, T) : 0;
  uint8_t* attn_ws = m->attn_tc ? ctx.alloc<uint8_t>(attn_ws_bytes) : nullptr;
  SVCB_TRY(ctx.check());
  {  // pre / hub on time-major inputs (vits/models.py:40-46)
    ConvParams p = std_conv(m->pre, ppg, x, B, T, T, 2);
    p.sxb = (long long)T * c.ppg_dim; p.sxc = 1; p.sxt = c.ppg_dim;
    p.lengths = lengths; p.flags = CONV_OUT_MASK | (ragged ? CONV_IN_MASK : 0);
    RUN(run_conv(m, m->pre, p, s));
    ConvParams q = std_conv(m->hub, vec, x, B, T, T, 2);
    q.sxb = (long long)T * c.vec_dim; q.sxc = 1; q.sxt = c.vec_dim;
    q.lengths = lengths; q.flags = p.flags; q.res = x;
    RUN(run_conv(m, m->hub, q, s));
  }
  RUN(launch_pitch_embed_add(x, pit, m->pit_emb, B, H, T, s));
  SVCB_TRY(tap(ctx, SVCB_TAP_ENC_FRONT, x, (size_t)B * H * T));
  RUN(launch_mask_mul(x, lengths, B, H, T, s));  // Encoder.forward: x = x * x_mask
  for (int i = 0; i < c.enc_layers; ++i) {
    const EncLayer& L = m->enc[i];
    RUN(run_conv(m, L.qkv, std_conv(L.qkv, x, qkv, B, T, T, 0), s));
    if (m->attn_tc) RUN(launch_rel_attention_tc(qkv, L.ek, L.ev, lengths, att, attn_ws, attn_ws_bytes, B, H, c.enc_heads, c.enc_window, T, s));
    else RUN(launch_rel_attention(qkv, L.ek, L.ev, lengths, att, B, H, c.enc_heads, c.enc_window, T, s));
    RUN(run_conv(m, L.o, std_conv(L.o, att, y, B, T, T, 0), s));
    RUN(launch_layernorm_c(x, y, L.ln1g, L.ln1b, x, B, H, T, 0, 1e-5f, s));
    const int pl = (c.enc_kernel - 1) / 2;
    ConvParams f1 = std_conv(L.ffn1, x, hbuf, B, T, T, pl);
    f1.lengths = lengths; f1.flags = CONV_IN_MASK; f1.act = ACT_RELU;
    RUN(run_conv(m, L.ffn1, f1, s));
    ConvParams f2 = std_conv(L.ffn2, hbuf, y, B, T, T, pl);
    f2.lengths = lengths; f2.flags = CONV_IN_MASK | CONV_OUT_MASK;
    RUN(run_conv(m, L.ffn2, f2, s));
    RUN(launch_layernorm_c(x, y, L.ln2g, L.ln2b, x, B, H, T, 0, 1e-5f, s));
    if (i < 6) SVCB_TRY(tap(ctx, SVCB_TAP_ENC_LAYER0 + i, x, (size_t)B * H * T));
  }
  ConvParams pj = std_conv(m->proj, x, stats, B, T, T, 0);
  pj.lengths = lengths; pj.flags = CONV_IN_MASK | CONV_OUT_MASK;
  RUN(run_conv(m, m->proj, pj, s));
  RUN(launch_reparam(stats, eps, lengths, z_p, B, C, T, s));
  SVCB_TRY(tap(ctx, SVCB_TAP_ZP, z_p, (size_t)B * C * T));
  return SVCB_OK;
}

// ----------------------------------------------------------------------------- flow (reverse)
static int run_flow(const svcb_model* m, Ctx& ctx, const float* z_p, const long long* lengths,
                    const float* spk, float* z, int B, int T) {
  const svcb_config& c = m->cfg;
  const int H = c.hidden_channels, C = c.inter_channels, half = C / 2;
  cudaStream_t s = ctx.stream;
  float* ya = ctx.alloc<float>((size_t)B * C * T);
  float* yb = ctx.alloc<float>((size_t)B * C * T);
  float* sp = ctx.alloc<float>((size_t)B * C);
  float* x0n = ctx.alloc<float>((size_t)B * half * T);
  float* h = ctx.alloc<float>((size_t)B * H * T);
  float* g = ctx.alloc<float>((size_t)B * H * T);
  float* rs = ctx.alloc<float>((size_t)B * 2 * H * T);
  float* out = ctx.alloc<float>((size_t)B * H * T);
  float* mm = ctx.alloc<float>((size_t)B * half * T);
  SVCB_TRY(ctx.check());
  const float* cur = z_p;
  for (int f = c.n_flows - 1; f >= 0; --f) {
    const FlowLayer& F = m->flow[f];
    float* Y = (f == 0) ? z : (((c.n_flows - 1 - f) & 1) ? yb : ya);
    RUN(launch_linear_small(spk, F.snac_w, F.snac_b, sp, B, c.spk_dim, C, s));
    RUN(launch_coupling_pre(cur, sp, lengths, Y, x0n, B, C, T, s));
    ConvParams pp = std_conv(F.pre, x0n, h, B, T, T, 0);
    pp.lengths = lengths; pp.flags = CONV_OUT_MASK;
    RUN(run_conv(m, F.pre, pp, s));
    const int nl = c.wn_layers;
    for (int l = 0; l < nl; ++l) {
      ConvParams pi = std_conv(F.in[l], h, g, B, T, T, (c.wn_kernel - 1) / 2);
      pi.flags = CONV_GATE;
      pi.syb = (long long)H * T;  // gated output has H channels
      RUN(run_conv(m, F.in[l], pi, s));
      RUN(run_conv(m, F.rs[l], std_conv(F.rs[l], g, rs, B, T, T, 0), s));
      RUN(launch_wn_update(h, out, rs, lengths, B, H, T, l == 0, l == nl - 1, s));
    }
    ConvParams po = std_conv(F.post, out, mm, B, T, T, 0);
    po.lengths = lengths; po.flags = CONV_OUT_MASK;
    RUN(run_conv(m, F.post, po, s));
    RUN(launch_coupling_post(cur, sp, mm, lengths, Y, B, C, T, s));
    if (f < 4) SVCB_TRY(tap(ctx, SVCB_TAP_FLOW0 + f, Y, (size_t)B * C * T));
    cur = Y;
  }
  return SVCB_OK;
}

// ----------------------------------------------------------------------------- generator
// The operands of one generator stage.  Its upsampler and noise conv write the stage input X from x and the source.
// Unit d of its AMP block j writes RA, RB, then ACC: each block adds its output to the stage mean there
// (generator.py:188-194), the first block writes it, the others accumulate, the last divides.
struct Stage {
  const float* x;             // the previous stage's output [B, 2C, L / rate]
  float* X;                   // stage input [B, C, L]
  float* ACC;
  float *T1, *T2, *RA, *RB;   // fp32 temporaries [B, C, L]; T1 also holds UPS_POLYPHASE's phases
  void *img_hi, *img_lo;      // snake_pack operand images (AMP_TC)
  void* s2d[4];               // two ping-pong S2D images, hi and lo each (AMP_S2D)
  const float *source, *SRCP; // [B][Ltot]; [B][Lpad] from SRC_PADF samples before the source, zero-padded (tensor-core forms)
  long long Ltot, Lpad;
  int B, C, L, nres, nsplit, hop, lscale;
  const int* lens;            // ragged batch (UPS_FUSED, AMP_TC, AMP_S2D): item b ends at lens[b] * lscale samples, or null
  const long long* len64;     // ragged batch (UPS_COMB): item b's length at the upsampler's input rate in len64[b], or null
  float* out(int d) const { return d == 0 ? RA : d == 1 ? RB : ACC; }
  bool accum(int d, int j) const { return d == 2 && j > 0; }
  float out_div(int d, int j) const { return d == 2 && j == nres - 1 ? (float)nres : 0.f; }
};

// An amp_s2d_link over the S2D image in = (hi, lo) of x[B, C, L]; with act, its epilogue also writes act(result) as the
// image out = (hi, lo).  The caller sets the weights, their tap plan, the bias, res and y.
static AmpS2dParams s2d_link_params(int B, int C, int L, int K, void* const* in, void* const* out, const SnakeW* act) {
  AmpS2dParams q;
  q.B = B; q.C = C; q.L = L; q.K = K; q.Rp = s2d_rows(L, s2d_link_factor(C));
  q.a_hi = in[0]; q.a_lo = in[1];
  if (act) {
    q.o_hi = out[0]; q.o_lo = out[1];
    q.ea = act->ea; q.ib = act->ib; q.fu = act->fu; q.fd = act->fd; q.taps = act->taps;
  }
  return q;
}

// An amp_conv_tc link over the snake_pack image (hi, lo) of x[B, C, L]; the caller sets the weights and the epilogue.
static AmpConvParams amp_conv_params(const void* hi, const void* lo, int B, int C, int L, int K, int nsplit) {
  AmpConvParams q;
  q.a_hi = hi; q.a_lo = lo; q.Lp = p8_rows(L);
  q.B = B; q.C = C; q.Cp = (C + 15) / 16 * 16; q.L = L; q.K = K; q.nsplit = nsplit;
  return q;
}

// narrow stages: every link = block-Toeplitz wgmma conv with the next SnakeAlias in its epilogue.  Link k = 2d + half
// is c1[d] from S2D image 0 to image 1 or c2[d] from image 1 to image 0 (a.s2d = hi, lo of each); its output image is
// SnakeAlias k + 1, none after the block's last conv.  Image 0 is written in the fold of the c1 link that reads it.
static int run_amp_s2d(Ctx& ctx, const Stage& a, const ResBlock& R, int j) {
  const SnakeW& s0 = R.act[0];
  RUN(launch_snake_pack_s2d(a.X, a.s2d[0], a.s2d[1], s0.ea, s0.ib, s0.fu, s0.fd, a.B, a.C, a.L, ctx.stream, &s0.taps, a.lens, a.lscale,
                            R.s2d1[0].fold));
  const float* cur = a.X;
  for (int k = 0; k < 6; ++k) {
    const int d = k / 2, half = k % 2;
    AmpS2dParams q = s2d_link_params(a.B, a.C, a.L, R.k, a.s2d + 2 * half, a.s2d + 2 - 2 * half, k < 5 ? &R.act[k + 1] : nullptr);
    q.wpk = half ? R.c2_s2d[d] : R.c1_s2d[d]; q.bias = half ? R.c2[d].b : R.c1[d].b;
    const S2dPlan& pl = half ? R.s2d2[d] : R.s2d1[d];
    q.ntaps = pl.ntaps; q.mlo = pl.mlo; q.tap_cols = pl.tap_cols; q.fin = pl.fold;
    if (half && d < 2) q.fout = R.s2d1[d + 1].fold;
    q.lens = a.lens; q.lscale = a.lscale;
    if (half) { q.res = cur; q.y = a.out(d); q.accum = a.accum(d, j); q.out_div = a.out_div(d, j); cur = q.y; }
    RUN(launch_amp_s2d_link(q, ctx.stream));
  }
  return SVCB_OK;
}

// narrow stages: the whole block (6 convs + 6 SnakeAlias + residuals) in one fp32 kernel
static int run_amp_block_fused(Ctx& ctx, const Stage& a, const ResBlock& R, int j) {
  AmpBlockParams q;
  q.x = a.X; q.y = a.ACC; q.B = a.B; q.C = a.C; q.L = a.L; q.K = R.k;
  for (int d = 0; d < 3; ++d) {
    q.dil[d] = R.dil[d];
    q.w1[d] = R.c1[d].w; q.b1[d] = R.c1[d].b; q.w2[d] = R.c2[d].w; q.b2[d] = R.c2[d].b;
  }
  q.cout_pad = R.c1[0].cout_pad;
  for (int k = 0; k < 6; ++k) { q.ea[k] = R.act[k].ea; q.ib[k] = R.act[k].ib; q.fu[k] = R.act[k].fu; q.fd[k] = R.act[k].fd; }
  q.accum = a.accum(2, j); q.out_div = a.out_div(2, j);   // (the block's last unit writes the stage mean)
  RUN(launch_amp_block_fused(q, ctx.stream));
  return SVCB_OK;
}

// tensor-core path: snake_pack -> amp_conv_tc, twice per unit
static int run_amp_tc(Ctx& ctx, const Stage& a, const ResBlock& R, int j) {
  void* lo = a.nsplit == 3 ? a.img_lo : nullptr;
  const float* cur = a.X;
  for (int d = 0; d < 3; ++d) {
    const SnakeW& s1 = R.act[2 * d];
    const SnakeW& s2 = R.act[2 * d + 1];
    AmpConvParams q = amp_conv_params(a.img_hi, lo, a.B, a.C, a.L, R.k, a.nsplit);
    RUN(launch_snake_pack(cur, a.img_hi, lo, s1.ea, s1.ib, s1.fu, s1.fd, a.B, a.C, a.L, ctx.stream, &s1.taps, a.lens, a.lscale));
    q.y = a.T2; q.wpk = R.c1_tc[d]; q.bias = R.c1[d].b; q.dil = R.dil[d];
    RUN(launch_amp_conv_tc(q, ctx.stream));
    RUN(launch_snake_pack(a.T2, a.img_hi, lo, s2.ea, s2.ib, s2.fu, s2.fd, a.B, a.C, a.L, ctx.stream, &s2.taps, a.lens, a.lscale));
    q.wpk = R.c2_tc[d]; q.bias = R.c2[d].b; q.dil = 1; q.res = cur;
    q.y = a.out(d); q.accum = a.accum(d, j); q.out_div = a.out_div(d, j);
    RUN(launch_amp_conv_tc(q, ctx.stream));
    cur = q.y;
  }
  return SVCB_OK;
}

static int run_amp_fp32(Ctx& ctx, const Stage& a, const ResBlock& R, int j) {
  const float* cur = a.X;
  for (int d = 0; d < 3; ++d) {
    const SnakeW& s1 = R.act[2 * d];
    const SnakeW& s2 = R.act[2 * d + 1];
    RUN(launch_snake_alias(cur, a.T1, s1.ea, s1.ib, s1.fu, s1.fd, a.B, a.C, a.L, ctx.stream));
    RUN(launch_conv1d(std_conv(R.c1[d], a.T1, a.T2, a.B, a.L, a.L, R.dil[d] * (R.k - 1) / 2, R.dil[d]), ctx.stream));
    RUN(launch_snake_alias(a.T2, a.T1, s2.ea, s2.ib, s2.fu, s2.fd, a.B, a.C, a.L, ctx.stream));
    ConvParams p = std_conv(R.c2[d], a.T1, a.out(d), a.B, a.L, a.L, (R.k - 1) / 2);
    p.res = cur; p.flags = a.accum(d, j) ? CONV_ACCUM : 0; p.out_div = a.out_div(d, j);
    RUN(launch_conv1d(p, ctx.stream));
    cur = p.y;
  }
  return SVCB_OK;
}

// wide stages: every phase AND the stage's noise conv in one tensor-core conv whose epilogue stores the interleaved
// samples — the stage input is read once, X is written once
static int run_ups_comb(Ctx& ctx, const UpStage& us, const Stage& a) {
  const int C = 2 * a.C, L = a.L / us.rate;
  ConvTcParams q = conv_tc_params(us.comb, a.x, (long long)C * L, L, 1, a.X, a.B, L, L, 1, us.taps - 1, a.nsplit);
  q.Cin = C; q.ilv = us.rate;
  q.x2 = a.SRCP + (SRC_PADF - us.sf / 2); q.sx2b = a.Lpad; q.sx2t = (long long)us.sf * us.rate;
  q.cin1 = us.comb_cin1; q.cin2 = us.comb_cin2;
  // ragged: rows past an item's end read as zero in both inputs; a lone call's row bound (tau < Tin) also drops
  // the source window of the row at its end, whose first sf/2 samples precede that end
  if (a.len64) { q.lengths = a.len64; q.flags = CONV_IN_MASK; }
  RUN(launch_conv_tc(q, ctx.stream));
  return SVCB_OK;
}

// narrow stages: transposed conv + noise conv + biases in one fp32 pass
static int run_ups_fused(Ctx& ctx, const UpStage& us, const Stage& a) {
  UpsFusedParams q;
  q.x = a.x; q.wph[0] = us.phase[0].w; q.wph[1] = us.phase[1].w; q.bias = us.bias;
  q.src = a.source; q.wn = us.noise.w; q.bn = us.noise.b; q.y = a.X;
  q.B = a.B; q.Cin = 2 * a.C; q.Cout = a.C; q.L = a.L / us.rate; q.Ln = a.L; q.rate = us.rate; q.M = us.taps; q.pad = us.pad;
  q.cout_pad = us.phase[0].cout_pad; q.Kn = us.noise.k; q.sf = us.sf; q.padn = us.sf / 2;
  q.cout_pad_n = us.noise.cout_pad; q.Ltot = a.Ltot;
  q.lens = a.lens; q.src_scale = a.hop;
  RUN(launch_ups_fused(q, ctx.stream));
  return SVCB_OK;
}

// `rate` polyphase sub-convolutions, each into its own contiguous slab of T1 (coalesced), interleaved + biased
// + (short) noise conv by ups_finalize
static int run_ups_polyphase(Ctx& ctx, const UpStage& us, const Stage& a) {
  const int C = 2 * a.C, L = a.L / us.rate;
  UpsFinalizeParams fp;
  fp.bias = us.bias; fp.y = a.X; fp.C = a.C; fp.Ln = a.L; fp.rate = us.rate; fp.pad = us.pad;
  fp.src = us.noise_form == NOISE_IN_UPS ? a.source : nullptr; fp.wn = us.noise.w; fp.bn = us.noise.b;
  fp.Kn = us.noise.k; fp.sf = us.sf; fp.padn = us.sf / 2; fp.cout_pad = us.noise.cout_pad; fp.Ltot = a.Ltot;
  size_t slab = 0;
  for (int r = 0; r < us.rate; ++r) {
    ConvParams p = std_conv(us.phase[r], a.x, nullptr, a.B, L, a.L, us.taps - 1);
    p.q0 = us.q0[r];
    p.nq = (a.L - 1 + us.pad - r) / us.rate - p.q0 + 1;   // up to the last output q of phase r
    p.y = a.T1 + slab;
    p.syb = (long long)a.C * p.nq; p.syc = p.nq; p.syt = 1;
    fp.tmp[r] = p.y; fp.nq[r] = p.nq; fp.q0[r] = p.q0;
    slab += (size_t)a.B * a.C * p.nq;
    if (us.phase_tc[r]) {
      // phase r is a stride-1 convolution with nq == L outputs: x index = t + j - (taps-1-q0)
      RUN(launch_conv_tc(conv_tc_params(us.phase[r], a.x, (long long)C * L, L, 1, p.y, a.B, L, L, 1, us.taps - 1 - p.q0, a.nsplit), ctx.stream));
    } else {
      RUN(launch_conv1d(p, ctx.stream));
    }
  }
  RUN(launch_ups_finalize(fp, a.B, ctx.stream));
  return SVCB_OK;
}

// long noise filter as Conv1d(sf -> C, K=2) over the space-to-depth view of the padded source:
// x[b, ci, t] = srcp[b][32 - sf/2 + sf*t + ci]
static int run_noise_tc(Ctx& ctx, const UpStage& us, const Stage& a) {
  ConvTcParams q = conv_tc_params(us.noise_tc, a.SRCP + (SRC_PADF - us.sf / 2), a.Lpad, 1, us.sf, a.X, a.B, a.L + 1, a.L, 1, 0, a.nsplit);
  q.flags = CONV_ACCUM;
  RUN(launch_conv_tc(q, ctx.stream));
  return SVCB_OK;
}

// long noise filters (K = 2*prod(later rates)): separate accumulate pass
static int run_noise_conv1d(Ctx& ctx, const UpStage& us, const Stage& a) {
  ConvParams p = std_conv(us.noise, a.source, a.X, a.B, (int)a.Ltot, a.L, us.sf / 2, 1, us.sf);
  p.flags = CONV_ACCUM;
  RUN(launch_conv1d(p, ctx.stream));
  return SVCB_OK;
}

// What the generator launches at T frames where that depends on the length: each AMP block's form (resolve()'s `form`
// where the S2D links fit the stage's length, else its `fallback`) and whether the tail runs as post_fused.  Everything
// else resolve() chose at model creation.  wave: where the tail writes (post_fused needs it 16-byte aligned).
struct GenPlan {
  AmpForm amp[SVCB_MAX_UPS * SVCB_MAX_RES];   // block j of stage i at i * n_res + j, as svcb_model::res
  bool post_fused;
  GenPlan(const svcb_model* m, long long T, const float* wave) {
    const svcb_config& c = m->cfg;
    long long L = T;
    for (int i = 0; i < c.n_ups; ++i) {
      L *= c.up_rates[i];
      for (int j = i * c.n_res; j < (i + 1) * c.n_res; ++j) amp[j] = s2d_fits(L, m->res[j].s2d_r) ? m->res[j].form : m->res[j].fallback;
    }
    // the stage mean the tail reads is an arena buffer, 256-byte aligned
    post_fused = !m->conv_post.b && post_fused_supported(m->conv_post.cin, (int)L, m->conv_post.k, wave, wave);
  }
};

// A ragged batch (svcb_infer_ragged) passes its lengths as lens (int32 frames, for the generator's own kernels) and
// len64 ([n_ups + 1][B] int64: item b's length at the input rate of stage i in row i, for zero_tail and conv_tc) and has
// been checked by ragged_forms(): every stage takes a form that reads them.  Item b then ends at its own length at
// every rate, and what a conv reads past that end is zero, as in a lone call's padding.
static int run_generator(const svcb_model* m, Ctx& ctx, const float* spk, const float* z,
                         const float* source, float* wave, int B, int T, const long long* len64 = nullptr,
                         const int* lens = nullptr, int min_n = 0) {
  const svcb_config& c = m->cfg;
  const GenPlan plan(m, T, wave);
  cudaStream_t s = ctx.stream;
  const int U = c.gen_input;
  const int nsplit = m->nsplit;
  const long long Ltot = (long long)T * m->hop;
  float* sc = ctx.alloc<float>((size_t)B * U);
  float* bi = ctx.alloc<float>((size_t)B * U);
  float* xa = ctx.alloc<float>((size_t)B * U * T);
  float* x0 = ctx.alloc<float>((size_t)B * c.gen_initial_channel * T);
  // temporaries and operand images sized for the largest stage
  size_t max_stage = 0, img_bytes = 0;
  {
    int ch = c.gen_initial_channel; long long L = T;
    for (int i = 0; i < c.n_ups; ++i) {
      ch /= 2; L *= c.up_rates[i];
      max_stage = std::max<size_t>(max_stage, (size_t)B * ch * L);
      if (nsplit) img_bytes = std::max<size_t>(img_bytes, p8_image_bytes(B, ch, (int)L));
    }
  }
  float* T1 = ctx.alloc<float>(max_stage);
  float* T2 = ctx.alloc<float>(max_stage);
  float* RA = ctx.alloc<float>(max_stage);
  float* RB = ctx.alloc<float>(max_stage);
  const long long Lpad = (SRC_PADF + Ltot + 128 + 3) / 4 * 4;
  float* SRCP = nsplit ? ctx.alloc<float>((size_t)B * Lpad) : nullptr;
  void* IMG_HI = img_bytes ? ctx.alloc<uint8_t>(img_bytes) : nullptr;
  void* IMG_LO = (img_bytes && nsplit == 3) ? ctx.alloc<uint8_t>(img_bytes) : nullptr;
  SVCB_TRY(ctx.check());

  if (nsplit && !ctx.dry) {
    dim3 grid((unsigned)((Lpad + 255) / 256), B);
    KernelScope ks("pad_source", s, 0.0, 8.0 * B * (double)Lpad);
    pad_source_kernel<<<grid, 256, 0, s>>>(source, SRCP, Ltot, Lpad, lens, m->hop);
    SVCB_LAUNCH_CHECK("pad_source");
  }
  RUN(launch_linear_small(spk, m->ad_sw, m->ad_sb, sc, B, c.spk_dim, U, s));
  RUN(launch_linear_small(spk, m->ad_bw, m->ad_bb, bi, B, c.spk_dim, U, s));
  RUN(launch_layernorm_c(z, nullptr, sc, bi, xa, B, U, T, U, 1e-5f, s));
  if (len64) RUN(launch_zero_tail(xa, len64, min_n, B, U, T, s));
  {
    ConvParams p = std_conv(m->conv_pre, xa, x0, B, T, T, 3);
    p.act = ACT_MISH;
    RUN(run_conv(m, m->conv_pre, p, s));
  }
  if (len64) RUN(launch_zero_tail(x0, len64, min_n, B, c.gen_initial_channel, T, s));
  SVCB_TRY(tap(ctx, SVCB_TAP_GEN_PRE, x0, (size_t)B * c.gen_initial_channel * T));

  const float* x = x0;
  int ch = c.gen_initial_channel;
  int L = T;
  for (int i = 0; i < c.n_ups; ++i) {
    const UpStage& us = m->ups[i];
    const int chn = ch / 2, Ln = L * us.rate;
    float* X = ctx.alloc<float>((size_t)B * chn * Ln);
    float* ACC = ctx.alloc<float>((size_t)B * chn * Ln);
    SVCB_TRY(ctx.check());
    Stage a{x, X, ACC, T1, T2, RA, RB, IMG_HI, IMG_LO, {nullptr, nullptr, nullptr, nullptr}, source, SRCP, Ltot, Lpad,
            B, chn, Ln, c.n_res, nsplit, m->hop, Ln / T, lens, len64 ? len64 + (size_t)i * B : nullptr};
    switch (us.form) {
      case UPS_COMB: SVCB_TRY(run_ups_comb(ctx, us, a)); break;
      case UPS_FUSED: SVCB_TRY(run_ups_fused(ctx, us, a)); break;
      case UPS_POLYPHASE: SVCB_TRY(run_ups_polyphase(ctx, us, a)); break;
    }
    switch (us.noise_form) {
      case NOISE_IN_UPS: break;
      case NOISE_TC: SVCB_TRY(run_noise_tc(ctx, us, a)); break;
      case NOISE_CONV1D: SVCB_TRY(run_noise_conv1d(ctx, us, a)); break;
    }
    SVCB_TRY(tap(ctx, SVCB_TAP_GEN_UP0 + i, X, (size_t)B * chn * Ln));

    const ResBlock* rb = &m->res[(size_t)i * c.n_res];
    const AmpForm* forms = &plan.amp[(size_t)i * c.n_res];
    const size_t mark = ctx.off;
    if (forms[0] == AMP_S2D) {   // (every block of a stage has the same channel count: all or none take this form)
      // two ping-pong S2D images (hi, lo each), cleared once per stage: rows outside the sequences are the
      // convolutions' zero padding; the writers store zeros over an item's first rows past its end (S2D_TAIL)
      const size_t ib = s2d_image_bytes(B, Ln, rb[0].s2d_r);
      uint8_t* base = ctx.alloc<uint8_t>(4 * ib);
      SVCB_TRY(ctx.check());
      for (int q = 0; q < 4; ++q) a.s2d[q] = base + (size_t)q * ib;
      if (!ctx.dry) {
        KernelScope ks("s2d_image_clear", s, 0.0, 4.0 * ib);
        SVCB_CUDA_CHECK(cudaMemsetAsync(base, 0, 4 * ib, s));
      }
    }
    for (int j = 0; j < c.n_res; ++j) {
      const ResBlock& R = rb[j];
      switch (forms[j]) {
        case AMP_S2D: SVCB_TRY(run_amp_s2d(ctx, a, R, j)); break;
        case AMP_BLOCK_FUSED: SVCB_TRY(run_amp_block_fused(ctx, a, R, j)); break;
        case AMP_TC: SVCB_TRY(run_amp_tc(ctx, a, R, j)); break;
        case AMP_FP32: SVCB_TRY(run_amp_fp32(ctx, a, R, j)); break;
      }
    }
    ctx.off = mark;
    // the next upsampler reads the stage mean with zero padding past each ragged item's end (post_fused stops there)
    if (len64 && i + 1 < c.n_ups) RUN(launch_zero_tail(ACC, len64 + (size_t)(i + 1) * B, (long long)min_n * (Ln / T), B, chn, Ln, s));
    SVCB_TRY(tap(ctx, SVCB_TAP_GEN_STAGE0 + i, ACC, (size_t)B * chn * Ln));
    x = ACC; ch = chn; L = Ln;
  }
  // activation_post + conv_post + tanh (generator.py:196-199)
  if (plan.post_fused) {
    RUN(launch_post_fused(x, wave, m->post_act.ea, m->post_act.ib, m->post_act.taps, m->conv_post_h.data(), B, ch, L, s,
                          lens, L / T));
    return SVCB_OK;
  }
  RUN(launch_snake_alias(x, T1, m->post_act.ea, m->post_act.ib, m->post_act.fu, m->post_act.fd, B, ch, L, s));
  {
    ConvParams p = std_conv(m->conv_post, T1, wave, B, L, L, 3);
    p.act = ACT_TANH;
    RUN(launch_conv1d(p, s));
  }
  return SVCB_OK;
}

// ----------------------------------------------------------------------------- model creation
int check_blob_device(const void* dev_blob) {
  if (((uintptr_t)dev_blob & 255) != 0) { set_error("weight blob must be 256-byte aligned"); return SVCB_E_BAD_ALIGN; }
  int dev = 0;
  SVCB_CUDA_CHECK(cudaGetDevice(&dev));
  cudaDeviceProp prop;
  SVCB_CUDA_CHECK(cudaGetDeviceProperties(&prop, dev));
  if (prop.major != 9 || prop.minor != 0) {
    set_error("libsvc_b200 is built for sm_90a only; device is sm_" + std::to_string(prop.major) +
              std::to_string(prop.minor));
    return SVCB_E_UNSUPPORTED;
  }
  return SVCB_OK;
}

int check_workspace(const void* ws, size_t ws_bytes, size_t need, const char* who) {
  if (ws && !((uintptr_t)ws & 255) && ws_bytes >= need) return SVCB_OK;
  set_error(std::string(who) + " workspace too small or misaligned: need " + std::to_string(need) +
            " bytes at a 256-byte boundary, have " + std::to_string(ws_bytes));
  return SVCB_E_WORKSPACE;
}

int check_ragged(const char* who, const int64_t* offsets_host, int32_t B, int32_t min_items, int64_t min_len,
                 const char* unit, const char* why) {
  if (B < min_items) {
    set_error(std::string(who) + ": B = " + std::to_string(B) + (min_items > 0 ? "; need at least one item" : " is negative"));
    return SVCB_E_BAD_SHAPE;
  }
  if (offsets_host[0] < 0) { set_error(std::string(who) + ": negative first offset"); return SVCB_E_BAD_SHAPE; }
  for (int b = 0; b < B; ++b) {
    const int64_t n = offsets_host[b + 1] - offsets_host[b];
    if (n < min_len) {
      set_error(std::string(who) + ": item " + std::to_string(b) + " has " + std::to_string(n) + " " + unit +
                "; need at least " + std::to_string(min_len) + (n < 0 ? " (the offsets decrease)" : "") +
                (why ? std::string("; ") + why : std::string()));
      return SVCB_E_BAD_SHAPE;
    }
  }
  return SVCB_OK;
}

int BlobTensors::read(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table, int32_t n) {
  const char* blob = static_cast<const char*>(dev_blob);
  for (int i = 0; i < n; ++i) {
    const svcb_tensor_entry& e = table[i];
    const std::string name(e.name, strnlen(e.name, sizeof(e.name)));
    if (e.offset_bytes % 256 != 0 || e.offset_bytes + e.numel * sizeof(float) > blob_bytes) {
      set_error("bad table entry: " + name);
      return SVCB_E_BAD_ALIGN;
    }
    map[name] = {reinterpret_cast<const float*>(blob + e.offset_bytes), e.numel};
  }
  return SVCB_OK;
}

struct Resolver : BlobTensors {
  ConvW conv(const std::string& prefix, int cin, int cout, int k, bool bias = true, bool tc = false) {
    ConvW w;
    w.cin = cin; w.cout = cout; w.k = k; w.cout_pad = (cout + 7) / 8 * 8;
    w.w = get(prefix + ".w", (uint64_t)cin * k * w.cout_pad);
    w.b = bias ? get(prefix + ".b", cout) : nullptr;
    if (tc) tc_image(w, prefix + ".tc", cin, cout, k);
    return w;
  }
  // w as a conv of cin -> cout channels and k taps with its tensor-core tile image (pack.py:pack_conv_tc_general)
  void tc_image(ConvW& w, const std::string& name, int cin, int cout, int k) {
    w.cin = cin; w.cout = cout; w.k = k; w.cout_pad = (cout + 7) / 8 * 8;
    tc_tiling(w);
    w.tc = reinterpret_cast<const uint8_t*>(get(name, (uint64_t)w.k * 2 * w.cin_pad * w.ntiles * w.bn / 2));
  }
  SnakeW snake(const std::string& prefix, int ch) {
    SnakeW s;
    s.ea = get(prefix + ".ea", ch); s.ib = get(prefix + ".ib", ch);
    s.fu = get(prefix + ".fu", 12); s.fd = get(prefix + ".fd", 12);
    if (s.fu && s.fd && snake_taps_from_device(s.fu, s.fd, &s.taps) != SVCB_OK) fail(prefix + ".fu/.fd (device read-back failed)");
    return s;
  }
};

static int resolve(svcb_model* m, Resolver& R) {
  const svcb_config& c = m->cfg;
  m->nsplit = c.precision;   // validate_cfg admits 0, 1 and 3, which are the split counts
  const bool tc = m->nsplit != 0;
  m->attn_tc = tc && c.enc_window == 4;   // (and 96 channels per head, which validate_cfg requires)
  const int H = c.hidden_channels, C = c.inter_channels;
  m->pre = R.conv("enc_p.pre", c.ppg_dim, H, 5, true, true);
  m->hub = R.conv("enc_p.hub", c.vec_dim, H, 5, true, true);
  m->pit_emb = R.get("enc_p.pit", 256ull * H);
  m->enc.resize(c.enc_layers);
  for (int i = 0; i < c.enc_layers; ++i) {
    const std::string p = "enc." + std::to_string(i);
    EncLayer& L = m->enc[i];
    L.qkv = R.conv(p + ".qkv", H, 3 * H, 1, true, true);
    L.o = R.conv(p + ".o", H, H, 1, true, true);
    L.ffn1 = R.conv(p + ".ffn1", H, c.filter_channels, c.enc_kernel, true, true);
    L.ffn2 = R.conv(p + ".ffn2", c.filter_channels, H, c.enc_kernel, true, true);
    const uint64_t nr = (uint64_t)(2 * c.enc_window + 1) * (H / c.enc_heads);
    L.ek = R.get(p + ".ek", nr); L.ev = R.get(p + ".ev", nr);
    L.ln1g = R.get(p + ".ln1.g", H); L.ln1b = R.get(p + ".ln1.b", H);
    L.ln2g = R.get(p + ".ln2.g", H); L.ln2b = R.get(p + ".ln2.b", H);
  }
  m->proj = R.conv("enc_p.proj", H, 2 * C, 1, true, true);
  m->flow.resize(c.n_flows);
  for (int f = 0; f < c.n_flows; ++f) {
    const std::string p = "flow." + std::to_string(f);
    FlowLayer& F = m->flow[f];
    F.pre = R.conv(p + ".pre", C / 2, H, 1, true, true);
    F.post = R.conv(p + ".post", H, C / 2, 1, true, true);
    F.snac_w = R.get(p + ".snac.w", (uint64_t)C * c.spk_dim);
    F.snac_b = R.get(p + ".snac.b", C);
    for (int l = 0; l < c.wn_layers; ++l) {
      F.in.push_back(R.conv(p + ".in." + std::to_string(l), H, 2 * H, c.wn_kernel, true, true));
      F.rs.push_back(R.conv(p + ".rs." + std::to_string(l), H, l + 1 < c.wn_layers ? 2 * H : H, 1, true, true));
    }
  }
  const int U = c.gen_input;
  m->ad_sw = R.get("dec.adapter.scale.w", (uint64_t)U * c.spk_dim);
  m->ad_sb = R.get("dec.adapter.scale.b", U);
  m->ad_bw = R.get("dec.adapter.bias.w", (uint64_t)U * c.spk_dim);
  m->ad_bb = R.get("dec.adapter.bias.b", U);
  m->conv_pre = R.conv("dec.conv_pre", U, c.gen_initial_channel, 7, true, true);
  m->merge_w = R.get("dec.merge_w", c.n_harmonics);
  m->merge_b = R.get("dec.merge_b", 1);
  m->ups.resize(c.n_ups);
  m->hop = 1;
  int ch = c.gen_initial_channel;
  for (int i = 0; i < c.n_ups; ++i) {
    UpStage& us = m->ups[i];
    us.rate = c.up_rates[i]; us.k = c.up_kernels[i];
    us.pad = (us.k - us.rate) / 2;
    us.taps = (us.k + us.rate - 1) / us.rate;
    for (int k2 = i + 1; k2 < c.n_ups; ++k2) us.sf *= c.up_rates[k2];
    m->hop *= us.rate;
    const std::string p = "dec.ups." + std::to_string(i);
    for (int r = 0; r < us.rate; ++r)
      us.phase.push_back(R.conv(p + ".ph" + std::to_string(r), ch, ch / 2, us.taps, false, true));
    us.bias = R.get(p + ".b", ch / 2);
    if (us.rate == 4 && us.taps == 2 && i + 1 < c.n_ups) {   // must match pack.py:pack_svc_state_dict (+ the stage's noise conv)
      us.comb_cin1 = (ch + 31) / 32 * 32;
      us.comb_cin2 = us.rate * us.sf + us.sf;         // source samples a frame's rate outputs reach (filter 2 sf, stride sf)
      R.tc_image(us.comb, p + ".comb.tc", us.comb_cin1 + us.comb_cin2, us.rate * (ch / 2), us.taps + 1);
      us.comb.b = R.get(p + ".comb.b", us.comb.cout);
    }
    const int sf = us.sf;
    const int nk = (i + 1 == c.n_ups) ? 1 : 2 * sf;
    us.noise = R.conv("dec.noise." + std::to_string(i), 1, ch / 2, nk);
    if (nk > 8) {
      R.tc_image(us.noise_tc, "dec.noise." + std::to_string(i) + ".tc", sf, ch / 2, 2);
      us.noise_tc.b = us.noise.b;
    }
    // the stage's kernels (comb and noise_tc exist only for stages before the last)
    if (tc && nk <= 8 && ups_fused_supported(ch, ch / 2, us.rate, us.taps, nk)) us.form = UPS_FUSED;
    else if (tc && us.comb.tc && sf / 2 <= SRC_PADF) us.form = UPS_COMB;
    else us.form = UPS_POLYPHASE;
    // phase r's outputs start at q0 (independent of L); with pad >= 0 it has exactly L of them, a stride-1 conv
    for (int r = 0; r < us.rate; ++r) {
      us.q0.push_back(us.pad - r > 0 ? (us.pad - r + us.rate - 1) / us.rate : 0);
      us.phase_tc.push_back(tc && us.phase[r].tc && us.pad >= 0 && us.taps - 1 - us.q0[r] >= 0);
    }
    if (us.form != UPS_POLYPHASE || nk <= 8) us.noise_form = NOISE_IN_UPS;
    else if (tc && us.noise_tc.tc && sf <= 2 * SRC_PADF) us.noise_form = NOISE_TC;
    else us.noise_form = NOISE_CONV1D;
    us.ragged = us.form != UPS_POLYPHASE || (us.noise_form == NOISE_TC && !std::count(us.phase_tc.begin(), us.phase_tc.end(), false));
    ch /= 2;
  }
  m->res.resize((size_t)c.n_ups * c.n_res);
  ch = c.gen_initial_channel;
  for (int i = 0; i < c.n_ups; ++i) {
    ch /= 2;
    for (int j = 0; j < c.n_res; ++j) {
      ResBlock& rb = m->res[(size_t)i * c.n_res + j];
      rb.k = c.res_kernels[j];
      const std::string p = "dec.res." + std::to_string(i * c.n_res + j);
      for (int d = 0; d < 3; ++d) {
        rb.dil[d] = c.res_dilations[j][d];
        rb.c1[d] = R.conv(p + ".c1." + std::to_string(d), ch, ch, rb.k);
        rb.c2[d] = R.conv(p + ".c2." + std::to_string(d), ch, ch, rb.k);
        const int cp = (ch + 15) / 16 * 16;
        const uint64_t tcn = (uint64_t)rb.k * 2 * cp * cp / 2;
        rb.c1_tc[d] = reinterpret_cast<const uint8_t*>(R.get(p + ".c1." + std::to_string(d) + ".tc", tcn));
        rb.c2_tc[d] = reinterpret_cast<const uint8_t*>(R.get(p + ".c2." + std::to_string(d) + ".tc", tcn));
      }
      rb.s2d_r = s2d_link_factor(ch);
      for (int d = 0; d < 3 && rb.s2d_r; ++d) {
        // c1 runs on the fold its plan picks (its blob entry holds the undilated conv's matrices when folded)
        s2d_tap_plan(rb.k, rb.dil[d], rb.s2d_r, rb.s2d1[d]);
        s2d_tap_plan(rb.k, 1, rb.s2d_r, rb.s2d2[d]);
        const uint64_t per_tap = 2ull * 160 * 160 / 2;   // fp32-typed elements of one (hi, lo) pair
        rb.c1_s2d[d] = reinterpret_cast<const uint8_t*>(R.get(p + ".c1." + std::to_string(d) + ".s2d", per_tap * rb.s2d1[d].ntaps));
        rb.c2_s2d[d] = reinterpret_cast<const uint8_t*>(R.get(p + ".c2." + std::to_string(d) + ".s2d", per_tap * rb.s2d2[d].ntaps));
      }
      for (int a = 0; a < 6; ++a) rb.act[a] = R.snake(p + ".act." + std::to_string(a), ch);
      rb.fallback = !tc ? AMP_FP32 : amp_block_fused_supported(ch, rb.k, rb.dil) ? AMP_BLOCK_FUSED : AMP_TC;
      rb.form = m->nsplit == 3 && rb.s2d_r ? AMP_S2D : rb.fallback;
    }
  }
  m->post_act = R.snake("dec.post.act", ch);
  m->conv_post = R.conv("dec.conv_post", ch, 1, 7, false);
  SVCB_TRY(R.status("packed blob"));
  {  // packed [cin][k][cout_pad]: keep output channel 0 of every tap on the host
    const ConvW& w = m->conv_post;
    std::vector<float> packed((size_t)w.cin * w.k * w.cout_pad);
    if (cudaMemcpy(packed.data(), w.w, packed.size() * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) {
      set_error("reading conv_post back failed");
      return SVCB_E_CUDA;
    }
    m->conv_post_h.resize((size_t)w.cin * w.k);
    for (int i = 0; i < w.cin * w.k; ++i) m->conv_post_h[i] = packed[(size_t)i * w.cout_pad];
  }
  return SVCB_OK;
}

// svcb_infer_ragged: SVCB_E_UNSUPPORTED unless the model is at precision 3, every upsampler stops items at their own ends,
// and the generator's plan at T frames takes only forms that do (AMP_TC, AMP_S2D, post_fused) and is its plan at every n[b].
static int ragged_forms(const svcb_model* m, const int32_t* n, int B, int T, const float* wave) {
  const svcb_config& c = m->cfg;
  const auto reject = [](const std::string& why) { set_error("svcb_infer_ragged: " + why); return SVCB_E_UNSUPPORTED; };
  const auto stage = [](int k) { return "generator stage " + std::to_string(k); };
  if (m->nsplit != 3) return reject("needs a model at precision 3; this one has precision " + std::to_string(c.precision));
  const std::string tail = "the generator's tail needs post_fused (a 16-byte aligned wave and 8 | samples)";
  const GenPlan plan(m, T, wave);
  for (int i = 0; i < c.n_ups; ++i) {
    if (!m->ups[i].ragged) return reject(stage(i) + "'s upsampler has no ragged form");
    for (int j = i * c.n_res; j < (i + 1) * c.n_res; ++j)
      if (plan.amp[j] != AMP_TC && plan.amp[j] != AMP_S2D) return reject(stage(i) + "'s AMP blocks have no ragged form");
  }
  if (!plan.post_fused) return reject(tail);
  for (int b = 0; b < B; ++b) {
    const GenPlan pb(m, n[b], wave);
    for (int j = 0; j < c.n_ups * c.n_res; ++j)
      if (pb.amp[j] != plan.amp[j]) return reject(stage(j / c.n_res) + " would leave the space-to-depth form at some length");
    if (!pb.post_fused) return reject(tail);
  }
  return SVCB_OK;
}

// n64[i][b] = n[b] * f.v[i]: each item's length at the input rate of generator stage i (i = 0: frames)
struct StageRates { long long v[SVCB_MAX_UPS + 1]; };
__global__ void stage_lens_kernel(const int* __restrict__ n, long long* __restrict__ n64, StageRates f, int B, int rows) {
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k < B * rows) n64[k] = n[k % B] * f.v[k / B];
}

// prior -> flow -> generator in the workspace (svcb_infer; svcb_workspace_bytes as a dry run).  ragged: first the region
// svcb_infer_ragged stages its lengths in (rl: those lengths, null in the dry run); the pipeline then reads them.
static int run_infer(const svcb_model* m, Ctx& ctx, const float* ppg, const float* vec, const float* pit, const float* spk,
                     const long long* lengths, const float* source, const float* eps, float* wave, int B, int T,
                     bool ragged = false, RaggedLens* rl = nullptr) {
  const int rows = m->cfg.n_ups + 1;
  int* lens = ragged ? ctx.alloc<int>(ragged_lens_bytes(B) / sizeof(int)) : nullptr;
  long long* len64 = ragged ? ctx.alloc<long long>((size_t)rows * B) : nullptr;
  float* zp = ctx.alloc<float>((size_t)B * m->cfg.inter_channels * T);
  float* z = ctx.alloc<float>((size_t)B * m->cfg.inter_channels * T);
  SVCB_TRY(ctx.check());
  if (rl) {
    SVCB_TRY(rl->stage(lens, ctx.stream));
    StageRates f = {{1}};
    for (int i = 0; i < m->cfg.n_ups; ++i) f.v[i + 1] = f.v[i] * m->cfg.up_rates[i];
    stage_lens_kernel<<<(B * rows + 255) / 256, 256, 0, ctx.stream>>>(lens, len64, f, B, rows);
    SVCB_LAUNCH_CHECK("stage_lens");
    lengths = len64;
  }
  const size_t mark = ctx.off;
  SVCB_TRY(run_prior(m, ctx, ppg, vec, pit, lengths, eps, zp, B, T, rl != nullptr));
  ctx.off = mark;
  SVCB_TRY(run_flow(m, ctx, zp, lengths, spk, z, B, T));
  ctx.off = mark;
  return run_generator(m, ctx, spk, z, source, wave, B, T, rl ? len64 : nullptr, rl ? lens : nullptr, rl ? rl->min_out : 0);
}

static int validate_cfg(const svcb_config& c) {
  if (c.precision != 0 && c.precision != 1 && c.precision != 3) { set_error("config: precision must be 0, 1 or 3"); return SVCB_E_UNSUPPORTED; }
  if (c.n_ups < 1 || c.n_ups > SVCB_MAX_UPS || c.n_res < 1 || c.n_res > SVCB_MAX_RES) {
    set_error("config: n_ups / n_res out of range");
    return SVCB_E_BAD_SHAPE;
  }
  if (c.inter_channels % 2 || c.hidden_channels % c.enc_heads || c.hidden_channels / c.enc_heads != 96) {
    set_error("config: hidden_channels/heads must be 96 and inter_channels even");
    return SVCB_E_UNSUPPORTED;
  }
  if (c.n_harmonics < 1 || c.n_harmonics > 32) { set_error("config: n_harmonics"); return SVCB_E_BAD_SHAPE; }
  if (c.gen_initial_channel % (1 << c.n_ups)) {
    set_error("config: gen_initial_channel must be divisible by 2^n_ups");
    return SVCB_E_BAD_SHAPE;
  }
  return SVCB_OK;
}

}  // namespace svcb

using namespace svcb;

extern "C" {

const char* svcb_last_error(void) { return g_err.c_str(); }
int svcb_version(void) { return 100; }
size_t svcb_sizeof(int32_t which) {
  switch (which) {
    case 0: return sizeof(svcb_config);
    case 1: return sizeof(svcb_tensor_entry);
    case 2: return sizeof(svcb_taps);
    case 3: return sizeof(svcb_ivf_config);
    default: return 0;
  }
}
int64_t svcb_last_launch_count(void) { return g_launches; }

void svcb_timing_enable(int32_t on) {
  g_timing = on != 0;
  if (on) {
    for (auto& t : g_timed) { cudaEventDestroy(t.e0); cudaEventDestroy(t.e1); }
    g_timed.clear();
  }
}

const char* svcb_timing_report(void) {
  // caller must have synchronised the stream(s); one line per kernel name:
  // name launches total_ms total_flops total_bytes total_aux_flops
  struct Agg { long n = 0; double ms = 0, flops = 0, bytes = 0, aux = 0; };
  std::map<std::string, Agg> agg;
  for (auto& t : g_timed) {
    float ms = 0.f;
    if (cudaEventElapsedTime(&ms, t.e0, t.e1) != cudaSuccess) continue;
    Agg& a = agg[t.name];
    a.n++; a.ms += ms; a.flops += t.flops; a.bytes += t.bytes; a.aux += t.aux;
  }
  g_report.clear();
  char buf[256];
  for (auto& kv : agg) {
    snprintf(buf, sizeof(buf), "%s %ld %.6f %.6e %.6e %.6e\n", kv.first.c_str(), kv.second.n, kv.second.ms,
             kv.second.flops, kv.second.bytes, kv.second.aux);
    g_report += buf;
  }
  return g_report.c_str();
}

int svcb_model_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host,
                      int32_t n_entries, const svcb_config* cfg_host, svcb_model** out) {
  if (!dev_blob || !table_host || !cfg_host || !out) { set_error("null argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_blob_device(dev_blob));
  SVCB_TRY(validate_cfg(*cfg_host));
  Resolver R;
  SVCB_TRY(R.read(dev_blob, blob_bytes, table_host, n_entries));
  auto m = std::make_unique<svcb_model>();
  m->cfg = *cfg_host;
  SVCB_TRY(resolve(m.get(), R));
  *out = m.release();
  return SVCB_OK;
}

void svcb_model_destroy(svcb_model* m) { delete m; }

size_t svcb_workspace_bytes(const svcb_model* m, int32_t B, int32_t T) {
  if (!m || B <= 0 || T <= 0) return 0;
  Ctx ctx;
  ctx.dry = true;
  run_infer(m, ctx, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, B, T, true);
  return std::max(ctx.peak, source_scan_ws_bytes(B, T, m->cfg.n_harmonics) + 256) + 4096;
}

size_t svcb_source_workspace_bytes(const svcb_model* m, int32_t B, int32_t T) {
  if (!m || B <= 0 || T <= 0) return 0;
  return source_scan_ws_bytes(B, T, m->cfg.n_harmonics) + 4096;
}

static int make_ctx(Ctx& ctx, void* ws, size_t ws_bytes, const svcb_taps* taps, svcb_stream stream) {
  if (!ws || ((uintptr_t)ws & 255)) { set_error("workspace must be non-null and 256-byte aligned"); return SVCB_E_BAD_ALIGN; }
  ctx.base = static_cast<char*>(ws); ctx.cap = ws_bytes; ctx.taps = taps;
  ctx.stream = static_cast<cudaStream_t>(stream);
  return SVCB_OK;
}

int svcb_source(const svcb_model* m, const float* f0, const float* rand_ini, const float* noise,
                float* source, int32_t B, int32_t T, void* ws, size_t ws_bytes, svcb_stream stream) {
  g_launches = 0;
  if (!m || B <= 0 || T <= 0) { set_error("svcb_source: bad shape"); return SVCB_E_BAD_SHAPE; }
  Ctx ctx;
  SVCB_TRY(make_ctx(ctx, ws, ws_bytes, nullptr, stream));
  double* scan = ctx.alloc<double>(source_scan_ws_bytes(B, T, m->cfg.n_harmonics) / sizeof(double));
  SVCB_TRY(ctx.check());
  return launch_source(f0, rand_ini, noise, m->merge_w, m->merge_b, source, scan, B, T, m->hop,
                       m->cfg.n_harmonics, (float)m->cfg.sampling_rate, ctx.stream);
}

int svcb_source2wav(const float* source, int16_t* out, size_t n, svcb_stream stream) {
  g_launches = 0;
  return launch_source2wav(source, out, n, static_cast<cudaStream_t>(stream));
}

int svcb_prior(const svcb_model* m, const float* ppg, const float* vec, const float* pit,
               const int64_t* lengths, const float* eps, float* z_p, int32_t B, int32_t T, void* ws,
               size_t ws_bytes, const svcb_taps* taps, svcb_stream stream) {
  g_launches = 0;
  if (!m || B <= 0 || T <= 0 || !lengths) { set_error("svcb_prior: bad shape or null lengths"); return SVCB_E_BAD_SHAPE; }
  Ctx ctx;
  SVCB_TRY(make_ctx(ctx, ws, ws_bytes, taps, stream));
  return run_prior(m, ctx, ppg, vec, pit, reinterpret_cast<const long long*>(lengths), eps, z_p, B, T);
}

int svcb_flow(const svcb_model* m, const float* z_p, const int64_t* lengths, const float* spk,
              float* z, int32_t B, int32_t T, void* ws, size_t ws_bytes, const svcb_taps* taps,
              svcb_stream stream) {
  g_launches = 0;
  if (!m || B <= 0 || T <= 0 || !lengths) { set_error("svcb_flow: bad shape or null lengths"); return SVCB_E_BAD_SHAPE; }
  Ctx ctx;
  SVCB_TRY(make_ctx(ctx, ws, ws_bytes, taps, stream));
  return run_flow(m, ctx, z_p, reinterpret_cast<const long long*>(lengths), spk, z, B, T);
}

int svcb_generator(const svcb_model* m, const float* spk, const float* z, const float* source,
                   float* wave, int32_t B, int32_t T, void* ws, size_t ws_bytes,
                   const svcb_taps* taps, svcb_stream stream) {
  g_launches = 0;
  if (!m || B <= 0 || T <= 0) { set_error("svcb_generator: bad shape"); return SVCB_E_BAD_SHAPE; }
  Ctx ctx;
  SVCB_TRY(make_ctx(ctx, ws, ws_bytes, taps, stream));
  return run_generator(m, ctx, spk, z, source, wave, B, T);
}

int svcb_infer(const svcb_model* m, const float* ppg, const float* vec, const float* pit,
               const float* spk, const int64_t* lengths, const float* source, const float* eps,
               float* wave, int32_t B, int32_t T, void* ws, size_t ws_bytes, const svcb_taps* taps,
               svcb_stream stream) {
  g_launches = 0;
  if (!m || B <= 0 || T <= 0 || !lengths) { set_error("svcb_infer: bad shape or null lengths"); return SVCB_E_BAD_SHAPE; }
  Ctx ctx;
  SVCB_TRY(make_ctx(ctx, ws, ws_bytes, taps, stream));
  return run_infer(m, ctx, ppg, vec, pit, spk, reinterpret_cast<const long long*>(lengths), source, eps, wave, B, T);
}

int svcb_infer_ragged(const svcb_model* m, const float* ppg, const float* vec, const float* pit, const float* spk,
                      const int32_t* n_frames_host, const float* source, const float* eps, float* wave, int32_t B,
                      int32_t T, void* ws, size_t ws_bytes, svcb_stream stream) {
  g_launches = 0;
  if (!m || B <= 0 || T <= 0 || !n_frames_host) { set_error("svcb_infer_ragged: bad shape or null lengths"); return SVCB_E_BAD_SHAPE; }
  RaggedLens rl;
  SVCB_TRY(rl.validate(n_frames_host, B, T, [](int n) { return n; }, "svcb_infer_ragged", "frames"));
  SVCB_TRY(ragged_forms(m, n_frames_host, B, T, wave));
  Ctx ctx;
  SVCB_TRY(make_ctx(ctx, ws, ws_bytes, nullptr, stream));
  return run_infer(m, ctx, ppg, vec, pit, spk, nullptr, source, eps, wave, B, T, true, &rl);
}

// ---- single-operator entry points
int svcb_op_conv1d(const float* x, const float* w_packed, const float* bias, float* y, int32_t B,
                   int32_t Cin, int32_t Cout, int32_t Tin, int32_t K, int32_t stride,
                   int32_t dilation, int32_t pad, int32_t act, svcb_stream stream) {
  g_launches = 0;
  const int Tout = (Tin + 2 * pad - dilation * (K - 1) - 1) / stride + 1;
  if (Tout <= 0) { set_error("conv1d: empty output"); return SVCB_E_BAD_SHAPE; }
  ConvW w; w.w = w_packed; w.b = bias; w.cin = Cin; w.cout = Cout; w.cout_pad = (Cout + 7) / 8 * 8; w.k = K;
  ConvParams p = std_conv(w, x, y, B, Tin, Tout, pad, dilation, stride);
  p.act = act;
  return launch_conv1d(p, static_cast<cudaStream_t>(stream));
}

int svcb_op_conv_tc(const float* x, const void* w_tc, const float* bias, float* y, const float* res,
                    const int64_t* lengths, int32_t B, int32_t Cin, int32_t Cout, int32_t T, int32_t K,
                    int32_t dilation, int32_t nsplit, int32_t flags, int32_t act, svcb_stream stream) {
  g_launches = 0;
  ConvW w; w.cin = Cin; w.cout = Cout; w.k = K; w.tc = static_cast<const uint8_t*>(w_tc); w.b = bias;
  tc_tiling(w);
  ConvTcParams q = conv_tc_params(w, x, (long long)Cin * T, T, 1, y, B, T, T, dilation, dilation * (K - 1) / 2, nsplit);
  q.res = res; q.lengths = reinterpret_cast<const long long*>(lengths); q.flags = flags; q.act = act;
  return launch_conv_tc(q, static_cast<cudaStream_t>(stream));
}

size_t svcb_op_amp_conv_tc_scratch_bytes(int32_t B, int32_t C, int32_t L) { return 2 * p8_image_bytes(B, C, L) + 512; }

int svcb_op_amp_conv_tc(const float* x, float* y, const float* res, const float* ea, const float* inv_b,
                        const float* fu, const float* fd, const void* w_tc, const float* bias, int32_t B,
                        int32_t C, int32_t L, int32_t K, int32_t dilation, int32_t nsplit, int32_t accum,
                        float out_div, void* scratch, size_t scratch_bytes, svcb_stream stream) {
  g_launches = 0;
  const size_t img = align256(p8_image_bytes(B, C, L));
  SVCB_TRY(check_workspace(scratch, scratch_bytes, 2 * img, "svcb_op_amp_conv_tc"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  void* hi = scratch;
  void* lo = nsplit == 3 ? static_cast<char*>(scratch) + img : nullptr;
  SVCB_TRY(launch_snake_pack(x, hi, lo, ea, inv_b, fu, fd, B, C, L, s));
  AmpConvParams q = amp_conv_params(hi, lo, B, C, L, K, nsplit);
  q.wpk = static_cast<const uint8_t*>(w_tc); q.bias = bias; q.dil = dilation;
  q.y = y; q.res = res; q.accum = accum; q.out_div = out_div;
  return launch_amp_conv_tc(q, s);
}

size_t svcb_op_amp_s2d_link_scratch_bytes(int32_t B, int32_t C, int32_t L) {
  const int r = s2d_link_factor(C);
  if (B <= 0 || !s2d_fits(L, r)) return 0;
  return 4 * align256(s2d_image_bytes(B, L, r)) + 512;
}

// lens_host (may be null): a ragged batch, item b ending at lens_host[b] samples; they go to the device through the
// scratch after the four images
static int op_amp_s2d_link(const char* who, const float* x, float* y, const float* res, float* y_act, const float* ea_in,
                           const float* ib_in, const float* ea_out, const float* ib_out, const float* fu,
                           const float* fd, const void* w_s2d, const float* bias, const int32_t* lens_host, int32_t B,
                           int32_t C, int32_t L, int32_t K, int32_t dilation, int32_t out_dilation, void* scratch,
                           size_t scratch_bytes, svcb_stream stream) {
  g_launches = 0;
  const int r = s2d_link_factor(C);
  if (B <= 0 || !s2d_fits(L, r)) { set_error(std::string(who) + ": need C in {40, 20, 10}, L % (160/C) == 0 and L % 8 == 0"); return SVCB_E_BAD_SHAPE; }
  S2dPlan pl;
  if (!s2d_tap_plan(K, dilation, r, pl)) { set_error(std::string(who) + ": too many taps"); return SVCB_E_BAD_SHAPE; }
  if (out_dilation < 1 || out_dilation > 5 || (out_dilation > 1 && (pl.fold > 1 || !y_act))) {
    set_error(std::string(who) + ": out_dilation must be in [1, 5], and > 1 only with y_act and an unfolded input");
    return SVCB_E_BAD_SHAPE;
  }
  const size_t img = align256(s2d_image_bytes(B, L, r));
  SVCB_TRY(check_workspace(scratch, scratch_bytes, 4 * img + (lens_host ? (size_t)B * sizeof(int32_t) : 0), who));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* b0 = static_cast<char*>(scratch);
  void* img4[4] = {b0, b0 + img, b0 + 2 * img, b0 + 3 * img};   // the input image (hi, lo), then the output image
  int* lens = nullptr;
  if (lens_host) {
    for (int b = 0; b < B; ++b)
      if (lens_host[b] < 8 || lens_host[b] > L || lens_host[b] % 8 || lens_host[b] % r) {
        set_error(std::string(who) + ": item " + std::to_string(b) + " has " + std::to_string(lens_host[b]) +
                  " samples; need a multiple of 8 and of 160/C in [8, L]");
        return SVCB_E_BAD_SHAPE;
      }
    lens = reinterpret_cast<int*>(b0 + 4 * img);
    SVCB_CUDA_CHECK(cudaMemcpyAsync(lens, lens_host, (size_t)B * sizeof(int32_t), cudaMemcpyHostToDevice, s));
  }
  SVCB_CUDA_CHECK(cudaMemsetAsync(b0, 0, 4 * img, s));
  SVCB_TRY(launch_snake_pack_s2d(x, img4[0], img4[1], ea_in, ib_in, fu, fd, B, C, L, s, nullptr, lens, 1, pl.fold));
  SnakeW act{ea_out, ib_out, fu, fd};
  if (y_act) SVCB_TRY(snake_taps_from_device(fu, fd, &act.taps));
  AmpS2dParams q = s2d_link_params(B, C, L, K, img4, img4 + 2, y_act ? &act : nullptr);
  q.wpk = static_cast<const uint8_t*>(w_s2d); q.bias = bias; q.res = res; q.y = y; q.lens = lens;
  q.mlo = pl.mlo; q.ntaps = pl.ntaps; q.tap_cols = pl.tap_cols; q.fin = pl.fold; q.fout = out_dilation;
  SVCB_TRY(launch_amp_s2d_link(q, s));
  if (y_act) SVCB_TRY(launch_s2d_unpack(q.o_hi, q.o_lo, y_act, B, C, L, s, out_dilation));
  return SVCB_OK;
}

int svcb_op_amp_s2d_link(const float* x, float* y, const float* res, float* y_act, const float* ea_in,
                         const float* ib_in, const float* ea_out, const float* ib_out, const float* fu,
                         const float* fd, const void* w_s2d, const float* bias, int32_t B, int32_t C, int32_t L,
                         int32_t K, int32_t dilation, int32_t out_dilation, void* scratch, size_t scratch_bytes,
                         svcb_stream stream) {
  return op_amp_s2d_link("svcb_op_amp_s2d_link", x, y, res, y_act, ea_in, ib_in, ea_out, ib_out, fu, fd, w_s2d, bias,
                         nullptr, B, C, L, K, dilation, out_dilation, scratch, scratch_bytes, stream);
}

int svcb_op_amp_s2d_link_ragged(const float* x, float* y, const float* res, float* y_act, const float* ea_in,
                                const float* ib_in, const float* ea_out, const float* ib_out, const float* fu,
                                const float* fd, const void* w_s2d, const float* bias, const int32_t* lens_host,
                                int32_t B, int32_t C, int32_t L, int32_t K, int32_t dilation, int32_t out_dilation,
                                void* scratch, size_t scratch_bytes, svcb_stream stream) {
  if (!lens_host) { set_error("svcb_op_amp_s2d_link_ragged: lens_host is null"); return SVCB_E_BAD_SHAPE; }
  return op_amp_s2d_link("svcb_op_amp_s2d_link_ragged", x, y, res, y_act, ea_in, ib_in, ea_out, ib_out, fu, fd, w_s2d,
                         bias, lens_host, B, C, L, K, dilation, out_dilation, scratch, scratch_bytes, stream);
}

int svcb_op_snake_alias(const float* x, float* y, const float* ea, const float* inv_b,
                        const float* fu, const float* fd, int32_t B, int32_t C, int32_t L,
                        svcb_stream stream) {
  g_launches = 0;
  return launch_snake_alias(x, y, ea, inv_b, fu, fd, B, C, L, static_cast<cudaStream_t>(stream));
}

int svcb_op_layernorm_c(const float* x, const float* r, const float* gamma, const float* beta,
                        float* y, int32_t B, int32_t C, int32_t T, int32_t gb_batch_stride,
                        float eps, svcb_stream stream) {
  g_launches = 0;
  return launch_layernorm_c(x, r, gamma, beta, y, B, C, T, gb_batch_stride, eps,
                            static_cast<cudaStream_t>(stream));
}

size_t svcb_op_rel_attention_tc_scratch_bytes(int32_t B, int32_t heads, int32_t T) {
  return (B > 0 && heads > 0 && T > 0) ? rel_attention_ws_bytes(B, heads, T) : 0;
}

int svcb_op_rel_attention_tc(const float* qkv, const float* emb_rel_k, const float* emb_rel_v,
                             const int64_t* lengths, float* out, int32_t B, int32_t H, int32_t heads,
                             int32_t window, int32_t T, void* scratch, size_t scratch_bytes, svcb_stream stream) {
  g_launches = 0;
  return launch_rel_attention_tc(qkv, emb_rel_k, emb_rel_v, reinterpret_cast<const long long*>(lengths), out, scratch,
                                 scratch_bytes, B, H, heads, window, T, static_cast<cudaStream_t>(stream));
}

int svcb_op_rel_attention(const float* qkv, const float* emb_rel_k, const float* emb_rel_v,
                          const int64_t* lengths, float* out, int32_t B, int32_t H, int32_t heads,
                          int32_t window, int32_t T, svcb_stream stream) {
  g_launches = 0;
  return launch_rel_attention(qkv, emb_rel_k, emb_rel_v, reinterpret_cast<const long long*>(lengths),
                              out, B, H, heads, window, T, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

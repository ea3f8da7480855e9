// Shared declarations for libsvc_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <algorithm>
#include <atomic>
#include <map>
#include <string>
#include <vector>

#include "svcb.h"

namespace svcb {

void set_error(const std::string& msg);
void count_launch();

// Handle creation (svcb_model_create, svcb_whisper_create, svcb_hubert_create).
// SVCB_E_BAD_ALIGN unless the blob is 256-byte aligned, SVCB_E_UNSUPPORTED unless the current device is sm_90.
int check_blob_device(const void* dev_blob);

// Workspaces: every region starts on a 256-byte boundary.
inline size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }
// A workspace laid out region by region: take(bytes) returns the next region's offset; off is then the bytes so far.
struct WsPlan {
  size_t off = 0;
  size_t take(size_t bytes) {
    const size_t o = off;
    off = align256(off + bytes);
    return o;
  }
};
// SVCB_E_WORKSPACE, with an error naming `who`, unless ws is non-null, 256-byte aligned and holds need bytes.
int check_workspace(const void* ws, size_t ws_bytes, size_t need, const char* who);
// The named tensors of a packed weight blob.
struct BlobTensors {
  std::map<std::string, std::pair<const float*, uint64_t>> map;
  bool ok = true;
  std::string missing;   // the first name get() failed on
  // SVCB_E_BAD_ALIGN for an entry that is not 256-byte aligned or runs past the blob's end
  int read(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table, int32_t n);
  void fail(const std::string& what) { if (ok) missing = what; ok = false; }
  // the tensor, or null when it is missing or has fewer than min_numel elements
  const float* get(const std::string& name, uint64_t min_numel = 0) {
    auto it = map.find(name);
    if (it != map.end() && it->second.second >= min_numel) return it->second.first;
    fail(name);
    return nullptr;
  }
  // SVCB_E_MISSING_TENSOR (with the first missing name) after a failed get()
  int status(const char* blob_kind) const {
    if (ok) return SVCB_OK;
    set_error(std::string("tensor missing or too small in ") + blob_kind + ": " + missing);
    return SVCB_E_MISSING_TENSOR;
  }
};

// Optional per-kernel CUDA-event timing (svcb_timing_enable): a KernelScope brackets one launch
// with two events on the launching stream and books its algorithmic FLOPs / bytes under `name`.
struct KernelScope {
  // flops = SURVEY.md §8(d) algorithmic FLOPs of the launch (conv / GEMM products only), bytes = its
  // algorithmic HBM bytes, aux = activation work (Snake ~70 FLOP per element) reported separately
  KernelScope(const char* name, cudaStream_t s, double flops, double bytes, double aux = 0.0);
  ~KernelScope();
  int slot;
  cudaStream_t stream;
};

#define SVCB_CUDA_CHECK(expr)                                                            \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ::svcb::set_error(std::string(#expr) + ": " + cudaGetErrorString(_e));             \
      return SVCB_E_CUDA;                                                                \
    }                                                                                    \
  } while (0)

#define SVCB_LAUNCH_CHECK(what)                                                          \
  do {                                                                                   \
    ::svcb::count_launch();                                                              \
    cudaError_t _e = cudaGetLastError();                                                 \
    if (_e != cudaSuccess) {                                                             \
      ::svcb::set_error(std::string("launch ") + what + ": " + cudaGetErrorString(_e));  \
      return SVCB_E_CUDA;                                                                \
    }                                                                                    \
  } while (0)

// Per-device caches: cudaFuncAttributeMaxDynamicSharedMemorySize and the SM count belong to a device
// (context), not to the process — a handle re-packed on another GPU of the same process must set the
// attribute again there.  Lock-free: a racing thread at worst repeats an idempotent call.
constexpr int kMaxDevices = 64;
struct DevSmemCache {
  std::atomic<size_t> bytes[kMaxDevices];
};
template <typename Kern>
inline cudaError_t ensure_dyn_smem(Kern kernel, size_t bytes, DevSmemCache& cache) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev < 0 || dev >= kMaxDevices)
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  size_t seen = cache.bytes[dev].load(std::memory_order_relaxed);
  if (bytes <= seen) return cudaSuccess;
  e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return e;
  while (seen < bytes && !cache.bytes[dev].compare_exchange_weak(seen, bytes, std::memory_order_relaxed)) {
  }
  return cudaSuccess;
}
int device_sm_count();   // of the current device (cached per device); 0 on error

#define SVCB_TRY(expr)            \
  do {                            \
    int _s = (expr);              \
    if (_s != SVCB_OK) return _s; \
  } while (0)

// Ragged batches of flat buffers with int64 host offsets (spec, resample, pcm16, VAD, speaker mel / embed).  A pass of
// up to G items rides in the kernel parameters: item b reads [in[b], in[b+1]) and writes [out[b], out[b+1]); output
// offsets count from the batch's first item.
template <int G>
struct ItemPass {
  int n;
  long long in[G + 1];
  long long out[G + 1];
};
// SVCB_E_BAD_SHAPE, with an error naming `who`, unless B >= min_items, offsets[0] >= 0 and every item is at least
// min_len `unit` long; `why`, when given, ends the message.
int check_ragged(const char* who, const int64_t* offsets_host, int32_t B, int32_t min_items, int64_t min_len,
                 const char* unit, const char* why);
// Runs body(pass, g0) on each pass of up to G items (g0 = its first item), with out[i + 1] = out[i] + out_len(item i's
// length) continued from the pass before.  Returns the first status that is not SVCB_OK.
template <int G, class OutLen, class Body>
int for_each_pass(const int64_t* offsets_host, int32_t B, OutLen out_len, Body body) {
  long long o = 0;
  for (int g0 = 0; g0 < B; g0 += G) {
    ItemPass<G> p;
    p.n = std::min(G, B - g0);
    p.out[0] = o;
    for (int i = 0; i <= p.n; ++i) p.in[i] = offsets_host[g0 + i];
    for (int i = 0; i < p.n; ++i) p.out[i + 1] = p.out[i] + out_len(p.in[i + 1] - p.in[i]);
    o = p.out[p.n];
    SVCB_TRY(body(static_cast<const ItemPass<G>&>(p), g0));
  }
  return SVCB_OK;
}
#ifdef __CUDACC__
// The item of a pass's offsets (in or out) that holds position x < off[n]: the first b' >= b with off[b' + 1] > x.
__device__ __forceinline__ int item_of(const long long* off, long long x, int b = 0) {
  while (off[b + 1] <= x) ++b;
  return b;
}
#endif

// sin() for the Snake activations of the tensor-core / fused paths: two-constant Cody-Waite reduction
// to [-pi, pi] followed by the hardware approximation.  `__sinf` alone multiplies by 1/2pi in fp32 first,
// so its absolute error grows like |x| * 2^-24: trained BigVGAN log-alphas reach e^alpha ~ 10-50, i.e.
// arguments in the hundreds (round-1 advice).  Reduced, the error stays at the MUFU level (~4e-7) for
// |x| < 1e5; four extra FMA-pipe instructions per value.
__device__ __forceinline__ float snake_sin(float x) {
  const float k = (fmaf(x, 0.15915494309189535f, 12582912.f)) - 12582912.f;   // rint(x / 2pi), |x| < 2^22
  float r = fmaf(k, -6.28125f, x);                   // 2pi = 6.28125 (exact in 8 bits) + 1.9353071795864769e-3
  r = fmaf(k, -1.9353071795864769e-3f, r);
  return __sinf(r);
}

// cos(2x) with the same reduction (for sin^2 x = (1 - cos 2x) / 2): x = k pi + r, |r| <= pi/2, cos 2x = cos 2r.
__device__ __forceinline__ float snake_cos2(float x) {
  const float k = (fmaf(x, 0.3183098861837907f, 12582912.f)) - 12582912.f;    // rint(x / pi)
  float r = fmaf(k, -3.140625f, x);                  // pi = 3.140625 (exact in 9 bits) + 9.6765358979e-4
  r = fmaf(k, -9.676535897932e-4f, r);
  return __cosf(r + r);
}

// The 12 + 12 alias-filter taps of a SnakeAlias BY VALUE, paired for the f32x2 pair FMAs (f2_fma; a tap pair is a uniform-
// register pair as an operand: no register holds a tap).  fup[j] = 2 * (up[11-2j], up[10-2j]) (UpSample1d's
// ratio gain folded in, exact); fdp[m] = (dn[2m+1], dn[2m+2]); the decimator's two end taps apart.
struct SnakeTapsV {
  float2 fup[6], fdp[5];
  float fd0, fd11;
};
inline SnakeTapsV snake_taps_pack(const float* up12, const float* dn12) {
  SnakeTapsV t;
  for (int j = 0; j < 6; ++j) t.fup[j] = make_float2(2.f * up12[11 - 2 * j], 2.f * up12[10 - 2 * j]);
  for (int m = 0; m < 5; ++m) t.fdp[m] = make_float2(dn12[2 * m + 1], dn12[2 * m + 2]);
  t.fd0 = dn12[0]; t.fd11 = dn12[11];
  return t;
}
bool post_fused_supported(int C, int L, int K, const float* x, const float* wave);
// lens (device, may be null): a ragged batch, item b ending at lens[b] * lscale samples; its later samples of wave are zero
int launch_post_fused(const float* x, float* wave, const float* ea, const float* inv_b, const SnakeTapsV& tp,
                      const float* w_host, int B, int C, int L, cudaStream_t s, const int* lens = nullptr, int lscale = 1);
// device taps -> SnakeTapsV through a synchronous copy (unit-test entry points; the model keeps host copies)
int snake_taps_from_device(const float* fu_dev, const float* fd_dev, SnakeTapsV* out);

#ifdef __CUDACC__
// f32x2 pair arithmetic, one correctly rounded fp32 operation per lane (Hopper has no packed FFMA2 / FMUL2 / FADD2:
// the pairs keep the even / odd phases of the FIRs together and compile to two scalar instructions each).
__device__ __forceinline__ float2 f2_mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 f2_add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }
__device__ __forceinline__ float2 f2_fma(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
#endif

#ifdef __CUDACC__
// SnakeAlias of 8 consecutive samples n0 .. n0+7 from the 24 inputs x[0..24) = signal[n0-8 .. n0+16)
// (alias/resample.py:25-33 up x2, alias/act.py:79-92 Snake, alias/filter.py:86-94 + resample.py:52-58 down x2),
// all FIR and range-reduction arithmetic as packed f32x2 FMAs: the pair V[p] = (v[2p], v[2p+1]) of the 2x signal
// is one f2_fma chain over the input pairs (x[p+2+j], x[p+3+j]); sin^2 = (1 - cos 2r) / 2 with the two-constant
// reduction of snake_cos2; the decimator sums five pair products + its two end taps.  hb = 0.5 / (exp(beta) + eps).
// first / last: the run starts at sample 0 / ends at the last sample — the 2x signal is replicate-padded there.
__device__ __forceinline__ void snake8_packed(const float (&x)[24], const SnakeTapsV& tp, float a_, float hb_, float (&o)[8],
                                              bool first = false, bool last = false) {
  float2 V[14];
  const float2 a2 = make_float2(a_, a_), hb2 = make_float2(hb_, hb_), nhb2 = make_float2(-hb_, -hb_);
#pragma unroll
  for (int p = 0; p < 14; ++p) {
    float2 U = f2_mul(make_float2(x[p + 2], x[p + 3]), tp.fup[0]);
#pragma unroll
    for (int j = 1; j < 6; ++j) U = f2_fma(make_float2(x[p + 2 + j], x[p + 3 + j]), tp.fup[j], U);
    const float2 t = f2_mul(U, a2);
    const float2 kq = f2_add(f2_fma(t, make_float2(0.3183098861837907f, 0.3183098861837907f), make_float2(12582912.f, 12582912.f)),
                                 make_float2(-12582912.f, -12582912.f));
    float2 rr = f2_fma(kq, make_float2(-3.140625f, -3.140625f), t);
    rr = f2_fma(kq, make_float2(-9.676535897932e-4f, -9.676535897932e-4f), rr);
    rr = f2_add(rr, rr);
    const float2 cs = make_float2(__cosf(rr.x), __cosf(rr.y));
    V[p] = f2_fma(nhb2, cs, f2_add(U, hb2));
  }
  if (first) {   // v[0 .. 6) = v[6]
    const float2 e = make_float2(V[3].x, V[3].x);
    V[0] = e; V[1] = e; V[2] = e;
  }
  if (last) {    // v[22 .. 28) = v[21]
    const float2 e = make_float2(V[10].y, V[10].y);
    V[11] = e; V[12] = e; V[13] = e;
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {   // o_i = sum_k v[2i + 1 + k] dn[k]
    float2 acc = f2_mul(V[i + 1], tp.fdp[0]);
#pragma unroll
    for (int m = 1; m < 5; ++m) acc = f2_fma(V[i + 1 + m], tp.fdp[m], acc);
    o[i] = fmaf(V[i].y, tp.fd0, fmaf(V[i + 6].x, tp.fd11, acc.x + acc.y));
  }
}
#endif

#ifdef __CUDACC__
// Direct fp32 DFT of real 1024-sample frames held in shared memory, for CTAs of 256 threads (spk_mel_kernel,
// spec_kernel).  tw[n] = (cos, sin)(2 pi n / 1024); bin k's twiddle for sample n is tw[k n mod 1024].
constexpr int kDftN = 1024, kDftThreads = 256;
__device__ __forceinline__ void dft1024_twiddles(float2* tw, int tid) {
  for (int n = tid; n < kDftN; n += kDftThreads) {
    float s, c;
    sincospif(2.f * (float)n / (float)kDftN, &s, &c);
    tw[n] = make_float2(c, s);
  }
}
// Bins tid and tid + 256 of FT frames xw[f][0..1024): one twiddle load feeds 2 x FT FMAs.  mg[h][f] = mag(re, im) of
// bin tid + 256 h, frame f.  Bin 512 (the alternating sum) is left to the caller.
template <int FT, class Mag>
__device__ __forceinline__ void dft1024_bins(const float2* tw, const float (*xw)[kDftN], int tid, float (&mg)[2][FT], Mag mag) {
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = tid + kDftThreads * h;
    float re[FT], im[FT];
#pragma unroll
    for (int f = 0; f < FT; ++f) { re[f] = 0.f; im[f] = 0.f; }
#pragma unroll 2
    for (int n = 0; n < kDftN; n += 4) {
      const float2 t0 = tw[(k * n) & (kDftN - 1)], t1 = tw[(k * (n + 1)) & (kDftN - 1)];
      const float2 t2 = tw[(k * (n + 2)) & (kDftN - 1)], t3 = tw[(k * (n + 3)) & (kDftN - 1)];
#pragma unroll
      for (int f = 0; f < FT; ++f) {
        const float4 x = *reinterpret_cast<const float4*>(&xw[f][n]);
        re[f] = fmaf(x.x, t0.x, re[f]); im[f] = fmaf(x.x, t0.y, im[f]);
        re[f] = fmaf(x.y, t1.x, re[f]); im[f] = fmaf(x.y, t1.y, im[f]);
        re[f] = fmaf(x.z, t2.x, re[f]); im[f] = fmaf(x.z, t2.y, im[f]);
        re[f] = fmaf(x.w, t3.x, re[f]); im[f] = fmaf(x.w, t3.y, im[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < FT; ++f) mg[h][f] = mag(re[f], im[f]);
  }
}
// Bin 512 of one frame: the alternating sum, accumulated pair by pair.
__device__ __forceinline__ float dft1024_nyquist(const float* x) {
  float s = 0.f;
  for (int n = 0; n < kDftN; n += 2) s += x[n] - x[n + 1];
  return s;
}
#endif

// ----------------------------------------------------------------------------- conv1d
enum ConvFlags : int {
  CONV_IN_MASK = 1,    // x[b,:,t] treated as 0 for t >= lengths[b]
  CONV_OUT_MASK = 2,   // result multiplied by (t_out < lengths[b])
  CONV_GATE = 4,       // packed channels are (tanh_c, sigmoid_c) pairs -> Cout/2 outputs
  CONV_ACCUM = 8,      // y = y_old + v
};
enum ConvAct : int { ACT_NONE = 0, ACT_RELU = 1, ACT_MISH = 2, ACT_GELU = 3, ACT_TANH = 4 };

struct ConvParams {
  const float* x = nullptr;
  long long sxb = 0, sxc = 0, sxt = 1;  // element strides of x[b, ci, t]
  const float* w = nullptr;             // packed [Cin][K][CoutPad]
  int cout_pad = 0;
  const float* bias = nullptr;          // [Cout] (packed order) or null
  float* y = nullptr;
  long long syb = 0, syc = 0, syt = 1;  // element strides of y[b, co, t]
  const float* res = nullptr;           // residual, indexed like y (same strides), or null
  const long long* lengths = nullptr;   // [B] int64 or null
  int B = 0, Cin = 0, Cout = 0, Tin = 0;
  int K = 1, stride = 1, dil = 1, pad = 0;
  int q0 = 0, nq = 0;                   // outputs q = q0 .. q0+nq-1 at y time index q - q0; x index = q*stride + j*dil - pad
  int flags = 0;
  int act = ACT_NONE;
  float out_div = 0.f;                  // if != 0: v = v / out_div (after accumulate)
};
int launch_conv1d(const ConvParams& p, cudaStream_t s);

// ----------------------------------------------------------------------------- tensor-core AMP conv
struct AmpConvParams {
  const void* a_hi = nullptr;   // operand image bf16 [B][Cp/8][Lp][8] written by snake_pack
  const void* a_lo = nullptr;   // low split part (nsplit == 3) or null
  int Lp = 0;                   // image rows = p8_rows(L)
  float* y = nullptr;           // [B, C, L]
  const float* res = nullptr;   // residual [B, C, L] or null
  const uint8_t* wpk = nullptr; // bf16 [K][2 (hi,lo)][Cp/8][Cp][8]  (pack.py:pack_conv_tc)
  const float* bias = nullptr;  // [C]
  int B = 0, C = 0, Cp = 0, L = 0, K = 1, dil = 1;
  int nsplit = 3;               // 1 = bf16, 3 = bf16x3 split
  int accum = 0;                // y = y_old + v
  float out_div = 0.f;          // then v / out_div when != 0
};
int launch_amp_conv_tc(const AmpConvParams& p, cudaStream_t s);
size_t amp_conv_tc_smem_bytes(int Cp, int K, int dil, int nsplit);
// SnakeAlias(x[B,C,L]) -> bf16 hi (and lo, may be null) operand images
// taps: host copy of the filter taps, or null (then read back from fu / fd with a synchronous copy: test entry points)
// lens (device, may be null): a ragged batch, item b ending at lens[b] * lscale samples; its later image rows are zero
int launch_snake_pack(const float* x, void* hi, void* lo, const float* ea, const float* inv_b, const float* fu,
                      const float* fd, int B, int C, int L, cudaStream_t s, const SnakeTapsV* taps = nullptr,
                      const int* lens = nullptr, int lscale = 1);
size_t p8_image_bytes(int B, int C, int L);
int p8_rows(int L);

// ----------------------------------------------------------------------------- space-to-depth AMP links (C = 20, 10)
struct AmpS2dParams {
  const void* a_hi = nullptr;   // input S2D image (bf16 hi) [B][20][Rp][8] — SnakeAlias already applied
  const void* a_lo = nullptr;
  void* o_hi = nullptr;         // output S2D image = SnakeAlias_next(result), or null
  void* o_lo = nullptr;
  const uint8_t* wpk = nullptr; // bf16 [ntaps][2 (hi, lo)][20][160][8], output columns in phase-group order
                                // (pack.py:pack_conv_s2d_slots)
  const float* bias = nullptr;  // [C]
  const float* res = nullptr;   // residual [B, C, L] fp32 or null
  float* y = nullptr;           // fp32 result [B, C, L] or null
  const float *ea = nullptr, *ib = nullptr, *fu = nullptr, *fd = nullptr;   // Snake of the output image
  SnakeTapsV taps = {};         // ... its filter taps BY VALUE: kernel parameters live in the constant bank, so the
                                // FIR FMAs take them as operands and no register holds a tap
  int B = 0, C = 0, L = 0, K = 0;   // K = taps of the original conv (bookkeeping only)
  int Rp = 0;                   // image rows per (item, octet) = s2d_rows(L, r)
  int fin = 1, fout = 1;        // folds of the input and the output image (amp_s2d.cu; at most one > 1)
  int ntaps = 0, mlo = 0;       // Toeplitz row offsets -mlo .. ntaps-1-mlo (pack.py:s2d_taps); row shift m * fin
  int halo = 0, stride = 0, a_off = 0;   // tile geometry (s2d_tile): set by launch_amp_s2d_link
  uint64_t tap_cols = 0;        // 3 bits per tap (s2d_tap_plan): the output columns its matrix can reach
  int accum = 0;               // y = y_old + v
  float out_div = 0.f;          // then / out_div when != 0
  const int* lens = nullptr;    // ragged batch: item b ends at lens[b] * lscale samples (a multiple of r), or null
  int lscale = 1;
};
// Head-major QKV layout the Whisper attention kernel reads (written by the QKV GEMM's epilogue 4): per item
// b, per w in {q, k, v}, per head h one block of Tp x 64 bf16 (Tp = T rounded up to 128 rows, pad rows zero);
// q blocks are [Tp/128][8 octets][128 rows][8], k and v blocks [Tp/64][8 octets][64 rows][8] — every operand
// tile of the attention MMAs is one contiguous SWIZZLE_NONE panel (K-major for q, k; MN-major for v).
__host__ __device__ inline int qkv_heads_tp(int T) { return (T + 127) / 128 * 128; }
__host__ __device__ inline size_t qkv_heads_off(int b, int w, int h, int t, int d, int heads, int Tp) {
  const size_t base = (((size_t)b * 3 + w) * heads + h) * (size_t)Tp * 64;
  return w == 0 ? base + (size_t)(t >> 7) * 8192 + (size_t)(d >> 3) * 1024 + (size_t)(t & 127) * 8 + (d & 7)
                : base + (size_t)(t >> 6) * 4096 + (size_t)(d >> 3) * 512 + (size_t)(t & 63) * 8 + (d & 7);
}
int launch_amp_s2d_link(const AmpS2dParams& p, cudaStream_t s);
int launch_snake_pack_s2d(const float* x, void* hi, void* lo, const float* ea, const float* inv_b, const float* fu,
                          const float* fd, int B, int C, int L, cudaStream_t s, const SnakeTapsV* taps = nullptr,
                          const int* lens = nullptr, int lscale = 1, int fold = 1);
int launch_s2d_unpack(const void* hi, const void* lo, float* y, int B, int C, int L, cudaStream_t s, int fold = 1);
int s2d_rows(int L, int r);
size_t s2d_image_bytes(int B, int L, int r);
// How a link runs: the fold of its input image, its Toeplitz taps over rows of r samples of that image (pack.py:
// s2d_taps of the conv, or of the undilated conv when folded) and, per tap, the output columns it reaches
// (pack.py:s2d_tap_cols) as AmpS2dParams::tap_cols
struct S2dPlan {
  int fold = 1, mlo = 0, ntaps = 0;
  uint64_t tap_cols = 0;
};
struct S2dTile {
  int halo = 0, stride = 0, a_off = 0;
};
// The plan of a c1 link, Conv1d(k, dil) (pack.py:s2d_fold); false when there are more taps than fit
bool s2d_tap_plan(int k, int dil, int r, S2dPlan& pl);
S2dTile s2d_tile(int r, int fin, int fout, int mlo, int mhi);

// ----------------------------------------------------------------------------- fused AMP block (C = 10, 20)
struct AmpBlockParams {
  const float* x = nullptr;      // [B, C, L] stage input
  float* y = nullptr;            // [B, C, L] stage accumulator
  int B = 0, C = 0, L = 0, K = 3;
  int dil[3] = {1, 3, 5};
  const float *w1[3], *b1[3], *w2[3], *b2[3];   // packed [ci][j][cout_pad] weights, [C] biases
  int cout_pad = 0;
  const float *ea[6], *ib[6], *fu[6], *fd[6];   // SnakeAlias parameters of activations 0..5
  int accum = 0;                 // y = y_old + block(x)
  float out_div = 0.f;           // then / out_div when != 0
};
int launch_amp_block_fused(const AmpBlockParams& p, cudaStream_t s);

// polyphase ConvTranspose1d (rate 2, 2 taps per phase) + short noise conv + biases in one pass
struct UpsFusedParams {
  const float* x = nullptr;            // [B][Cin][L]
  const float* wph[2] = {nullptr, nullptr};  // phase sub-filters, packed [Cin][M][cout_pad]
  const float* bias = nullptr;         // [Cout]
  const float* src = nullptr;          // harmonic source [B][Ltot]
  const float* wn = nullptr;           // noise conv, packed [1][Kn][cout_pad_n]
  const float* bn = nullptr;           // [Cout]
  float* y = nullptr;                  // [B][Cout][Ln]
  int B = 0, Cin = 0, Cout = 0, L = 0, Ln = 0, rate = 0, M = 0, pad = 0, cout_pad = 0;
  int Kn = 0, sf = 1, padn = 0, cout_pad_n = 0;
  long long Ltot = 0;
  const int* lens = nullptr;           // ragged batch: item b's source ends at lens[b] * src_scale samples, or null
  int src_scale = 1;
};
int launch_ups_fused(const UpsFusedParams& p, cudaStream_t s);
// lens (device, may be null): per-item sample counts of a ragged batch, each in [201, N]
int launch_log_mel(const float* audio, const float* filt, const float* noise, float gain, float* out,
                   unsigned* scratch, int B, int N, int n_mels, cudaStream_t s, const int* lens = nullptr);
bool ups_fused_supported(int Cin, int Cout, int rate, int taps, int Kn);
bool amp_block_fused_supported(int C, int K, const int* dil);

// ----------------------------------------------------------------------------- general tensor-core conv
constexpr int kConvTcKch = 32;   // input channels per chunk (the K of one A panel)
struct ConvTcParams {
  const float* x = nullptr;
  long long sxb = 0, sxc = 0, sxt = 1;   // element strides of x[b, ci, t]
  const uint8_t* wpk = nullptr;          // bf16 tiles [K][ncc][2][ntiles][kConvTcKch/8][bn][8] (pack.py:pack_conv_tc_general)
  const float* bias = nullptr;           // [Cout] (packed order) or null
  float* y = nullptr;                    // [B, Cout(/2 if gated), Tout] contiguous
  const float* res = nullptr;            // indexed like y, or null
  const long long* lengths = nullptr;
  int B = 0, Cin = 0, cin_pad = 0, Cout = 0, Tin = 0, Tout = 0;
  int K = 1, dil = 1, pad = 0;
  int bn = 128, ntiles = 1;
  int nsplit = 3;
  int flags = 0, act = 0;
  // optional second input (pack.py:ups_combined): packed input channels cin1 .. cin1 + cin2 are x2[b][t * sx2t + c]
  // (channel-contiguous, e.g. windows of the padded harmonic source); channels Cin .. cin1 are zero padding
  const float* x2 = nullptr;
  long long sx2b = 0, sx2t = 0;
  int cin1 = 0, cin2 = 0;
  int ilv = 0;   // 2 or 4: output channel cp = co * ilv + s is sample ilv * t + s of y[b, co, :] (y is [B, Cout / ilv, Tout * ilv]):
                 // the combined polyphase form of a transposed convolution (pack.py:ups_combined); no res / accumulate / gate
};
int launch_conv_tc(const ConvTcParams& p, cudaStream_t s);

// ----------------------------------------------------------------------------- snake alias
int launch_snake_alias(const float* x, float* y, const float* ea, const float* inv_b,
                       const float* fu, const float* fd, int B, int C, int L, cudaStream_t s);

// ----------------------------------------------------------------------------- norm / attention / small ops
int launch_layernorm_c(const float* x, const float* r, const float* gamma, const float* beta,
                       float* y, int B, int C, int T, int gb_batch_stride, float eps,
                       cudaStream_t s);
// tensor-core form (csrc/rel_attn_tc.cu): bf16x3 split operands, scratch = rel_attention_ws_bytes()
size_t rel_attention_ws_bytes(int B, int heads, int T);
int launch_rel_attention_tc(const float* qkv, const float* ek, const float* ev, const long long* lengths, float* out,
                            void* ws, size_t ws_bytes, int B, int H, int heads, int window, int T, cudaStream_t s);
int launch_rel_attention(const float* qkv, const float* ek, const float* ev,
                         const long long* lengths, float* out, int B, int H, int heads, int window,
                         int T, cudaStream_t s);
// y[b,o] = bias[o] + sum_i W[o,i] x[b,i]
int launch_linear_small(const float* x, const float* W, const float* bias, float* y, int B,
                        int In, int Out, cudaStream_t s);
// x[b,c,t] += emb[f0_to_coarse(pit[b,t])][c]   (vits/utils.py:20-33 + models.py:47)
int launch_pitch_embed_add(float* x, const float* pit, const float* emb, int B, int C, int T,
                           cudaStream_t s);
// z_p = (m + eps*exp(logs)) * mask, stats = [B,2C,T] (m | logs)   (models.py:50-51)
int launch_reparam(const float* stats, const float* eps, const long long* lengths, float* z_p,
                   int B, int C, int T, cudaStream_t s);
// coupling layer front: xin [B,C,T] (pre-flip), s [B,C] = snac(spk) (m | v):
//   y[:, :C/2] = flip(xin)[:, :C/2];  x0n = (x0 - s_m) * exp(-s_v) * mask
int launch_coupling_pre(const float* xin, const float* s, const long long* lengths, float* y,
                        float* x0n, int B, int C, int T, cudaStream_t s_);
// coupling layer back: y[:, C/2:] = (s_m + ((x1 - m) * mask) * exp(s_v)) * mask, x1 = flip(xin)[:, C/2:]
int launch_coupling_post(const float* xin, const float* s, const float* m, const long long* lengths,
                         float* y, int B, int C, int T, cudaStream_t s_);
// WN layer tail (modules.py:196-202): rs [B,2H,T] (or [B,H,T] when last):
//   not last: x = (x + rs[:, :H]) * mask ; out (+)= rs[:, H:]      last: out (+)= rs ; out *= mask
int launch_wn_update(float* x, float* out, const float* rs, const long long* lengths, int B, int H,
                     int T, int first, int last, cudaStream_t s);

// ----------------------------------------------------------------------------- NSF source
int launch_source(const float* f0, const float* rand_ini, const float* noise, const float* merge_w,
                  const float* merge_b, float* source, double* scan_ws, int B, int T, int hop,
                  int n_harm, float sampling_rate, cudaStream_t s);
size_t source_scan_ws_bytes(int B, int T, int n_harm);
int launch_source2wav(const float* src, int16_t* out, size_t n, cudaStream_t s);

// ----------------------------------------------------------------------------- Whisper / HuBERT transformer kernels
// bf16 wgmma GEMM over tile images with fused epilogues (each one is described in whisper_gemm.cu)
enum GemmEpi : int { EPI_GELU_BF16_IMAGE = 1, EPI_RESID_F32 = 2, EPI_GELU_ADD_F32 = 3, EPI_QKV_HEADS = 4,
                     EPI_GELU_CONV2_IMG = 5, EPI_GELU_VALID_S2_IMG = 6, EPI_GELU_ADD_F32_LD = 7, EPI_IVF_TOPK = 8 };
// lens (device, may be null): per-item frame counts of a ragged batch, read by epilogue 5 only
int launch_gemm_tc(const void* A_bf16, const void* W_bf16, const float* bias, void* out, const float* res,
                   int M, int N, int K, GemmEpi epi, cudaStream_t s, int res_mod = 0, int aux = 0, const int* lens = nullptr);
int launch_im2col_s1_image(const float* mel, void* img, int B, int n_mels, int n, cudaStream_t s);
int launch_im2col_rows_image(const float* x, void* img, int B, int T, int ld, int c0, int cg, int taps, int pad, cudaStream_t s,
                             const int* lens = nullptr);
// ragged batches: host ints -> device dst[0, n), stream-ordered, without a host-to-device copy
int launch_stage_ints(const int* host, int n, int* dst, cudaStream_t s);
// ragged batches: zero the rows t >= lens[b] (device array, every lens[b] >= min_len) of each item of fp32 [B * T, width]
int launch_zero_tail_rows(float* out, const int* lens, int B, int T, int width, int min_len, cudaStream_t s);
// The per-item lengths of a ragged batch (svcb_whisper_encode_ragged, svcb_hubert_units_ragged) and the output rows each
// item gets.  validate() checks them on the host before any launch; stage() puts both in the workspace region of
// ragged_lens_bytes(B) the layout owns.  Without lengths (a dense batch) nothing is staged and lens / out_lens stay null.
inline size_t ragged_lens_bytes(int B) { return 8 * (size_t)B; }
struct RaggedLens {
  std::vector<int> host;   // [lengths of items 0 .. B-1][output lengths of items 0 .. B-1]
  int B = 0, min_out = 0;
  const int *lens = nullptr, *out_lens = nullptr;   // on the device, after stage()
  // each len[b] must be in [1, max_len] and give out_len(len[b]) >= 1
  template <class OutLen>
  int validate(const int32_t* len, int batch, int max_len, OutLen out_len, const char* who, const char* unit) {
    if (!len) return SVCB_OK;
    B = batch;
    host.resize(2 * (size_t)B);
    for (int b = 0; b < B; ++b) {
      const int n = len[b], r = n >= 1 && n <= max_len ? out_len(n) : 0;
      if (r < 1) {
        set_error(std::string(who) + ": item " + std::to_string(b) + " has " + std::to_string(n) + " " + unit + "; need 1.." +
                  std::to_string(max_len) + " and at least one output row");
        return SVCB_E_BAD_SHAPE;
      }
      host[b] = n;
      host[B + b] = r;
    }
    min_out = *std::min_element(host.begin() + B, host.end());
    return SVCB_OK;
  }
  int stage(void* region, cudaStream_t s) {
    if (host.empty()) return SVCB_OK;
    int* d = static_cast<int*>(region);
    lens = d;
    out_lens = d + B;
    return launch_stage_ints(host.data(), (int)host.size(), d, s);
  }
  // zero the rows past each item's own of the fp32 output [B * T, width]
  int zero_tail(float* out, int T, int width, cudaStream_t s) const {
    return out_lens ? launch_zero_tail_rows(out, out_lens, B, T, width, min_out, s) : SVCB_OK;
  }
};
int launch_rowmajor_to_image(const void* src, void* dst, int R, int K, int rows, cudaStream_t s);
int launch_image_to_rowmajor(const void* src, void* dst, int R, int K, cudaStream_t s);
int launch_qkv_rowmajor_to_heads(const void* src, void* dst, int B, int T, int D, cudaStream_t s);
// lens (device, may be null): per-item position counts of a ragged batch, each in [1, T]
int launch_whisper_attention_tc(const void* qkv_img, void* out_img, int B, int T, int D, int heads, int vswap, cudaStream_t s,
                                const int* lens = nullptr);
// row LayerNorm of fp32 [M, D]: bf16 tile image (A operand of the next GEMM; y32 also gets the fp32 rows) or fp32 rows
int launch_ln_rows(const float* x, const float* gamma, const float* beta, void* y, int M, int D, bool out_bf16,
                   cudaStream_t s, float* y32 = nullptr);

// ----------------------------------------------------------------------------- IVF retrieval (csrc/retrieval_api.cu)
// query rows x [M, d] fp32 -> the coarse search's A image [x_hi | x_lo | x_hi] ([ceil(M/128) * 128][3 d] bf16)
int launch_ivf_pack(const float* x, void* img, int M, int d, cudaStream_t s);
// gemm_tc epilogue 8 over that image and the centroid image: cand [M][N/16][nprobe] int2 {score bits, column}
int launch_ivf_coarse_tc(const void* A_img, const void* W_img, const float* cnorm, void* cand, int M, int N, int K, int nprobe,
                         cudaStream_t s);
// cursor[b] = sum_{b' < b} count[b'] over n buckets (ivf_order_kernel, one CTA)
int launch_bucket_offsets(const int* count, int* cursor, int n, cudaStream_t s);

}  // namespace svcb

// Salience-based F0 (pitch/inference.py:31-44 compute_f0_salience: libf0's salience() of pitch/core/salience.py at
// Fs=16000, N=2048, H=320, F_min=45, F_max=1760, defaults otherwise), for a ragged batch of float32 clips at 16 kHz, in
// fp64 on the device.  Before the host's np.repeat and moving average.
//
//   stft    = per CTA 8 consecutive frames of one item: the centred, zero-padded, Hann-windowed direct DFT of bins
//             0 .. 231 (the only bins whose instantaneous frequency can fall below 1760 Hz: |f - 7.8125 k| <= 25 Hz)
//   bin     = per frame one CTA: instantaneous frequency of each bin from the phase advance since the frame before
//             (salience.py:180-198; frame 0 takes frame 1's), the log-frequency bin, |X|^2 added into its bin in
//             ascending k order (np.add.at), then the np.hanning(11) smoothing along frequency and the frame's maximum
//   harm    = per frame one CTA: the item's maximum, the threshold (salience.py:246-248), the harmonic summation
//             (scipy's correlate1d at the reference's origin: Z[i] = sum_j w[j] Y[i + j - 4]), the frame's maximum of Z
//   dp      = per item one CTA, one thread per bin: the threshold of Z with the item's maximum (salience.py:269-270),
//             log(Z + eps32), and the max-plus recursion of compute_trajectory_dp over all 636 predecessors of the
//             previous column (first index of the maximum), back-pointers in the workspace, the trace back by thread 0
//
// Every stage of an item reads only that item, with a fixed thread mapping and summation order, so each item's F0 is
// bitwise that of a lone call.  oracle/salience_oracle.py restates the same algorithm in numpy.
#include <cmath>
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int SF_FS = 16000, SF_N = 2048, SF_H = 320;
constexpr double SF_FMIN = 45.0, SF_FMAX = 1760.0;
constexpr int SF_B = 636;                       // floor(120 log2(1760 / 45) + 0.5) + 1 log-frequency bins
constexpr int SF_KB = 232;                      // STFT bins computed: 7.8125 k - 25 < 1760 needs k <= 228, plus margin
constexpr int SF_FT = 8;                        // frames per STFT CTA
constexpr int SF_SPAN = SF_N + SF_H * (SF_FT - 1);   // samples those frames read
constexpr int SF_T = 256;                       // threads of the per-frame CTAs
constexpr int SF_DPT = 640;                     // threads of the DP CTA (one per bin, rounded up to warps)
constexpr int SF_SMOOTH = 11, SF_SHALF = 5;     // np.hanning(11)
constexpr int SF_NHARM = 10, SF_HWIN = 11;      // harmonics, cos^2 window taps of each
constexpr int SF_NTAPS = SF_NHARM * SF_HWIN;    // non-zero taps of the 641-tap weighting vector (the windows never overlap)
constexpr int SF_CORR_LO = 4;                   // Z[i] reads Y[i + j - 4]
constexpr int SF_CORR_HI = 399 + SF_HWIN - 1 - SF_CORR_LO;   // ... up to Y[i + 405]
constexpr int SF_GROUP = 128;                   // items per pass
constexpr int SF_MIN_SAMPLES = SF_H;            // two frames: the phase advance needs a pair
constexpr double SF_EPS32 = 1.1920928955078125e-07;   // np.finfo(np.float32).eps
constexpr double SF_TWO_PI = 6.283185307179586;       // 2 * np.pi

static_assert(SF_B <= SF_DPT && SF_KB <= SF_T, "one thread per bin");

__device__ double g_sf_win[SF_N];          // scipy.signal.get_window('hann', 2048, fftbins=True)
__device__ double2 g_sf_tw[SF_N];          // (cos, sin)(2 pi m / 2048)
__device__ double g_sf_hz[SF_B];           // 45 * 2 ** (b * 10 / 1200)
__constant__ double c_sf_smooth[SF_SMOOTH];
__constant__ double c_sf_tapw[SF_NTAPS];   // weights of the harmonic taps, j ascending
__constant__ int c_sf_tapj[SF_NTAPS];      // their positions j in the weighting vector

inline long long salience_frames(long long n) { return n / SF_H + 1; }

struct SfWs {
  double2* X;        // [frame][SF_KB] spectrum of bins 0 .. 231
  double* S;         // [frame][SF_B] smoothed Y, then Z in place
  double *ymax, *zmax;   // [frame] maxima
  int16_t* bp;       // [frame][SF_B] back-pointers
};

__device__ __forceinline__ double warp_max_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// CTA-wide max of NT threads; every thread gets it
template <int NT>
__device__ double cta_max(double v, double* red) {
  v = warp_max_d(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  double m = red[0];
  for (int i = 1; i < NT / 32; ++i) m = fmax(m, red[i]);
  return m;
}
// the maximum of an item's per-frame maxima
template <int NT>
__device__ double item_max(const double* fmax_, long long F, double* red) {
  double m = 0.0;
  for (long long i = threadIdx.x; i < F; i += NT) m = fmax(m, fmax_[i]);
  return cta_max<NT>(m, red);
}
// salience.py:246-248 with gamma = 0: kept while 20 log10(v / max + eps32) < 0; a 0 / 0 keeps nothing
__device__ __forceinline__ double sf_threshold(double v, double mx) {
  return __dadd_rn(__ddiv_rn(v, mx), SF_EPS32) < 1.0 ? v : 0.0;
}

// The spectrum of frames t0 .. t0 + 7 of one item: thread k < 232 sums bin k over the 2048 windowed samples.
__global__ void __launch_bounds__(SF_T) salience_stft_kernel(const float* __restrict__ x, ItemPass<SF_GROUP> it, SfWs w) {
  extern __shared__ double sm_stft[];
  double* xs = sm_stft;              // [SF_SPAN]
  double* win = xs + SF_SPAN;        // [SF_N]
  double2* tw = reinterpret_cast<double2*>(win + SF_N);   // [SF_N]
  const int b = blockIdx.y, tid = threadIdx.x;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, t0 = (long long)blockIdx.x * SF_FT;
  if (t0 >= F) return;
  const long long n = it.in[b + 1] - it.in[b];
  const float* xb = x + it.in[b];
  const long long s0 = t0 * SF_H - SF_N / 2;
  for (int i = tid; i < SF_SPAN; i += SF_T) {
    const long long s = s0 + i;
    xs[i] = s >= 0 && s < n ? (double)xb[s] : 0.0;
  }
  for (int i = tid; i < SF_N; i += SF_T) { win[i] = g_sf_win[i]; tw[i] = g_sf_tw[i]; }
  __syncthreads();
  const int k = tid;
  if (k >= SF_KB) return;
  double re[SF_FT], im[SF_FT];
#pragma unroll
  for (int f = 0; f < SF_FT; ++f) { re[f] = 0.0; im[f] = 0.0; }
  for (int m = 0; m < SF_N; ++m) {
    const double2 c = tw[(k * m) & (SF_N - 1)];
    const double wm = win[m];
#pragma unroll
    for (int f = 0; f < SF_FT; ++f) {
      const double v = wm * xs[f * SF_H + m];
      re[f] = fma(v, c.x, re[f]);
      im[f] = fma(-v, c.y, im[f]);
    }
  }
#pragma unroll
  for (int f = 0; f < SF_FT; ++f)
    if (t0 + f < F) w.X[(fo + t0 + f) * SF_KB + k] = make_double2(re[f], im[f]);
}

struct SfBinSmem {
  int bin[SF_KB];
  double pw[SF_KB];
  double y[SF_B + 2 * SF_SHALF];   // binned frame with 5 zeros on each side
  double red[SF_T / 32];
};

// One CTA per frame: instantaneous frequencies, the binning in ascending k order, the smoothing and the frame's max.
__global__ void __launch_bounds__(SF_T) salience_bin_kernel(ItemPass<SF_GROUP> it, SfWs w, double* __restrict__ ytap) {
  __shared__ SfBinSmem sm;
  const int b = blockIdx.y, tid = threadIdx.x;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, t = blockIdx.x;
  if (t >= F) return;
  const long long tp = t > 0 ? t : 1;   // frame 0 repeats frame 1's instantaneous frequencies
  for (int k = tid; k < SF_KB; k += SF_T) {
    const double2 a = w.X[(fo + tp) * SF_KB + k], p = w.X[(fo + tp - 1) * SF_KB + k];
    // salience.py:181-190, each operation rounded once in the reference's order
    const double omega = __ddiv_rn(__dmul_rn(SF_TWO_PI, (double)k), (double)SF_N);
    double hpi = __dsub_rn(__dsub_rn(atan2(a.y, a.x), atan2(p.y, p.x)), __dmul_rn(omega, (double)SF_H));
    hpi = __dsub_rn(hpi, __dmul_rn(SF_TWO_PI, __dsub_rn(rint(__dadd_rn(__ddiv_rn(hpi, SF_TWO_PI), 1.0)), 1.0)));
    const double f = __ddiv_rn(__dmul_rn(__dadd_rn(omega, __ddiv_rn(hpi, (double)SF_H)), (double)SF_FS), SF_TWO_PI);
    sm.bin[k] = f >= SF_FMIN && f < SF_FMAX ? (int)floor(__dadd_rn(__dmul_rn(120.0, log2(__ddiv_rn(f, SF_FMIN))), 0.5)) : -1;
    const double2 c = w.X[(fo + t) * SF_KB + k];
    const double mag = hypot(c.x, c.y);
    sm.pw[k] = __dmul_rn(mag, mag);
  }
  if (tid < 2 * SF_SHALF) sm.y[tid < SF_SHALF ? tid : SF_B + tid] = 0.0;
  __syncthreads();
  for (int i = tid; i < SF_B; i += SF_T) {
    // the STFT bins that can land in bin i: frequencies within 25 Hz of 7.8125 k, with two bins of margin
    const double lo = SF_FMIN * exp2((i - 0.5) / 120.0) - 25.0, hi = SF_FMIN * exp2((i + 0.5) / 120.0) + 25.0;
    const int k0 = max(0, (int)floor(lo / 7.8125) - 2), k1 = min(SF_KB - 1, (int)ceil(hi / 7.8125) + 2);
    double s = 0.0;
    for (int k = k0; k <= k1; ++k)
      if (sm.bin[k] == i) s = __dadd_rn(s, sm.pw[k]);
    sm.y[SF_SHALF + i] = s;
    if (ytap) ytap[SF_B * fo + (long long)i * F + t] = s;
  }
  __syncthreads();
  double mx = 0.0;
  for (int i = tid; i < SF_B; i += SF_T) {
    double s = 0.0;
#pragma unroll
    for (int j = 0; j < SF_SMOOTH; ++j) s = fma(c_sf_smooth[j], sm.y[i + j], s);
    w.S[(fo + t) * SF_B + i] = s;
    mx = fmax(mx, s);
  }
  mx = cta_max<SF_T>(mx, sm.red);
  if (tid == 0) w.ymax[fo + t] = mx;
}

struct SfHarmSmem {
  double y[SF_CORR_LO + SF_B + SF_CORR_HI];   // the thresholded frame, zero-padded for the correlation
  double red[SF_T / 32];
};

// One CTA per frame: the threshold with the item's max of the smoothed Y, the harmonic summation, the frame's max of Z.
__global__ void __launch_bounds__(SF_T) salience_harm_kernel(ItemPass<SF_GROUP> it, SfWs w) {
  __shared__ SfHarmSmem sm;
  const int b = blockIdx.y, tid = threadIdx.x;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, t = blockIdx.x;
  if (t >= F) return;
  const double ymx = item_max<SF_T>(w.ymax + fo, F, sm.red);
  double* row = w.S + (fo + t) * SF_B;
  for (int i = tid; i < SF_CORR_LO + SF_B + SF_CORR_HI; i += SF_T) {
    const int q = i - SF_CORR_LO;
    sm.y[i] = q >= 0 && q < SF_B ? sf_threshold(row[q], ymx) : 0.0;
  }
  __syncthreads();
  double mx = 0.0;
  for (int i = tid; i < SF_B; i += SF_T) {
    double s = 0.0;
    for (int q = 0; q < SF_NTAPS; ++q) s = fma(c_sf_tapw[q], sm.y[i + c_sf_tapj[q]], s);
    row[i] = s;
    mx = fmax(mx, s);
  }
  mx = cta_max<SF_T>(mx, sm.red);
  if (tid == 0) w.zmax[fo + t] = mx;
}

struct SfDpArgs {
  const double* zext;   // the DP-only entry: Z as [SF_B][F] per item; null: the workspace's, thresholded here
  double* ztap;         // [SF_B][F] per item, or null
  int32_t* path;        // [frame], or null
  double* f0;           // [frame], or null
  double tl_near, tl_far;   // log(1 + eps32), log(0.01 + eps32)
};

// One CTA per item, bin b in thread b: the max-plus recursion, first index of the maximum, then the trace back.
__global__ void __launch_bounds__(SF_DPT) salience_dp_kernel(ItemPass<SF_GROUP> it, SfWs w, SfDpArgs a) {
  __shared__ double D[2][SF_B];
  __shared__ double red[SF_DPT / 32];
  __shared__ int redi[SF_DPT / 32];
  const int it_b = blockIdx.x, b = threadIdx.x;
  const long long fo = it.out[it_b], F = it.out[it_b + 1] - fo;
  const bool act = b < SF_B;
  const double zmx = a.zext ? 0.0 : item_max<SF_DPT>(w.zmax + fo, F, red);
  auto zlog = [&](long long n) {
    double z;
    if (a.zext) {
      z = a.zext[SF_B * it.in[it_b] + (long long)b * F + n];   // the given Z sits at the caller's own offsets
    } else {
      z = sf_threshold(w.S[(fo + n) * SF_B + b], zmx);
      if (a.ztap) a.ztap[SF_B * fo + (long long)b * F + n] = z;
    }
    return log(__dadd_rn(z, SF_EPS32));
  };
  if (act) D[0][b] = zlog(0);
  for (long long n = 1; n < F; ++n) {
    const double* Dp = D[(n - 1) & 1];
    __syncthreads();
    if (act) {
      const double zl = zlog(n);
      double best = -INFINITY;
      int arg = 0;
      const int lo = max(0, b - 5), hi = min(SF_B - 1, b + 5);
      for (int q = 0; q < lo; ++q) {
        const double s = __dadd_rn(a.tl_far, Dp[q]);
        if (s > best) { best = s; arg = q; }
      }
      for (int q = lo; q <= hi; ++q) {
        const double s = __dadd_rn(a.tl_near, Dp[q]);
        if (s > best) { best = s; arg = q; }
      }
      for (int q = hi + 1; q < SF_B; ++q) {
        const double s = __dadd_rn(a.tl_far, Dp[q]);
        if (s > best) { best = s; arg = q; }
      }
      D[n & 1][b] = __dadd_rn(best, zl);
      w.bp[(fo + n - 1) * SF_B + b] = (int16_t)arg;
    }
  }
  __syncthreads();
  // the first argmax of the last column: (value, index) with ties to the smaller index
  double v = act ? D[(F - 1) & 1][b] : -INFINITY;
  int vi = act ? b : SF_B;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, vi, o);
    if (ov > v || (ov == v && oi < vi)) { v = ov; vi = oi; }
  }
  if ((b & 31) == 0) { red[b >> 5] = v; redi[b >> 5] = vi; }
  __syncthreads();   // also publishes every thread's back-pointers to thread 0
  if (b != 0) return;
  double bv = red[0];
  int e = redi[0];
  for (int i = 1; i < SF_DPT / 32; ++i)
    if (red[i] > bv || (red[i] == bv && redi[i] < e)) { bv = red[i]; e = redi[i]; }
  for (long long n = F - 1; n >= 0; --n) {
    if (a.path) a.path[fo + n] = e;
    if (a.f0) a.f0[fo + n] = g_sf_hz[e];
    if (n > 0) e = w.bp[(fo + n - 1) * SF_B + e];
  }
}

// Host tables, each computed as numpy / scipy compute them.
struct SfTables {
  double win[SF_N], hz[SF_B], smooth[SF_SMOOTH], tapw[SF_NTAPS];
  double2 tw[SF_N];
  int tapj[SF_NTAPS];
  SfTables() {
    const double pi = 3.141592653589793;
    // get_window('hann', 2048, fftbins=True) = 0.5 + 0.5 cos(linspace(-pi, pi, 2049)[m])
    const double step = 2.0 * pi / SF_N;
    for (int m = 0; m < SF_N; ++m) {
      win[m] = 0.5 + 0.5 * std::cos(-pi + m * step);
      tw[m] = make_double2(std::cos(2.0 * pi * m / SF_N), std::sin(2.0 * pi * m / SF_N));
    }
    for (int b = 0; b < SF_B; ++b) hz[b] = SF_FMIN * std::pow(2.0, (b * 10.0) / 1200.0);
    for (int j = 0; j < SF_SMOOTH; ++j) smooth[j] = 0.5 + 0.5 * std::cos(pi * (2 * j - (SF_SMOOTH - 1)) / (SF_SMOOTH - 1));
    // the weighting vector: cos^2(linspace(-1, 1, 11) pi / 2) * 0.9 ** idx at round(120 log2 h)
    for (int idx = 0; idx < SF_NHARM; ++idx) {
      const int h = (int)std::lround(std::log2((double)(idx + 1)) * 120.0);
      for (int m = 0; m < SF_HWIN; ++m) {
        const double c = std::cos((-1.0 + m * 0.2) * pi / 2.0);
        tapw[idx * SF_HWIN + m] = c * c * std::pow(0.9, idx);
        tapj[idx * SF_HWIN + m] = h + m;
      }
    }
  }
};

// the tables belong to a device: upload them once per device
int salience_upload_tables() {
  static const SfTables tab;
  static std::atomic<bool> done[kMaxDevices];
  int dev = 0;
  SVCB_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 0 && dev < kMaxDevices && done[dev].load()) return SVCB_OK;
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(g_sf_win, tab.win, sizeof(tab.win)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(g_sf_tw, tab.tw, sizeof(tab.tw)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(g_sf_hz, tab.hz, sizeof(tab.hz)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_sf_smooth, tab.smooth, sizeof(tab.smooth)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_sf_tapw, tab.tapw, sizeof(tab.tapw)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_sf_tapj, tab.tapj, sizeof(tab.tapj)));
  if (dev >= 0 && dev < kMaxDevices) done[dev].store(true);
  return SVCB_OK;
}

// workspace regions, in the order the entry point carves them; Ft bounds the frames of the batch
struct SfPlan {
  size_t X, S, ymax, zmax, bp, bytes;
  explicit SfPlan(long long Ft, bool dp_only = false) {
    WsPlan p;
    X = p.take(dp_only ? 0 : 16 * (size_t)SF_KB * (size_t)Ft);
    S = p.take(dp_only ? 0 : 8 * (size_t)SF_B * (size_t)Ft);
    ymax = p.take(dp_only ? 0 : 8 * (size_t)Ft);
    zmax = p.take(dp_only ? 0 : 8 * (size_t)Ft);
    bp = p.take(2 * (size_t)SF_B * (size_t)Ft);
    bytes = p.off;
  }
  SfWs carve(void* ws) const {
    char* base = static_cast<char*>(ws);
    SfWs w;
    w.X = reinterpret_cast<double2*>(base + X);
    w.S = reinterpret_cast<double*>(base + S);
    w.ymax = reinterpret_cast<double*>(base + ymax);
    w.zmax = reinterpret_cast<double*>(base + zmax);
    w.bp = reinterpret_cast<int16_t*>(base + bp);
    return w;
  }
};

DevSmemCache g_sf_stft_smem;
constexpr size_t SF_STFT_SMEM = 8 * (size_t)(SF_SPAN + SF_N) + 16 * (size_t)SF_N;

SfDpArgs dp_args() {
  SfDpArgs a{};
  a.tl_near = std::log(1.0 + SF_EPS32);
  a.tl_far = std::log(0.01 + SF_EPS32);
  return a;
}

int launch_salience_dp(const ItemPass<SF_GROUP>& it, const SfWs& w, const SfDpArgs& a, cudaStream_t s) {
  const double frames = (double)(it.out[it.n] - it.out[0]);
  KernelScope ks("salience_dp", s, 2.0 * SF_B * SF_B * frames, (8.0 + 2.0) * SF_B * frames);
  salience_dp_kernel<<<(unsigned)it.n, SF_DPT, 0, s>>>(it, w, a);
  SVCB_LAUNCH_CHECK("salience_dp");
  return SVCB_OK;
}

}  // namespace svcb

using namespace svcb;

extern "C" {

size_t svcb_salience_f0_workspace_bytes(int64_t total_samples, int32_t B) {
  if (total_samples < 0 || B < 1) return 0;
  return SfPlan(total_samples / SF_H + B).bytes;
}

int svcb_salience_f0_ragged(const float* x, const int64_t* offsets_host, int32_t B, double* f0, double* y_tap,
                            double* z_tap, int32_t* path_tap, void* ws, size_t ws_bytes, svcb_stream stream) {
  static const char* who = "svcb_salience_f0_ragged";
  if (!x || !f0 || !offsets_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, offsets_host, B, 1, SF_MIN_SAMPLES, "samples", "shorter than one 320-sample hop"));
  const long long N = offsets_host[B] - offsets_host[0];
  const SfPlan plan(N / SF_H + B);
  SVCB_TRY(check_workspace(ws, ws_bytes, plan.bytes, who));
  SVCB_TRY(salience_upload_tables());
  SVCB_CUDA_CHECK(ensure_dyn_smem(salience_stft_kernel, SF_STFT_SMEM, g_sf_stft_smem));
  const SfWs w = plan.carve(ws);
  SfDpArgs a = dp_args();
  a.ztap = z_tap;
  a.path = path_tap;
  a.f0 = f0;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return for_each_pass<SF_GROUP>(offsets_host, B, [](long long n) { return salience_frames(n); },
                                 [&](const ItemPass<SF_GROUP>& it, int) -> int {
    long long fmax = 0;
    for (int i = 0; i < it.n; ++i) fmax = std::max(fmax, it.out[i + 1] - it.out[i]);
    const double frames = (double)(it.out[it.n] - it.out[0]);
    const unsigned items = (unsigned)it.n;
    {
      KernelScope ks("salience_stft", s, 4.0 * SF_N * SF_KB * frames, 16.0 * SF_KB * frames);
      salience_stft_kernel<<<dim3((unsigned)((fmax + SF_FT - 1) / SF_FT), items), SF_T, SF_STFT_SMEM, s>>>(x, it, w);
      SVCB_LAUNCH_CHECK("salience_stft");
    }
    {
      KernelScope ks("salience_bin", s, 0.0, (2.0 * 16.0 * SF_KB + 8.0 * SF_B) * frames);
      salience_bin_kernel<<<dim3((unsigned)fmax, items), SF_T, 0, s>>>(it, w, y_tap);
      SVCB_LAUNCH_CHECK("salience_bin");
    }
    {
      KernelScope ks("salience_harm", s, 2.0 * SF_NTAPS * SF_B * frames, 16.0 * SF_B * frames);
      salience_harm_kernel<<<dim3((unsigned)fmax, items), SF_T, 0, s>>>(it, w);
      SVCB_LAUNCH_CHECK("salience_harm");
    }
    return launch_salience_dp(it, w, a, s);
  });
}

size_t svcb_salience_dp_workspace_bytes(int64_t total_frames) {
  if (total_frames < 0) return 0;
  return SfPlan(total_frames, true).bytes;
}

int svcb_salience_dp_ragged(const double* z, const int64_t* frame_offsets_host, int32_t B, int32_t* path, void* ws,
                            size_t ws_bytes, svcb_stream stream) {
  static const char* who = "svcb_salience_dp_ragged";
  if (!z || !path || !frame_offsets_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, frame_offsets_host, B, 1, 1, "frames", nullptr));
  const SfPlan plan(frame_offsets_host[B] - frame_offsets_host[0], true);
  SVCB_TRY(check_workspace(ws, ws_bytes, plan.bytes, who));
  SVCB_TRY(salience_upload_tables());
  const SfWs w = plan.carve(ws);
  SfDpArgs a = dp_args();
  a.zext = z;
  a.path = path;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return for_each_pass<SF_GROUP>(frame_offsets_host, B, [](long long n) { return n; },
                                 [&](const ItemPass<SF_GROUP>& it, int) -> int { return launch_salience_dp(it, w, a, s); });
}

}  // extern "C"

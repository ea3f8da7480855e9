// Praat's autocorrelation pitch (prepare/preprocess_f0_mouth.py:11-22: parselmouth.Sound(x, 16000).to_pitch_ac(
// time_step=0.01, voicing_threshold=0.5, pitch_floor=30, pitch_ceiling=1000).selected_array['frequency'], before the
// np.pad) for a ragged batch of float64 clips at 16 kHz, in fp64 on the device.
//
//   peak       = per item, max |x - mean(x)| (the global peak)
//   frame      = per frame one CTA: the frame's centre on Praat's centred grid, the local mean over one longest period
//                either side, the local peak, the Hanning-windowed frame in shared memory, its direct autocorrelation
//                at lags 0 .. 607, Boersma's eq. (9) division by the window's own normalised autocorrelation; then in
//                the first warp the local maxima, their parabolic + windowed-sinc refinement (Newton on the
//                interpolant, depth 70), strengths, and the 14 strongest kept in lag order after the unvoiced one
//   viterbi    = per item one warp (candidates in lanes), sequential over the frames, back-pointers in the workspace,
//                then the trace back by lane 0
//
// Every stage of an item reads only that item, with a fixed thread mapping and summation order, so each item's F0 is
// bitwise that of a lone call.  oracle/praat_f0_oracle.py restates the same algorithm in numpy and documents each rule.
#include <cmath>
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int PR_FS = 16000;
constexpr double PR_DX = 1.0 / PR_FS, PR_DT = 0.01, PR_WIN_DUR = 0.1;
constexpr double PR_FLOOR = 30.0, PR_SILENCE = 0.03, PR_VOICING = 0.5;
constexpr double PR_OCTAVE = 0.01, PR_OCTAVE_JUMP = 0.35, PR_VUV = 0.14;
constexpr int PR_W = 1600, PR_HALF = 800;      // window samples: 3 periods of 30 Hz
constexpr int PR_P = 533;                      // one longest period: the local mean runs over 2 P samples
constexpr int PR_MINLAG = 16, PR_MAXLAG = 535; // max(2, floor(fs / 1000)), floor(W / 3) + 2
constexpr int PR_DEPTH = 70;                   // sinc interpolation depth
constexpr int PR_NLAG = PR_MAXLAG + PR_DEPTH + 2;   // lags 0 .. 606 are read
constexpr int PR_LG = 8;                       // lags per thread of the autocorrelation
constexpr int PR_NGRP = (PR_NLAG + PR_LG - 1) / PR_LG;   // 76 lag groups (608 lags)
constexpr int PR_SLICES = 3;                   // the j range of a lag group is cut into 3 slices
constexpr int PR_NCAND = 15;                   // the unvoiced candidate + 14 voiced
constexpr int PR_MAXMAX = (PR_MAXLAG - PR_MINLAG) / 2 + 2;   // local maxima a frame can have
constexpr int PR_GROUP = 128;                  // items per pass
constexpr int PR_T = 256;                      // threads of the peak and frame CTAs
constexpr int PR_VW = 4;                       // Viterbi: items (warps) per CTA
constexpr int PR_NEWTON = 8;
constexpr int PR_MIN_SAMPLES = 1600;           // duration >= the 0.1 s window: one frame

static_assert(PR_NGRP * PR_SLICES <= PR_T, "one autocorrelation unit per thread");

__device__ double g_hann[PR_W];
__device__ double g_rwn[PR_NLAG];

// Frames of n samples (the oracle's n_frames): floor((n dx - 0.1) / 0.01) + 1, each operation rounded once.
inline long long praat_frames(long long n) {
  const double dur = (double)n * PR_DX;
  if (dur < PR_WIN_DUR) return 0;
  return std::max(0ll, (long long)std::floor((dur - PR_WIN_DUR) / PR_DT) + 1);
}

struct PrWs {
  double *gpeak, *cf, *cs;
  int* cnt;
  uint8_t* bp;
  int g0;   // the pass's first item
};

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// CTA-wide reduction in a fixed order (lanes by butterfly, then warps 0 .. 7); every thread gets the result
template <bool MAX>
__device__ double cta_reduce(double v, double* red) {
  const int tid = threadIdx.x;
  v = MAX ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if ((tid & 31) == 0) red[tid >> 5] = v;
  __syncthreads();
  double t = red[0];
  for (int i = 1; i < PR_T / 32; ++i) t = MAX ? fmax(t, red[i]) : t + red[i];
  return t;
}

// the global peak: max |x - mean| over the item
__global__ void __launch_bounds__(PR_T) praat_peak_kernel(const double* __restrict__ x, ItemPass<PR_GROUP> it, PrWs w) {
  __shared__ double red[PR_T / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const double* xb = x + it.in[b];
  const long long n = it.in[b + 1] - it.in[b];
  double s = 0.0;
  for (long long i = tid; i < n; i += PR_T) s += xb[i];
  const double mean = cta_reduce<false>(s, red) / (double)n;
  double m = 0.0;
  for (long long i = tid; i < n; i += PR_T) m = fmax(m, fabs(xb[i] - mean));
  m = cta_reduce<true>(m, red);
  if (tid == 0) w.gpeak[w.g0 + b] = m;
}

// g, g', g'' of the windowed sinc at d = u - q (sp, cp = sin, cos of pi u; sign = (-1)^q)
__device__ __forceinline__ void praat_g(double d, double sp, double cp, double sign, double& g, double& g1, double& g2) {
  const double pi = M_PI, bw = M_PI / (PR_DEPTH + 0.5);
  double s, s1, s2;
  if (fabs(d) < 1e-3) {
    const double p2 = (pi * d) * (pi * d);
    s = 1.0 - p2 / 6.0 + p2 * p2 / 120.0;
    s1 = -pi * pi * d / 3.0 + pi * pi * pi * pi * d * d * d / 30.0;
    s2 = -pi * pi / 3.0 + pi * pi * pi * pi * d * d / 10.0;
  } else {
    s = sign * sp / (pi * d);
    s1 = (sign * cp - s) / d;
    s2 = -pi * pi * s - 2.0 * s1 / d;
  }
  double sn, c;
  sincos(bw * d, &sn, &c);
  const double wv = 0.5 + 0.5 * c, w1 = -0.5 * bw * sn, w2 = -0.5 * bw * bw * c;
  g = s * wv;
  g1 = s1 * wv + s * w1;
  g2 = s2 * wv + 2.0 * s1 * w1 + s * w2;
}

// the sinc interpolant of r (lags 0 .. PR_NLAG - 1, mirrored below 0) and its derivatives at lag t
__device__ void praat_interp(const double* r, double t, double& f, double& f1, double& f2) {
  const double m = floor(t), u = t - m;
  const int mi = (int)m;
  double sp, cp;
  sincospi(u, &sp, &cp);
  f = f1 = f2 = 0.0;
  for (int q = -PR_DEPTH + 1; q <= PR_DEPTH; ++q) {
    double g, g1, g2;
    praat_g(u - (double)q, sp, cp, (q & 1) ? -1.0 : 1.0, g, g1, g2);
    const double v = r[abs(mi + q)];
    f += v * g;
    f1 += v * g1;
    f2 += v * g2;
  }
}

// the lag and interpolated r of the maximum near the local maximum at lag k (the oracle's refine)
__device__ void praat_refine(const double* r, int k, double& t_out, double& v_out) {
  const double a = r[k - 1], b = r[k], c = r[k + 1];
  const double den = a - 2.0 * b + c;
  double t = den < 0.0 ? (double)k + 0.5 * (a - c) / den : (double)k;
  if (!(t >= k - 1 && t <= k + 1)) t = (double)k;
  double f, f1, f2;
  for (int s = 0; s < PR_NEWTON; ++s) {
    praat_interp(r, t, f, f1, f2);
    if (!(f2 < 0.0)) break;
    const double step = f1 / f2, tn = t - step;
    if (!(tn >= k - 1 && tn <= k + 1)) break;
    t = tn;
    if (fabs(step) < 1e-10) break;
  }
  praat_interp(r, t, f, f1, f2);
  t_out = t;
  v_out = f;
}

struct PrFrameSmem {
  double a[PR_W + 2 * PR_LG];                 // the windowed frame, zero past W
  double part[PR_SLICES][PR_NGRP * PR_LG];    // autocorrelation partial sums per slice
  double r[PR_NGRP * PR_LG];                  // normalised autocorrelation
  double ct[PR_MAXMAX], cv[PR_MAXMAX];        // refined lag and strength of each local maximum
  int lag[PR_MAXMAX];
  double red[PR_T / 32];
};

// One CTA per frame: the autocorrelation and the candidates.
__global__ void __launch_bounds__(PR_T) praat_frame_kernel(const double* __restrict__ x, ItemPass<PR_GROUP> it, PrWs w) {
  __shared__ PrFrameSmem sm;
  const int b = blockIdx.y, tid = threadIdx.x, lane = tid & 31;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, i = blockIdx.x;
  if (i >= F) return;
  const long long n = it.in[b + 1] - it.in[b];
  const double* xb = x + it.in[b];
  // the frame's centre and its sample `left`, each operation rounded once as in the oracle
  const double dur = __dmul_rn((double)n, PR_DX);
  const double t0 = __dadd_rn(__dsub_rn(__dmul_rn(0.5, dur), __dmul_rn(__dmul_rn(0.5, (double)F), PR_DT)), __dmul_rn(0.5, PR_DT));
  const double tc = __dadd_rn(t0, __dmul_rn((double)i, PR_DT));
  long long left = (long long)floor(__dsub_rn(tc, __dmul_rn(0.5, PR_DX)) / PR_DX);
  left = min(max(left, (long long)PR_HALF - 1), n - 1 - PR_HALF);   // a no-op: the frames fit the signal
  // local mean over samples left - 532 .. left + 533
  double s = 0.0;
  for (int k = tid; k < 2 * PR_P; k += PR_T) s += xb[left - PR_P + 1 + k];
  const double lm = cta_reduce<false>(s, sm.red) / (double)(2 * PR_P);
  const double* xs = xb + left - PR_HALF + 1;
  double lp = 0.0;
  for (int j = tid; j < PR_W; j += PR_T) {
    const double d = xs[j] - lm;
    lp = fmax(lp, fabs(d));
    sm.a[j] = d * g_hann[j];
  }
  if (tid < 2 * PR_LG) sm.a[PR_W + tid] = 0.0;
  lp = cta_reduce<true>(lp, sm.red);   // its barriers also publish sm.a
  // autocorrelation: unit tid = (slice, lag group); lags k0 .. k0 + 7, j over its slice of [0, W - k0) in steps of 8
  if (tid < PR_NGRP * PR_SLICES) {
    const int grp = tid % PR_NGRP, sl = tid / PR_NGRP, k0 = grp * PR_LG;
    const int nb = (PR_W - k0) / PR_LG, jb = sl * nb / PR_SLICES * PR_LG, je = (sl + 1) * nb / PR_SLICES * PR_LG;
    double acc[PR_LG], win[2 * PR_LG];
#pragma unroll
    for (int l = 0; l < PR_LG; ++l) { acc[l] = 0.0; win[l] = sm.a[jb + k0 + l]; }
    for (int j = jb; j < je; j += PR_LG) {
#pragma unroll
      for (int l = 0; l < PR_LG; ++l) win[PR_LG + l] = sm.a[j + k0 + PR_LG + l];
#pragma unroll
      for (int jj = 0; jj < PR_LG; ++jj) {
        const double aj = sm.a[j + jj];
#pragma unroll
        for (int l = 0; l < PR_LG; ++l) acc[l] = fma(aj, win[jj + l], acc[l]);
      }
#pragma unroll
      for (int l = 0; l < PR_LG; ++l) win[l] = win[PR_LG + l];
    }
#pragma unroll
    for (int l = 0; l < PR_LG; ++l) sm.part[sl][k0 + l] = acc[l];
  }
  __syncthreads();
  const double ra0 = (sm.part[0][0] + sm.part[1][0]) + sm.part[2][0];
  for (int k = tid; k < PR_NLAG; k += PR_T) {
    const double ra = (sm.part[0][k] + sm.part[1][k]) + sm.part[2][k];
    sm.r[k] = ra0 == 0.0 ? 0.0 : (ra / ra0) / g_rwn[k];
  }
  __syncthreads();
  if (tid >= 32) return;
  // candidates, in the first warp
  const double gp = w.gpeak[w.g0 + b];
  const double ratio = gp > 0.0 ? lp / gp : 0.0;
  const double unv = PR_VOICING + fmax(0.0, 2.0 - ratio / (PR_SILENCE / (1.0 + PR_VOICING)));
  int nc = 0;
  if (ra0 != 0.0) {
    const double thr = 0.5 * PR_VOICING;
    for (int k0 = PR_MINLAG; k0 <= PR_MAXLAG; k0 += 32) {
      const int k = k0 + lane;
      const bool is = k <= PR_MAXLAG && sm.r[k] > thr && sm.r[k] > sm.r[k - 1] && sm.r[k] >= sm.r[k + 1];
      const unsigned m = __ballot_sync(0xffffffffu, is);
      if (is) sm.lag[nc + __popc(m & ((1u << lane) - 1))] = k;
      nc += __popc(m);
    }
    __syncwarp();
    for (int c = lane; c < nc; c += 32) {
      double t, v;
      praat_refine(sm.r, sm.lag[c], t, v);
      sm.ct[c] = t;
      sm.cv[c] = v - PR_OCTAVE * log2(PR_FLOOR * t / PR_FS);
    }
    __syncwarp();
  }
  // keep the 14 strongest (a tie to the smaller lag), in lag order, after the unvoiced candidate
  const long long row = (fo + i) * PR_NCAND;
  int kept = 0;
  for (int c0 = 0; c0 < nc; c0 += 32) {
    const int c = c0 + lane;
    bool keep = c < nc;
    if (keep && nc > PR_NCAND - 1) {
      int rank = 0;
      for (int o = 0; o < nc; ++o) rank += sm.cv[o] > sm.cv[c] || (sm.cv[o] == sm.cv[c] && o < c);
      keep = rank < PR_NCAND - 1;
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int q = 1 + kept + __popc(m & ((1u << lane) - 1));
      w.cf[row + q] = PR_FS / sm.ct[c];
      w.cs[row + q] = sm.cv[c];
    }
    kept += __popc(m);
  }
  if (lane == 0) {
    w.cf[row] = 0.0;
    w.cs[row] = unv;
    w.cnt[fo + i] = 1 + kept;
  }
}

__device__ __forceinline__ double praat_transition(double f1, double f2) {
  if (f1 == 0.0 && f2 == 0.0) return 0.0;
  if (f1 == 0.0 || f2 == 0.0) return PR_VUV * (0.01 / PR_DT);
  return PR_OCTAVE_JUMP * fabs(log2(f1 / f2)) * (0.01 / PR_DT);
}

// The path finder: one warp per item, candidate c in lane c, frames in order; ties to the lowest candidate index.
__global__ void __launch_bounds__(32 * PR_VW) praat_viterbi_kernel(double* __restrict__ out, ItemPass<PR_GROUP> it, PrWs w) {
  const int b = blockIdx.x * PR_VW + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= it.n) return;
  const long long fo = it.out[b], F = it.out[b + 1] - fo;
  int n = w.cnt[fo];
  double fc = lane < n ? w.cf[fo * PR_NCAND + lane] : 0.0;
  double delta = lane < n ? w.cs[fo * PR_NCAND + lane] : -INFINITY;
  for (long long i = 1; i < F; ++i) {
    const int np = n;
    const double fp = fc, dp = delta;
    n = w.cnt[fo + i];
    const long long row = (fo + i) * PR_NCAND;
    fc = lane < n ? w.cf[row + lane] : 0.0;
    double best = -INFINITY;
    int arg = 0;
    for (int p = 0; p < np; ++p) {
      const double v = __shfl_sync(0xffffffffu, dp, p) - praat_transition(__shfl_sync(0xffffffffu, fp, p), fc);
      if (v > best) { best = v; arg = p; }
    }
    if (lane < n) {
      delta = best + w.cs[row + lane];
      w.bp[row + lane] = (uint8_t)arg;
    } else {
      delta = -INFINITY;
    }
  }
  // the last frame's best candidate, then the trace back by lane 0
  double best = -INFINITY;
  int c = 0;
  for (int q = 0; q < n; ++q) {
    const double v = __shfl_sync(0xffffffffu, delta, q);
    if (v > best) { best = v; c = q; }
  }
  __syncwarp();   // every lane's back-pointers are visible to lane 0
  if (lane != 0) return;
  for (long long i = F - 1; i >= 0; --i) {
    const long long row = (fo + i) * PR_NCAND;
    out[fo + i] = w.cf[row + c];
    if (i > 0) c = w.bp[row + c];
  }
}

// Host copies of the Hanning window and of its normalised autocorrelation (the oracle's hanning, window_r).
struct PrTables {
  double hann[PR_W], rwn[PR_NLAG];
  PrTables() {
    const double pi = 3.1415926535897932384626433832795;
    for (int j = 0; j < PR_W; ++j) hann[j] = 0.5 - 0.5 * std::cos(2.0 * pi * (j + 1.0) / (PR_W + 1.0));
    double rw0 = 0.0;
    for (int k = 0; k < PR_NLAG; ++k) {
      double s = 0.0;
      for (int j = 0; j + k < PR_W; ++j) s += hann[j] * hann[j + k];
      if (k == 0) rw0 = s;
      rwn[k] = s / rw0;
    }
  }
};

// the tables belong to a device: upload them once per device
int praat_upload_tables() {
  static const PrTables tab;
  static std::atomic<bool> done[kMaxDevices];
  int dev = 0;
  SVCB_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 0 && dev < kMaxDevices && done[dev].load()) return SVCB_OK;
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(g_hann, tab.hann, sizeof(tab.hann)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(g_rwn, tab.rwn, sizeof(tab.rwn)));
  if (dev >= 0 && dev < kMaxDevices) done[dev].store(true);
  return SVCB_OK;
}

// workspace regions, in the order the entry point carves them; frames in all <= total samples / 160
struct PrPlan {
  size_t gpeak, cf, cs, cnt, bp, bytes;
  PrPlan(long long N, int B) {
    const long long Ft = N / 160 + B;
    WsPlan p;
    gpeak = p.take(8 * (size_t)B);
    cf = p.take(8 * (size_t)PR_NCAND * (size_t)Ft);
    cs = p.take(8 * (size_t)PR_NCAND * (size_t)Ft);
    cnt = p.take(4 * (size_t)Ft);
    bp = p.take((size_t)PR_NCAND * (size_t)Ft);
    bytes = p.off;
  }
};

}  // namespace svcb

using namespace svcb;

extern "C" {

size_t svcb_praat_f0_workspace_bytes(int64_t total_samples, int32_t B) {
  if (total_samples < 0 || B < 1) return 0;
  return PrPlan(total_samples, B).bytes;
}

int svcb_praat_f0_ragged(const double* x, const int64_t* offsets_host, int32_t B, double* out, void* ws, size_t ws_bytes,
                         svcb_stream stream) {
  static const char* who = "svcb_praat_f0_ragged";
  if (!x || !out || !offsets_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, offsets_host, B, 1, PR_MIN_SAMPLES, "samples", "shorter than the 0.1 s analysis window"));
  const long long N = offsets_host[B] - offsets_host[0];
  const PrPlan plan(N, B);
  SVCB_TRY(check_workspace(ws, ws_bytes, plan.bytes, who));
  SVCB_TRY(praat_upload_tables());
  char* base = static_cast<char*>(ws);
  PrWs w;
  w.gpeak = reinterpret_cast<double*>(base + plan.gpeak);
  w.cf = reinterpret_cast<double*>(base + plan.cf);
  w.cs = reinterpret_cast<double*>(base + plan.cs);
  w.cnt = reinterpret_cast<int*>(base + plan.cnt);
  w.bp = reinterpret_cast<uint8_t*>(base + plan.bp);
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return for_each_pass<PR_GROUP>(offsets_host, B, [](long long n) { return praat_frames(n); },
                                 [&](const ItemPass<PR_GROUP>& it, int g0) -> int {
    w.g0 = g0;
    long long fmax = 0, samples = it.in[it.n] - it.in[0], frames = it.out[it.n] - it.out[0];
    for (int i = 0; i < it.n; ++i) fmax = std::max(fmax, it.out[i + 1] - it.out[i]);
    const unsigned items = (unsigned)it.n;
    {
      KernelScope ks("praat_peak", s, 0.0, 16.0 * samples);
      praat_peak_kernel<<<items, PR_T, 0, s>>>(x, it, w);
      SVCB_LAUNCH_CHECK("praat_peak");
    }
    {
      // the autocorrelation's products over the lags it reads, as the direct sum needs them (not the zero padding)
      const double acf = (double)PR_NLAG * PR_W - (double)PR_NLAG * (PR_NLAG - 1) / 2.0;
      KernelScope ks("praat_frame", s, 2.0 * acf * frames, 8.0 * (PR_W + 2.0 * PR_NCAND) * frames);
      praat_frame_kernel<<<dim3((unsigned)fmax, items), PR_T, 0, s>>>(x, it, w);
      SVCB_LAUNCH_CHECK("praat_frame");
    }
    {
      KernelScope ks("praat_viterbi", s, 0.0, (16.0 + 1.0) * PR_NCAND * frames);
      praat_viterbi_kernel<<<(items + PR_VW - 1) / PR_VW, 32 * PR_VW, 0, s>>>(out, it, w);
      SVCB_LAUNCH_CHECK("praat_viterbi");
    }
    return SVCB_OK;
  });
}

}  // extern "C"

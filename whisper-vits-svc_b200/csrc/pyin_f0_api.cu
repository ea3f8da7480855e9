// pYIN F0 (libf0's pyin() of pitch/core/pyin.py at Fs=16000, N=2048, H=160, F_min=50, F_max=1000, defaults otherwise;
// the wrapper pyin_f0.compute_f0_pyin is this project's, no reference command calls pyin), for a ragged batch of
// float32 clips at 16 kHz, in fp64 on the device.
//
//   cmndf  = per CTA 8 consecutive frames of one item, one warp per frame: the difference function of lags 1 .. 320 as
//            the direct sum of (x_j - x_{j+tau})^2, each square rounded and added in ascending j (lane l holds lags
//            l + 1 + 32 k); the iterative mean, the CMNDF and the frame's RMS by lane 0, in the reference's order
//   thresh = one warp per frame: the strict local minima, their parabolic interpolation written back (including the
//            reference's handling of the minima at 16 and 319, see below), the 99 thresholds' lags, values and bins,
//            the observation column and its normalisation, the column's maximum
//   viterbi = per item one CTA: the dense Viterbi of viterbi_log_likelihood, restated exactly on each column's
//            predecessors with A > 0 plus one more: every other predecessor k scores log(tiny) + D[k], so the best of
//            them is the first k whose rounded score equals log(tiny) + max D; uint16 back-pointers in the workspace;
//            the trace back
//   tail   = one thread per frame: f0 of the path, f0[0] = 0, RMS < 0.01 -> 0, conf, refine_estimates_yin
//
// Every stage of an item reads only that item, with a fixed thread mapping and summation order, so each item's result
// is bitwise that of a lone call.  oracle/pyin_oracle.py restates the same algorithm in numpy.
#include <cmath>
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int PY_N = 2048, PY_H = 160;
constexpr int PY_B = 518;                       // int(log2(1000 / 50) * 120) pitch bins
constexpr int PY_S = 2 * PY_B;                  // HMM states: voiced bins, then unvoiced
constexpr int PY_PMIN = 16, PY_PMAX = 320;      // ceil(16000 / 1000), ceil(16000 / 50)
constexpr int PY_LAGS = PY_PMAX + 1;            // CMNDF values per frame
constexpr int PY_NTHR = 99;                     // np.arange(0.01, 1, 0.01)
constexpr int PY_BAND = 12;                     // predecessors with A > 0 per column, at most
constexpr int PY_LPL = PY_PMAX / 32;            // lags per lane of the difference function
constexpr int PY_FT = 8;                        // frames per CMNDF CTA (one warp each)
constexpr int PY_SPAN = PY_N + PY_H * (PY_FT - 1);   // samples those frames read
constexpr int PY_TW = 4;                        // frames (warps) per thresholding CTA
constexpr int PY_VT = 384;                      // threads of the Viterbi CTA
constexpr int PY_VS = (PY_S + PY_VT - 1) / PY_VT;    // states per Viterbi thread
constexpr int PY_GROUP = 128;                   // items per pass
constexpr double PY_EPS = 2.220446049250313e-16;      // np.finfo(np.float64).eps
constexpr double PY_TINY = 2.2250738585072014e-308;   // np.finfo(0.).tiny
constexpr double PY_FS = 16000.0;

static_assert(PY_LPL * 32 == PY_PMAX, "lags 1 .. 320 over 32 lanes");
static_assert(PY_VS * PY_VT >= PY_S && PY_S <= 65535, "states per thread, uint16 back-pointers");

// The host tables (svcb.h SVCB_PYIN_TAB_*): thresholds, Beta weights, F_axis, each column's predecessors (as exact
// doubles, -1 past the end) and their log(A + tiny); and log(1 / 1036 + tiny), log(tiny).
struct PyTab {
  const double* thr;
  const double* beta;
  const double* fax;
  const double* bidx;   // [PY_S][PY_BAND]
  const double* blog;   // [PY_S][PY_BAND]
  double log_init, log_tiny;
};

struct PyWs {
  double* cmndf;   // [frame][PY_LAGS]
  double* rms;     // [frame]
  double* obs;     // [frame][PY_S]
  double* omax;    // [frame]
  double* lag;     // [frame][PY_NTHR] the thresholds' float lags
  double* val;     // [frame][PY_NTHR] and their CMNDF values
  int32_t* path;   // [frame]
  uint16_t* bp;    // [frame][PY_S] back-pointers
};

inline long long pyin_frames(long long n) { return n / PY_H + 1; }

// The CMNDF and RMS of frames t0 .. t0 + 7 of one item; warp w takes frame t0 + w.
__global__ void __launch_bounds__(PY_FT * 32) pyin_cmndf_kernel(const float* __restrict__ x, ItemPass<PY_GROUP> it,
                                                                PyWs w, double* __restrict__ ctap) {
  extern __shared__ double sm_py[];
  double* xs = sm_py;                  // [PY_SPAN]
  double* dsm = xs + PY_SPAN;          // [PY_FT][PY_LAGS]
  const int b = blockIdx.y, tid = threadIdx.x, wp = tid >> 5, lane = tid & 31;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, t0 = (long long)blockIdx.x * PY_FT;
  if (t0 >= F) return;
  const long long n = it.in[b + 1] - it.in[b];
  const float* xb = x + it.in[b];
  const long long s0 = t0 * PY_H - PY_N / 2;
  for (int i = tid; i < PY_SPAN; i += PY_FT * 32) {
    const long long s = s0 + i;
    xs[i] = s >= 0 && s < n ? (double)xb[s] : 0.0;
  }
  __syncthreads();
  const long long t = t0 + wp;
  if (t >= F) return;
  const double* fr = xs + wp * PY_H;
  double* d = dsm + wp * PY_LAGS;
  double acc[PY_LPL];
#pragma unroll
  for (int k = 0; k < PY_LPL; ++k) acc[k] = 0.0;
  // every lag has at least 2048 - 320 terms; lane l's lags are l + 1 + 32 k
  for (int j = 0; j < PY_N - PY_PMAX; ++j) {
    const double xj = fr[j];
#pragma unroll
    for (int k = 0; k < PY_LPL; ++k) {
      const double e = __dsub_rn(xj, fr[j + lane + 1 + 32 * k]);
      acc[k] = __dadd_rn(acc[k], __dmul_rn(e, e));
    }
  }
#pragma unroll
  for (int k = 0; k < PY_LPL; ++k) {
    const int tau = lane + 1 + 32 * k;
    double a = acc[k];
    for (int j = PY_N - PY_PMAX; j < PY_N - tau; ++j) {
      const double e = __dsub_rn(fr[j], fr[j + tau]);
      a = __dadd_rn(a, __dmul_rn(e, e));
    }
    d[tau] = a;
  }
  __syncwarp();
  if (lane == 0) {
    // yin.py: diff_mean = diff_mean * (tau - 1) / tau + diff / tau; cmndf = diff / (diff_mean + eps)
    double mean = 0.0;
    d[0] = 1.0;
    for (int tau = 1; tau < PY_LAGS; ++tau) {
      const double df = d[tau];
      mean = __dadd_rn(__ddiv_rn(__dmul_rn(mean, (double)(tau - 1)), (double)tau), __ddiv_rn(df, (double)tau));
      d[tau] = __ddiv_rn(df, __dadd_rn(mean, PY_EPS));
    }
    double e = 0.0;
    for (int j = 0; j < PY_N; ++j) e = __dadd_rn(e, __dmul_rn(fr[j], fr[j]));
    w.rms[fo + t] = sqrt(__ddiv_rn(e, (double)PY_N));
  }
  __syncwarp();
  for (int tau = lane; tau < PY_LAGS; tau += 32) {
    w.cmndf[(fo + t) * PY_LAGS + tau] = d[tau];
    if (ctap) ctap[PY_LAGS * fo + (long long)tau * F + t] = d[tau];
  }
}

// yin.py:parabolic_interpolation, each operation rounded once in the reference's order
__device__ __forceinline__ void parabolic(double y1, double y2, double y3, double& xi, double& yi) {
  const double a = __dadd_rn(PY_EPS, __ddiv_rn(__dsub_rn(__dadd_rn(y1, y3), __dmul_rn(2.0, y2)), 2.0));
  const double b = __ddiv_rn(__dsub_rn(y3, y1), 2.0);
  xi = __ddiv_rn(-b, __dmul_rn(2.0, a));
  yi = __dsub_rn(y2, __ddiv_rn(__dmul_rn(b, b), __dmul_rn(4.0, a)));
}

// np.argmin order: a NaN first (the first NaN), else the smaller value, ties to the smaller index
__device__ __forceinline__ bool argmin_before(double v, int i, double ov, int oi) {
  const bool n = isnan(v), on = isnan(ov);
  if (n != on) return n;
  if (n || v == ov) return i < oi;
  return v < ov;
}

struct PyThrSmem {
  double c[PY_TW][PY_LAGS];
  double ov[PY_TW][PY_B];       // the voiced half of the observation column
  double wgt[PY_TW][PY_NTHR];   // each threshold's weight
  int bin[PY_TW][PY_NTHR];      // and bin
  int16_t mins[PY_TW][PY_LAGS / 2 + 1];
};

// One warp per frame: pyin.py:probabilistic_thresholding and the column's normalisation (yin_multi_thr).
__global__ void __launch_bounds__(PY_TW * 32) pyin_thresh_kernel(ItemPass<PY_GROUP> it, PyWs w, PyTab tb,
                                                                 double* __restrict__ otap) {
  __shared__ PyThrSmem sm;
  const int b = blockIdx.y, wp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, t = (long long)blockIdx.x * PY_TW + wp;
  if (t >= F) return;
  const long long fr = fo + t;
  double* c = sm.c[wp];
  int16_t* mins = sm.mins[wp];
  for (int i = lane; i < PY_LAGS; i += 32) c[i] = i < PY_PMIN || i >= PY_PMAX ? INFINITY : w.cmndf[fr * PY_LAGS + i];
  __syncwarp();
  // strict local minima in 1 .. 319, ascending
  int k = 0;
  for (int base = 0; base < PY_LAGS; base += 32) {
    const int i = base + lane;
    const bool m = i >= 1 && i < PY_LAGS - 1 && c[i] < c[i - 1] && c[i] < c[i + 1];
    const unsigned bal = __ballot_sync(0xffffffffu, m);
    if (m) mins[k + __popc(bal & ((1u << lane) - 1u))] = (int16_t)i;
    k += __popc(bal);
  }
  __syncwarp();
  double* lagw = w.lag + fr * PY_NTHR;
  double* valw = w.val + fr * PY_NTHR;
  double* obs = w.obs + fr * PY_S;
  if (k == 0) {   // no minimum: a zero column, lags p_min, values 1
    for (int i = lane; i < PY_NTHR; i += 32) { lagw[i] = PY_PMIN; valw[i] = 1.0; }
    for (int i = lane; i < PY_B; i += 32) sm.ov[wp][i] = 0.0;
  } else {
    // delete_numba(arr, np.argwhere(arr == 319)) drops the element at position 0 when some minimum's lag equals the
    // position of 319 in the list (k - 1); nothing else is dropped, and the minima at 16 and 319 are interpolated
    bool hit = false;
    for (int i = lane; i < k; i += 32) hit |= mins[i] == k - 1;
    const bool drop0 = mins[k - 1] == PY_PMAX - 1 && __any_sync(0xffffffffu, hit);
    const int first = drop0 ? 1 : 0;
    double corr0 = 0.0;   // p_corr[0]: 0 when a minimum sits at 16, else the first interpolated minimum's correction
    for (int i = first + lane; i < k; i += 32) {
      const int m = mins[i];
      double xi, yi;
      parabolic(c[m - 1], c[m], c[m + 1], xi, yi);   // strict minima are never neighbours: no read sees a write
      if (i == first) corr0 = xi;
      c[m] = yi;
    }
    corr0 = __shfl_sync(0xffffffffu, corr0, 0);   // i == first ran on lane 0
    if (mins[0] == PY_PMIN) corr0 = 0.0;
    __syncwarp();
    // the frame's argmin and min, NaN first
    double av = INFINITY;
    int ai = PY_LAGS;
    for (int i = lane; i < PY_LAGS; i += 32)
      if (argmin_before(c[i], i, av, ai)) { av = c[i]; ai = i; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double ov = __shfl_xor_sync(0xffffffffu, av, o);
      const int oi = __shfl_xor_sync(0xffffffffu, ai, o);
      if (argmin_before(ov, oi, av, ai)) { av = ov; ai = oi; }
    }
    for (int i = lane; i < PY_NTHR; i += 32) {
      const double th = tb.thr[i];
      int q = 0;
      while (q < k && !(c[mins[q]] < th)) ++q;
      double lag, val, am;
      if (q == k) {
        lag = (double)ai;
        val = av;
        am = 0.01;   // absolute_min_prob
      } else {
        lag = __dadd_rn((double)mins[q], corr0);
        val = c[mins[q]];
        am = 1.0;
      }
      if (lag < PY_PMIN) lag = PY_PMIN;
      else if (lag >= PY_PMAX) lag = PY_PMAX - 1;
      lagw[i] = lag;
      valw[i] = val;
      // the first argmin of |1200 log2(F_axis / (16000 / lag))|: the distance falls then rises along the axis, so the
      // minimum lies within two bins of the nearest one
      const double f = __ddiv_rn(PY_FS, lag);
      const int b0 = (int)rint(120.0 * log2(f / 50.0));
      const int lo = max(0, b0 - 3), hi = min(PY_B - 1, b0 + 3);
      int best = lo;
      double bd = INFINITY;
      for (int q2 = lo; q2 <= hi; ++q2) {
        const double dist = fabs(__dmul_rn(1200.0, log2(__ddiv_rn(tb.fax[q2], f))));
        if (dist < bd) { bd = dist; best = q2; }
      }
      sm.bin[wp][i] = best;
      sm.wgt[wp][i] = __dmul_rn(am, tb.beta[i]);
    }
    __syncwarp();
    // O_m[bin] += weight in threshold order
    for (int q = lane; q < PY_B; q += 32) {
      double s = 0.0;
      for (int i = 0; i < PY_NTHR; ++i)
        if (sm.bin[wp][i] == q) s = __dadd_rn(s, sm.wgt[wp][i]);
      sm.ov[wp][q] = s;
    }
  }
  __syncwarp();
  // O[:B] *= voicing_prob; O[B:] = (1 - vp) (1 - sum of O[:B], ascending) / B
  double u = 0.0;
  if (lane == 0) {
    double s = 0.0;
    for (int q = 0; q < PY_B; ++q) s = __dadd_rn(s, __dmul_rn(sm.ov[wp][q], 0.5));
    u = __ddiv_rn(__dmul_rn(0.5, __dsub_rn(1.0, s)), (double)PY_B);
  }
  u = __shfl_sync(0xffffffffu, u, 0);
  double mx = u;
  for (int q = lane; q < PY_S; q += 32) {
    const double o = q < PY_B ? __dmul_rn(sm.ov[wp][q], 0.5) : u;
    obs[q] = o;
    if (otap) otap[PY_S * fo + (long long)q * F + t] = o;
    mx = fmax(mx, o);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  if (lane == 0) w.omax[fr] = mx;
}

struct PyVitArgs {
  const double* oext;   // the DP-only entry: O as [PY_S][F] per item at the caller's offsets; null: the workspace's
  int32_t* path;        // [frame]
};

struct PyVitSmem {
  double D[2][PY_S];
  double blog[PY_S][PY_BAND];
  int16_t bidx[PY_S][PY_BAND];
  double red[PY_VT / 32];
  int redi[PY_VT / 32];
};

// The block's first argmax of v (NaN-free), every thread gets it
__device__ __forceinline__ int block_first_argmax(double v, int i, PyVitSmem& sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ov > v || (ov == v && oi < i)) { v = ov; i = oi; }
  }
  __syncthreads();
  if ((threadIdx.x & 31) == 0) { sm.red[threadIdx.x >> 5] = v; sm.redi[threadIdx.x >> 5] = i; }
  __syncthreads();
  double bv = sm.red[0];
  int bi = sm.redi[0];
  for (int q = 1; q < PY_VT / 32; ++q)
    if (sm.red[q] > bv || (sm.red[q] == bv && sm.redi[q] < bi)) { bv = sm.red[q]; bi = sm.redi[q]; }
  return bi;
}

// The block's smallest i, every thread gets it
__device__ __forceinline__ int block_min_index(int i, PyVitSmem& sm) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) i = min(i, __shfl_xor_sync(0xffffffffu, i, o));
  __syncthreads();
  if ((threadIdx.x & 31) == 0) sm.redi[threadIdx.x >> 5] = i;
  __syncthreads();
  int b = sm.redi[0];
  for (int q = 1; q < PY_VT / 32; ++q) b = min(b, sm.redi[q]);
  return b;
}

// One CTA per item: viterbi_log_likelihood(A, 1 / 1036, O), states tid + 384 r.
__global__ void __launch_bounds__(PY_VT) pyin_viterbi_kernel(ItemPass<PY_GROUP> it, PyWs w, PyTab tb, PyVitArgs a) {
  extern __shared__ __align__(16) unsigned char sm_raw[];
  PyVitSmem& sm = *reinterpret_cast<PyVitSmem*>(sm_raw);
  const int ib = blockIdx.x, tid = threadIdx.x;
  const long long fo = it.out[ib], F = it.out[ib + 1] - fo;
  for (int i = tid; i < PY_S * PY_BAND; i += PY_VT) {
    (&sm.blog[0][0])[i] = tb.blog[i];
    (&sm.bidx[0][0])[i] = (int16_t)tb.bidx[i];
  }
  auto lo = [&](long long n, int s) {
    const double o = a.oext ? a.oext[PY_S * it.in[ib] + (long long)s * F + n] : w.obs[(fo + n) * PY_S + s];
    return log(__dadd_rn(o, PY_TINY));
  };
#pragma unroll
  for (int r = 0; r < PY_VS; ++r) {
    const int s = tid + r * PY_VT;
    if (s < PY_S) sm.D[0][s] = __dadd_rn(tb.log_init, lo(0, s));
  }
  for (long long n = 1; n < F; ++n) {
    const double* Dp = sm.D[(n - 1) & 1];
    double* Dn = sm.D[n & 1];
    __syncthreads();
    double v = -INFINITY;
    int vi = PY_S;
#pragma unroll
    for (int r = 0; r < PY_VS; ++r) {
      const int s = tid + r * PY_VT;
      if (s < PY_S && Dp[s] > v) { v = Dp[s]; vi = s; }
    }
    // every predecessor outside a column's list adds log(tiny); the rounded sum can absorb the last bits of D, so the
    // best of them is the first k whose log(tiny) + D[k] rounds to the largest such sum, not always the argmax of D
    const double vg = __dadd_rn(tb.log_tiny, Dp[block_first_argmax(v, vi, sm)]);
    int gi = PY_S;
#pragma unroll
    for (int r = PY_VS - 1; r >= 0; --r) {
      const int s = tid + r * PY_VT;
      if (s < PY_S && __dadd_rn(tb.log_tiny, Dp[s]) == vg) gi = s;
    }
    const int g = block_min_index(gi, sm);
#pragma unroll
    for (int r = 0; r < PY_VS; ++r) {
      const int s = tid + r * PY_VT;
      if (s >= PY_S) continue;
      double best = -INFINITY;
      int arg = 0;
      bool in = false;
      for (int q = 0; q < PY_BAND; ++q) {
        const int kq = sm.bidx[s][q];
        if (kq < 0) break;
        in |= kq == g;
        const double c = __dadd_rn(sm.blog[s][q], Dp[kq]);
        if (c > best) { best = c; arg = kq; }
      }
      if (!in && (vg > best || (vg == best && g < arg))) { best = vg; arg = g; }
      Dn[s] = __dadd_rn(best, lo(n, s));
      w.bp[(fo + n - 1) * PY_S + s] = (uint16_t)arg;
    }
  }
  __syncthreads();
  const double* Dl = sm.D[(F - 1) & 1];
  double v = -INFINITY;
  int vi = PY_S;
#pragma unroll
  for (int r = 0; r < PY_VS; ++r) {
    const int s = tid + r * PY_VT;
    if (s < PY_S && Dl[s] > v) { v = Dl[s]; vi = s; }
  }
  int e = block_first_argmax(v, vi, sm);   // its barriers also publish every thread's back-pointers to thread 0
  if (tid != 0) return;
  for (long long n = F - 1; n >= 0; --n) {
    a.path[fo + n] = e;
    if (n > 0) e = w.bp[(fo + n - 1) * PY_S + e];
  }
}

// One thread per frame: the f0 of the path, the suppressions, conf and refine_estimates_yin.
__global__ void pyin_tail_kernel(ItemPass<PY_GROUP> it, PyWs w, PyTab tb, double* __restrict__ f0,
                                 double* __restrict__ conf) {
  const long long fr = it.out[0] + (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (fr >= it.out[it.n]) return;
  const int b = item_of(it.out, fr);
  const long long t = fr - it.out[b];
  const int p = w.path[fr];
  double f = p < PY_B ? tb.fax[p] : 0.0;
  if (t == 0 || w.rms[fr] < 0.01) f = 0.0;
  conf[fr] = __ddiv_rn(w.obs[fr * PY_S + p], w.omax[fr]);
  if (f > 0.0) {
    // the thresholds' frequencies within 10 cents of f; the smallest CMNDF value among them (NaN first, then first)
    int best = -1;
    double bv = 0.0;
    for (int i = 0; i < PY_NTHR; ++i) {
      const double fi = __ddiv_rn(PY_FS, w.lag[fr * PY_NTHR + i]);
      if (fabs(__dmul_rn(1200.0, log2(__ddiv_rn(fi, f)))) < 10.0) {
        const double vi = w.val[fr * PY_NTHR + i];
        if (best < 0 || argmin_before(vi, i, bv, best)) { best = i; bv = vi; }
      }
    }
    if (best >= 0) f = __ddiv_rn(PY_FS, w.lag[fr * PY_NTHR + best]);
  }
  f0[fr] = f;
}

// workspace regions, in the order the entry point carves them; Ft bounds the frames of the batch
struct PyPlan {
  size_t cmndf, rms, obs, omax, lag, val, path, bp, bytes;
  explicit PyPlan(long long Ft, bool dp_only = false) {
    const size_t f = (size_t)Ft, z = dp_only ? 0 : 1;
    WsPlan p;
    cmndf = p.take(z * 8 * PY_LAGS * f);
    rms = p.take(z * 8 * f);
    obs = p.take(z * 8 * PY_S * f);
    omax = p.take(z * 8 * f);
    lag = p.take(z * 8 * PY_NTHR * f);
    val = p.take(z * 8 * PY_NTHR * f);
    path = p.take(z * 4 * f);
    bp = p.take(2 * PY_S * f);
    bytes = p.off;
  }
  PyWs carve(void* ws) const {
    char* base = static_cast<char*>(ws);
    PyWs w;
    w.cmndf = reinterpret_cast<double*>(base + cmndf);
    w.rms = reinterpret_cast<double*>(base + rms);
    w.obs = reinterpret_cast<double*>(base + obs);
    w.omax = reinterpret_cast<double*>(base + omax);
    w.lag = reinterpret_cast<double*>(base + lag);
    w.val = reinterpret_cast<double*>(base + val);
    w.path = reinterpret_cast<int32_t*>(base + path);
    w.bp = reinterpret_cast<uint16_t*>(base + bp);
    return w;
  }
};

// the device table's regions; log(1 / 1036 + tiny) and log(tiny) by the C library's log, as numba takes them
int pyin_tab(const double* tab, PyTab& tb) {
  if (!tab) { set_error("pyin: null table"); return SVCB_E_BAD_SHAPE; }
  tb.thr = tab + SVCB_PYIN_TAB_THR;
  tb.beta = tab + SVCB_PYIN_TAB_BETA;
  tb.fax = tab + SVCB_PYIN_TAB_FAXIS;
  tb.bidx = tab + SVCB_PYIN_TAB_BIDX;
  tb.blog = tab + SVCB_PYIN_TAB_BLOG;
  tb.log_init = std::log(1.0 / PY_S + PY_TINY);
  tb.log_tiny = std::log(PY_TINY);
  return SVCB_OK;
}

DevSmemCache g_py_cmndf_smem, g_py_vit_smem;
constexpr size_t PY_CMNDF_SMEM = 8 * (size_t)(PY_SPAN + PY_FT * PY_LAGS);

int launch_pyin_viterbi(const ItemPass<PY_GROUP>& it, const PyWs& w, const PyTab& tb, const PyVitArgs& a,
                        cudaStream_t s) {
  const double frames = (double)(it.out[it.n] - it.out[0]);
  KernelScope ks("pyin_viterbi", s, 2.0 * (PY_BAND + 1) * PY_S * frames, (8.0 + 2.0) * PY_S * frames);
  pyin_viterbi_kernel<<<(unsigned)it.n, PY_VT, sizeof(PyVitSmem), s>>>(it, w, tb, a);
  SVCB_LAUNCH_CHECK("pyin_viterbi");
  return SVCB_OK;
}

}  // namespace svcb

using namespace svcb;

extern "C" {

size_t svcb_pyin_f0_workspace_bytes(int64_t total_samples, int32_t B) {
  if (total_samples < 0 || B < 1) return 0;
  return PyPlan(total_samples / PY_H + B).bytes;
}

int svcb_pyin_f0_ragged(const float* x, const int64_t* offsets_host, int32_t B, const double* tab, double* f0,
                        double* conf, double* cmndf_tap, double* obs_tap, int32_t* path_tap, void* ws, size_t ws_bytes,
                        svcb_stream stream) {
  static const char* who = "svcb_pyin_f0_ragged";
  if (!x || !f0 || !conf || !offsets_host || !tab) {
    set_error(std::string(who) + ": null pointer");
    return SVCB_E_BAD_SHAPE;
  }
  SVCB_TRY(check_ragged(who, offsets_host, B, 1, 1, "samples", "an empty item has no frame"));
  const long long N = offsets_host[B] - offsets_host[0];
  const PyPlan plan(N / PY_H + B);
  SVCB_TRY(check_workspace(ws, ws_bytes, plan.bytes, who));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PyTab tb;
  SVCB_TRY(pyin_tab(tab, tb));
  SVCB_CUDA_CHECK(ensure_dyn_smem(pyin_cmndf_kernel, PY_CMNDF_SMEM, g_py_cmndf_smem));
  SVCB_CUDA_CHECK(ensure_dyn_smem(pyin_viterbi_kernel, sizeof(PyVitSmem), g_py_vit_smem));
  const PyWs w = plan.carve(ws);
  PyVitArgs a{};
  return for_each_pass<PY_GROUP>(offsets_host, B, [](long long n) { return pyin_frames(n); },
                                 [&](const ItemPass<PY_GROUP>& it, int) -> int {
    long long fmax = 0;
    for (int i = 0; i < it.n; ++i) fmax = std::max(fmax, it.out[i + 1] - it.out[i]);
    const long long total = it.out[it.n] - it.out[0];
    const double frames = (double)total;
    const unsigned items = (unsigned)it.n;
    {
      const double terms = 0.5 * (2.0 * PY_N - PY_PMAX - 1) * PY_PMAX;   // sum over tau of 2048 - tau
      KernelScope ks("pyin_cmndf", s, 3.0 * terms * frames, 4.0 * PY_N / PY_H * frames + 8.0 * PY_LAGS * frames);
      pyin_cmndf_kernel<<<dim3((unsigned)((fmax + PY_FT - 1) / PY_FT), items), PY_FT * 32, PY_CMNDF_SMEM, s>>>(
          x, it, w, cmndf_tap);
      SVCB_LAUNCH_CHECK("pyin_cmndf");
    }
    {
      KernelScope ks("pyin_thresh", s, 0.0, (8.0 * PY_LAGS + 8.0 * PY_S + 16.0 * PY_NTHR) * frames);
      pyin_thresh_kernel<<<dim3((unsigned)((fmax + PY_TW - 1) / PY_TW), items), PY_TW * 32, 0, s>>>(it, w, tb, obs_tap);
      SVCB_LAUNCH_CHECK("pyin_thresh");
    }
    a.path = w.path;
    SVCB_TRY(launch_pyin_viterbi(it, w, tb, a, s));
    {
      KernelScope ks("pyin_tail", s, 0.0, (16.0 * PY_NTHR + 48.0) * frames);
      pyin_tail_kernel<<<(unsigned)((total + 255) / 256), 256, 0, s>>>(it, w, tb, f0, conf);
      SVCB_LAUNCH_CHECK("pyin_tail");
    }
    if (path_tap) {
      SVCB_CUDA_CHECK(cudaMemcpyAsync(path_tap + it.out[0], w.path + it.out[0], 4 * (size_t)total,
                                      cudaMemcpyDeviceToDevice, s));
    }
    return SVCB_OK;
  });
}

size_t svcb_pyin_dp_workspace_bytes(int64_t total_frames) {
  if (total_frames < 0) return 0;
  return PyPlan(total_frames, true).bytes;
}

int svcb_pyin_dp_ragged(const double* obs, const int64_t* frame_offsets_host, int32_t B, const double* tab,
                        int32_t* path, void* ws, size_t ws_bytes, svcb_stream stream) {
  static const char* who = "svcb_pyin_dp_ragged";
  if (!obs || !path || !frame_offsets_host || !tab) {
    set_error(std::string(who) + ": null pointer");
    return SVCB_E_BAD_SHAPE;
  }
  SVCB_TRY(check_ragged(who, frame_offsets_host, B, 1, 1, "frames", nullptr));
  const PyPlan plan(frame_offsets_host[B] - frame_offsets_host[0], true);
  SVCB_TRY(check_workspace(ws, ws_bytes, plan.bytes, who));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  PyTab tb;
  SVCB_TRY(pyin_tab(tab, tb));
  SVCB_CUDA_CHECK(ensure_dyn_smem(pyin_viterbi_kernel, sizeof(PyVitSmem), g_py_vit_smem));
  const PyWs w = plan.carve(ws);
  PyVitArgs a{};
  a.oext = obs;
  a.path = path;
  return for_each_pass<PY_GROUP>(frame_offsets_host, B, [](long long n) { return n; },
                                 [&](const ItemPass<PY_GROUP>& it, int) -> int {
                                   return launch_pyin_viterbi(it, w, tb, a, s);
                                 });
}

}  // extern "C"

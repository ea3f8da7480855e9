// WORLD's DIO + StoneMask F0 (prepare/preprocess_f0.py:28-30: pyworld.dio(x, 16000, f0_ceil=900, frame_period=10),
// then pyworld.stonemask) for a ragged batch of float64 clips at 16 kHz, in fp64 on the device.
//
//   y          = [x, 0] - mean  (WORLD's y_length = n + 1: one trailing zero, then the mean of all n + 1 removed)
//   low-cut    = y through the 641-tap zero-phase Hann low-cut (50 Hz), a direct FIR over y zero-extended
//   band k     = the low-cut signal through a Nuttall window of 4 h_k taps delayed by 2 h_k, h_k = round(8000 / boundary_k)
//   WORLD does both filters as one product of spectra with an FFT long enough that nothing wraps; in exact arithmetic
//   that is this linear convolution, so no FFT is needed.
//   events     = per band, the refined falling zero crossings of the band, of its negation and of its first difference
//                both ways (ZeroCrossingEngine), compacted in order by one CTA per (band, item)
//   candidates = per frame and band, the four interval families interpolated onto the 10 ms grid (interp1 + histc:
//                end segments extrapolated), their mean and spread, the range rejection; then the best band per frame
//   fix        = FixF0Contour's four steps, sequential in time, one thread per item
//   StoneMask  = per voiced frame one warp: the Blackman window and its difference window, direct DFT bins of
//                harmonics 1-2 and then 1-6, the amplitude-weighted instantaneous frequency, the 20 % rule
//
// Every stage of an item reads only that item, with a fixed thread mapping, so each item's F0 is bitwise that of a
// lone call.  oracle/f0_oracle.py restates the same algorithm in numpy.
#include <cmath>
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int F0_FS = 16000;
constexpr double F0_PERIOD_MS = 10.0, F0_FLOOR = 71.0, F0_CEIL = 900.0, F0_ALLOWED = 0.1;
constexpr double F0_SAFE = 1e-12, F0_MAX_SCORE = 100000.0, F0_FLOOR_SM = 40.0;
constexpr int F0_BANDS = 8;
constexpr int F0_LC = 641, F0_LC_HALF = 320;   // low-cut taps: 2 round(fs / 50) + 1
constexpr int F0_YPAD = 480;                   // zeros either side of y: the bands reach the low-cut 2 h_max - 1 < 160 out
constexpr int F0_LPAD = 160;                   // low-cut positions kept either side of y
constexpr int F0_VRM = 3;                      // voice_range_minimum = int(0.5 + 1000 / 10 / 71) * 2 + 1
constexpr int F0_GROUP = 128;                  // items per pass
constexpr int F0_T = 256;                      // threads of the FIR / event CTAs
constexpr int F0_EV = 8;                       // positions per thread per event chunk
constexpr int F0_SM_WARPS = 2;                 // StoneMask: frames (warps) per CTA
constexpr int F0_SM_MAXL = 2 * 601 + 1;        // the window of the lowest F0 StoneMask refines (just above 40 Hz)

__constant__ double c_lowcut[F0_LC];
__constant__ double c_nuttall[4 * (80 + 56 + 40 + 28 + 20 + 14 + 10 + 7)];
__constant__ int c_half[F0_BANDS];             // h_k
__constant__ int c_noff[F0_BANDS];             // band k's first tap in c_nuttall
__constant__ double c_boundary[F0_BANDS];

inline int matlab_round_h(double x) { return x > 0 ? (int)(x + 0.5) : (int)(x - 0.5); }
__device__ __forceinline__ int matlab_round_d(double x) { return x > 0 ? (int)(x + 0.5) : (int)(x - 0.5); }

// Where an item's buffers sit in the workspace: all sizes are linear in the batch's samples before the item (S) and its
// index in the batch (g), so no table is needed.  Frame arrays are indexed by the pass's output offsets.
struct F0Ws {
  double *mean, *ypad, *ylc, *band, *fe, *cand, *best, *s1, *s2, *dio;
  int *cnt, *neg, *pos;
  long long in0;   // offsets_host[0]
  int g0;          // the pass's first item
};
struct F0Item {
  long long n, yl, S;
  int g;
};
__device__ __forceinline__ F0Item f0_item(const ItemPass<F0_GROUP>& it, const F0Ws& w, int b) {
  F0Item r;
  r.n = it.in[b + 1] - it.in[b];
  r.yl = r.n + 1;
  r.S = it.in[b] - w.in0;
  r.g = w.g0 + b;
  return r;
}
__device__ __forceinline__ double* ypad_of(const F0Ws& w, const F0Item& t) { return w.ypad + t.S + (long long)t.g * (1 + 2 * F0_YPAD); }
__device__ __forceinline__ double* ylc_of(const F0Ws& w, const F0Item& t) { return w.ylc + t.S + (long long)t.g * (1 + 2 * F0_LPAD); }
__device__ __forceinline__ double* band_of(const F0Ws& w, const F0Item& t, int k) { return w.band + F0_BANDS * (t.S + t.g) + k * t.yl; }
__device__ __forceinline__ double* fe_of(const F0Ws& w, const F0Item& t, int k, int f) {
  return w.fe + 4 * F0_BANDS * (t.S + t.g) + (k * 4 + f) * t.yl;
}

// mean of y = [x, 0]: sum(x) / (n + 1)
__global__ void __launch_bounds__(F0_T) f0_mean_kernel(const double* __restrict__ x, ItemPass<F0_GROUP> it, F0Ws w) {
  __shared__ double part[F0_T / 32];
  const int b = blockIdx.x, tid = threadIdx.x;
  const F0Item t = f0_item(it, w, b);
  const double* xb = x + it.in[b];
  double s = 0.0;
  for (long long i = tid; i < t.n; i += F0_T) s += xb[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((tid & 31) == 0) part[tid >> 5] = s;
  __syncthreads();
  if (tid == 0) {
    double tot = 0.0;
    for (int i = 0; i < F0_T / 32; ++i) tot += part[i];
    w.mean[t.g] = tot / (double)t.yl;
  }
}

// ypad[j] = y[j - 480], zero outside [0, n]
__global__ void __launch_bounds__(F0_T) f0_center_kernel(const double* __restrict__ x, ItemPass<F0_GROUP> it, F0Ws w) {
  const int b = blockIdx.y;
  const F0Item t = f0_item(it, w, b);
  const long long len = t.yl + 2 * F0_YPAD, j = (long long)blockIdx.x * F0_T + threadIdx.x;
  if (j >= len) return;
  const long long p = j - F0_YPAD;
  const double m = w.mean[t.g];
  ypad_of(w, t)[j] = p >= 0 && p < t.n ? x[it.in[b] + p] - m : (p == t.n ? -m : 0.0);
}

// ylc[j] = low-cut at position j - 160 = sum_t lowcut[t] y[j - 160 - (t - 320)] = sum_t lowcut[t] ypad[j + 640 - t]
__global__ void __launch_bounds__(F0_T) f0_lowcut_kernel(ItemPass<F0_GROUP> it, F0Ws w) {
  const int b = blockIdx.y;
  const F0Item t = f0_item(it, w, b);
  const long long len = t.yl + 2 * F0_LPAD, j = (long long)blockIdx.x * F0_T + threadIdx.x;
  if (j >= len) return;
  const double* yp = ypad_of(w, t) + j + 2 * F0_LC_HALF;
  double s = 0.0;
#pragma unroll 8
  for (int k = 0; k < F0_LC; ++k) s += c_lowcut[k] * yp[-k];
  ylc_of(w, t)[j] = s;
}

// band_k[i] = sum_{q < 4h} nuttall_k[q] lowcut(i + 2h - q), i = 0 .. y_length - 1
__global__ void __launch_bounds__(F0_T) f0_band_kernel(ItemPass<F0_GROUP> it, F0Ws w) {
  const int b = blockIdx.y, k = blockIdx.z;
  const F0Item t = f0_item(it, w, b);
  const long long i = (long long)blockIdx.x * F0_T + threadIdx.x;
  if (i >= t.yl) return;
  const int h = c_half[k];
  const double* wk = c_nuttall + c_noff[k];
  const double* lp = ylc_of(w, t) + F0_LPAD + i + 2 * h;
  double s = 0.0;
#pragma unroll 4
  for (int q = 0; q < 4 * h; ++q) s += wk[q] * lp[-q];
  band_of(w, t, k)[i] = s;
}

// The four event families of band k of one item, in order: family 0 falls through zero on f, 1 on -f, 2 on the
// difference d[i] = f[i+1] - f[i] (peaks), 3 on -d (dips).  A falling crossing of s sits at e where s[e-1] > 0 >= s[e];
// its refined place is e - s[e-1] / (s[e] - s[e-1]), the same for s and -s.  Each chunk of F0_T * F0_EV positions
// counts its crossings per family (four 16-bit counts in one 64-bit word), scans them across the CTA and writes
// the refined places after those of the earlier chunks.
__global__ void __launch_bounds__(F0_T) f0_events_kernel(ItemPass<F0_GROUP> it, F0Ws w) {
  __shared__ unsigned long long wtot[F0_T / 32];
  __shared__ long long run[4];
  const int k = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const F0Item t = f0_item(it, w, b);
  const double* f = band_of(w, t, k);
  double* fe[4];
#pragma unroll
  for (int q = 0; q < 4; ++q) fe[q] = fe_of(w, t, k, q);
  const long long L0 = t.yl, L1 = t.yl - 1;   // signal lengths of families 0-1 and 2-3
  if (tid < 4) run[tid] = 0;
  __syncthreads();
  for (long long base = 0; base < L0; base += (long long)F0_T * F0_EV) {
    const long long i0 = base + (long long)tid * F0_EV;
    double v[F0_EV + 2];
#pragma unroll
    for (int e = 0; e < F0_EV + 2; ++e) v[e] = i0 + e < L0 ? f[i0 + e] : 0.0;
    unsigned mask[4] = {0u, 0u, 0u, 0u};   // bit e: a crossing between positions i0 + e and i0 + e + 1
#pragma unroll
    for (int e = 0; e < F0_EV; ++e) {
      const long long i = i0 + e;
      if (i + 1 < L0) {
        if (v[e] > 0.0 && v[e + 1] <= 0.0) mask[0] |= 1u << e;
        if (-v[e] > 0.0 && -v[e + 1] <= 0.0) mask[1] |= 1u << e;
      }
      if (i + 1 < L1) {
        const double d0 = v[e + 1] - v[e], d1 = v[e + 2] - v[e + 1];
        if (d0 > 0.0 && d1 <= 0.0) mask[2] |= 1u << e;
        if (-d0 > 0.0 && -d1 <= 0.0) mask[3] |= 1u << e;
      }
    }
    const unsigned long long own = (unsigned long long)__popc(mask[0]) | (unsigned long long)__popc(mask[1]) << 16 |
                                   (unsigned long long)__popc(mask[2]) << 32 | (unsigned long long)__popc(mask[3]) << 48;
    unsigned long long inc = own;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned long long u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (lane == 31) wtot[warp] = inc;
    __syncthreads();
    unsigned long long ex = inc - own, tot = 0;
    for (int q = 0; q < F0_T / 32; ++q) {
      if (q < warp) ex += wtot[q];
      tot += wtot[q];
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      long long o = run[q] + (long long)((ex >> (16 * q)) & 0xffffu);
      unsigned m = mask[q];
      while (m) {
        const int e = __ffs(m) - 1;
        m &= m - 1;
        double a, c;   // s[e'-1], s[e'] at the crossing e' = i0 + e + 1 (the sign of s does not change the place)
        if (q < 2) { a = v[e]; c = v[e + 1]; } else { a = v[e + 1] - v[e]; c = v[e + 2] - v[e + 1]; }
        fe[q][o++] = (double)(i0 + e + 1) - a / (c - a);
      }
    }
    __syncthreads();
    if (tid < 4) run[tid] += (long long)((tot >> (16 * tid)) & 0xffffu);
    __syncthreads();
  }
  if (tid < 4) w.cnt[t.g * 4 * F0_BANDS + k * 4 + tid] = (int)run[tid];
}

// interp1 of one family at time tp: m = number of intervals (>= 3), interval q at (fe[q] + fe[q+1]) / 2 / fs with
// value fs / (fe[q+1] - fe[q]); histc's segment index clipped to 1 .. m - 1
__device__ __forceinline__ double f0_interp(const double* __restrict__ fe, int m, double tp) {
  const double fs = (double)F0_FS;
  auto loc = [&](int q) { return (fe[q] + fe[q + 1]) / 2.0 / fs; };
  int lo = 0, hi = m;   // the number of locations <= tp
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (loc(mid) <= tp) lo = mid + 1; else hi = mid;
  }
  const int q = min(max(lo, 1), m - 1);
  const double x0 = loc(q - 1), x1 = loc(q);
  const double y0 = fs / (fe[q] - fe[q - 1]), y1 = fs / (fe[q + 1] - fe[q]);
  const double s = (tp - x0) / (x1 - x0);
  return y0 + s * (y1 - y0);
}

// One thread per frame: the eight bands' candidates (kept for the contour fix) and the best of them.
__global__ void __launch_bounds__(128) f0_candidates_kernel(ItemPass<F0_GROUP> it, F0Ws w) {
  const int b = blockIdx.y;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, i = (long long)blockIdx.x * 128 + threadIdx.x;
  if (i >= F) return;
  const F0Item t = f0_item(it, w, b);
  const double tp = (double)i * F0_PERIOD_MS / 1000.0;
  const int* cnt = w.cnt + t.g * 4 * F0_BANDS;
  double best = 0.0, bscore = 0.0;
  for (int k = 0; k < F0_BANDS; ++k) {
    bool ok = true;
#pragma unroll
    for (int q = 0; q < 4; ++q) ok = ok && cnt[k * 4 + q] - 1 >= 3;
    double c = 0.0, sc = F0_MAX_SCORE;
    if (ok) {
      double a[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) a[q] = f0_interp(fe_of(w, t, k, q), cnt[k * 4 + q] - 1, tp);
      c = (a[0] + a[1] + a[2] + a[3]) / 4.0;
      sc = sqrt(((a[0] - c) * (a[0] - c) + (a[1] - c) * (a[1] - c) + (a[2] - c) * (a[2] - c) + (a[3] - c) * (a[3] - c)) / 3.0);
      const double bd = c_boundary[k];
      if (c > bd || c < bd / 2.0 || c > F0_CEIL || c < F0_FLOOR) {
        c = 0.0;
        sc = F0_MAX_SCORE;
      }
    }
    sc = sc / (c + F0_SAFE);
    w.cand[F0_BANDS * fo + k * F + i] = c;
    if (k == 0 || bscore > sc) {
      bscore = sc;
      best = c;
    }
  }
  w.best[fo + i] = best;
}

__device__ double f0_select_best(double cur, double past, const double* __restrict__ cand, long long F, long long j) {
  const double ref = (cur * 3.0 - past) / 2.0;
  double err = fabs(ref - cand[j]), best = cand[j];
  for (int k = 1; k < F0_BANDS; ++k) {
    const double e = fabs(ref - cand[k * F + j]);
    if (e < err) {
      err = e;
      best = cand[k * F + j];
    }
  }
  return fabs(1.0 - best / ref) > F0_ALLOWED ? 0.0 : best;   // 0 / 0 is NaN, not rejected: best is then 0 anyway
}

// FixF0Contour, one thread per item, in time order.  At most F0_VRM frames: WORLD returns without writing; the
// caller's zeroed buffer stays, so the output is zero.
__global__ void f0_fix_kernel(ItemPass<F0_GROUP> it, F0Ws w) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= it.n) return;
  const long long fo = it.out[b], F = it.out[b + 1] - fo;
  const double* best = w.best + fo;
  const double* cand = w.cand + F0_BANDS * fo;
  double *s1 = w.s1 + fo, *s2 = w.s2 + fo, *out = w.dio + fo;
  int *neg = w.neg + fo, *pos = w.pos + fo;
  if (F <= F0_VRM) {
    for (long long i = 0; i < F; ++i) out[i] = 0.0;
    return;
  }
  auto base = [&](long long i) { return i >= F0_VRM && i < F - F0_VRM ? best[i] : 0.0; };
  for (long long i = 0; i < F0_VRM; ++i) s1[i] = 0.0;
  for (long long i = F0_VRM; i < F; ++i) {
    const double v = base(i);
    s1[i] = fabs((v - base(i - 1)) / (F0_SAFE + v)) < F0_ALLOWED ? v : 0.0;
  }
  const int c = (F0_VRM - 1) / 2;
  for (long long i = 0; i < F; ++i) {
    double v = s1[i];
    if (i >= c && i < F - c)
      for (int j = -c; j <= c; ++j)
        if (s1[i + j] == 0) { v = 0.0; break; }
    s2[i] = v;
  }
  long long nn = 0, np = 0;
  for (long long i = 1; i < F; ++i) {
    if (s2[i] == 0 && s2[i - 1] != 0) neg[nn++] = (int)(i - 1);
    else if (s2[i - 1] == 0 && s2[i] != 0) pos[np++] = (int)i;
  }
  double* s3 = s1;   // step 1 is done with
  for (long long i = 0; i < F; ++i) s3[i] = s2[i];
  for (long long i = 0; i < nn; ++i) {
    const long long limit = i == nn - 1 ? F - 1 : neg[i + 1];
    for (long long j = neg[i]; j < limit; ++j) {
      s3[j + 1] = f0_select_best(s3[j], s3[j - 1], cand, F, j + 1);
      if (s3[j + 1] == 0) break;
    }
  }
  for (long long i = 0; i < F; ++i) out[i] = s3[i];
  for (long long i = np - 1; i >= 0; --i) {
    const long long limit = i == 0 ? 1 : pos[i - 1];
    for (long long j = pos[i]; j > limit; --j) {
      out[j - 1] = f0_select_best(out[j], out[j + 1], cand, F, j - 1);
      if (out[j - 1] == 0) break;
    }
  }
}

// StoneMask's FixF0 over bins idx[0 .. nh) of the warp's windowed frame (vm, vd in shared memory, L samples, DFT of
// size N): the amplitude-weighted instantaneous frequency.  A bin above N / 2 lies outside WORLD's half spectrum and
// counts as zero power.
template <int NH>
__device__ double f0_fix_bins(const double* vm, const double* vd, int L, int N, double f0, int lane) {
  const double fs = (double)F0_FS;
  int idx[NH];
  double mr[NH], mi[NH], dr[NH], di[NH];
#pragma unroll
  for (int h = 0; h < NH; ++h) {
    idx[h] = matlab_round_d(f0 * N / fs * (h + 1));
    mr[h] = mi[h] = dr[h] = di[h] = 0.0;
  }
  for (int k = lane; k < L; k += 32) {
    const double a = vm[k], d = vd[k];
#pragma unroll
    for (int h = 0; h < NH; ++h) {
      const int r = (int)(((long long)idx[h] * k) & (N - 1));
      double s, c;
      sincospi(2.0 * (double)r / (double)N, &s, &c);
      mr[h] += a * c; mi[h] -= a * s;
      dr[h] += d * c; di[h] -= d * s;
    }
  }
  double num = 0.0, den = 0.0;
#pragma unroll
  for (int h = 0; h < NH; ++h) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mr[h] += __shfl_xor_sync(0xffffffffu, mr[h], o);
      mi[h] += __shfl_xor_sync(0xffffffffu, mi[h], o);
      dr[h] += __shfl_xor_sync(0xffffffffu, dr[h], o);
      di[h] += __shfl_xor_sync(0xffffffffu, di[h], o);
    }
    const double p = idx[h] > N / 2 ? 0.0 : mr[h] * mr[h] + mi[h] * mi[h];
    const double ni = mr[h] * di[h] - mi[h] * dr[h];
    const double ifreq = p == 0.0 ? 0.0 : (double)idx[h] * fs / N + ni / p * fs / 2.0 / M_PI;
    const double amp = sqrt(p);
    num += amp * ifreq;
    den += amp * (h + 1.0);
  }
  return num / (den + F0_SAFE);
}

// StoneMask: one warp per frame of DIO's contour.
__global__ void __launch_bounds__(32 * F0_SM_WARPS) f0_stonemask_kernel(const double* __restrict__ x, double* __restrict__ out,
                                                                       ItemPass<F0_GROUP> it, F0Ws w) {
  __shared__ double sv[F0_SM_WARPS][2][F0_SM_MAXL];
  const int b = blockIdx.y, lane = threadIdx.x & 31, wp = threadIdx.x >> 5;
  const long long fo = it.out[b], F = it.out[b + 1] - fo, i = (long long)blockIdx.x * F0_SM_WARPS + wp;
  if (i >= F) return;
  const double fs = (double)F0_FS, f0 = w.dio[fo + i], tp = (double)i * F0_PERIOD_MS / 1000.0;
  if (f0 <= F0_FLOOR_SM || f0 > fs / 12.0) {
    if (lane == 0) out[fo + i] = 0.0;
    return;
  }
  const long long n = it.in[b + 1] - it.in[b];
  const double* xb = x + it.in[b];
  const int hw = (int)(1.5 * fs / f0 + 1.0), L = 2 * hw + 1;
  const double wlt = (2.0 * hw + 1.0) / fs;
  const int N = 1 << (2 + (31 - __clz(L)));   // 2^(2 + int(log2 L)); L is odd, so log2 L is never an integer
  auto raw = [&](int k) { return matlab_round_d((tp + (double)(-hw + k) / fs) * fs); };
  auto win = [&](int k) {
    const double u = (double)(raw(k) - 1.0) / fs - tp;
    return 0.42 + 0.5 * cos(2.0 * M_PI * u / wlt) + 0.08 * cos(4.0 * M_PI * u / wlt);
  };
  double* vm = sv[wp][0];
  double* vd = sv[wp][1];
  for (int k = lane; k < L; k += 32) vm[k] = win(k);
  __syncwarp();
  for (int k = lane; k < L; k += 32) {
    const double d = k == 0 ? -vm[1] / 2.0 : (k == L - 1 ? vm[L - 2] / 2.0 : -(vm[k + 1] - vm[k - 1]) / 2.0);
    const long long q = min(max((long long)raw(k) - 1, 0ll), n - 1);
    vd[k] = xb[q] * d;
  }
  __syncwarp();
  for (int k = lane; k < L; k += 32) {
    const long long q = min(max((long long)raw(k) - 1, 0ll), n - 1);
    vm[k] = xb[q] * vm[k];
  }
  __syncwarp();
  const double t = f0_fix_bins<2>(vm, vd, L, N, f0, lane);
  const double mean = t <= 0.0 || t > f0 * 2 ? 0.0 : f0_fix_bins<6>(vm, vd, L, N, t, lane);
  if (lane == 0) out[fo + i] = fabs(mean - f0) > f0 * 0.2 ? f0 : mean;
}

// Host copies of the taps, computed as WORLD computes them (DesignLowCutFilter, NuttallWindow).
struct F0Taps {
  double lowcut[F0_LC];
  double nuttall[4 * (80 + 56 + 40 + 28 + 20 + 14 + 10 + 7)];
  int half[F0_BANDS], noff[F0_BANDS];
  double boundary[F0_BANDS];
  F0Taps() {
    const double pi = 3.1415926535897932384626433832795;
    double sum = 0.0;
    for (int i = 1; i <= F0_LC; ++i) {
      lowcut[i - 1] = 0.5 - 0.5 * std::cos(i * 2.0 * pi / (F0_LC + 1));
      sum += lowcut[i - 1];
    }
    for (int i = 0; i < F0_LC; ++i) lowcut[i] = -lowcut[i] / sum;
    lowcut[F0_LC_HALF] += 1.0;
    int off = 0;
    for (int k = 0; k < F0_BANDS; ++k) {
      boundary[k] = F0_FLOOR * std::pow(2.0, (k + 1) / 2.0);
      half[k] = matlab_round_h(F0_FS / boundary[k] / 2.0);
      noff[k] = off;
      const int n = 4 * half[k];
      for (int i = 0; i < n; ++i) {
        const double u = i / (n - 1.0);
        nuttall[off + i] = 0.355768 - 0.487396 * std::cos(2.0 * pi * u) + 0.144232 * std::cos(4.0 * pi * u) -
                           0.012604 * std::cos(6.0 * pi * u);
      }
      off += n;
    }
  }
};

// the constant banks belong to a device: upload them once per device
int f0_upload_taps() {
  static const F0Taps taps;
  static std::atomic<bool> done[kMaxDevices];
  int dev = 0;
  SVCB_CUDA_CHECK(cudaGetDevice(&dev));
  if (dev >= 0 && dev < kMaxDevices && done[dev].load()) return SVCB_OK;
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_lowcut, taps.lowcut, sizeof(taps.lowcut)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_nuttall, taps.nuttall, sizeof(taps.nuttall)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_half, taps.half, sizeof(taps.half)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_noff, taps.noff, sizeof(taps.noff)));
  SVCB_CUDA_CHECK(cudaMemcpyToSymbol(c_boundary, taps.boundary, sizeof(taps.boundary)));
  if (dev >= 0 && dev < kMaxDevices) done[dev].store(true);
  return SVCB_OK;
}

// workspace regions, in the order f0_workspace carves them
struct F0Plan {
  size_t mean, ypad, ylc, band, fe, cand, best, s1, s2, dio, cnt, neg, pos, bytes;
  F0Plan(long long N, int B) {
    const long long Ft = N / 160 + B;   // sum of n_b // 160 + 1
    WsPlan p;
    mean = p.take(8 * (size_t)B);
    ypad = p.take(8 * (size_t)(N + (long long)B * (1 + 2 * F0_YPAD)));
    ylc = p.take(8 * (size_t)(N + (long long)B * (1 + 2 * F0_LPAD)));
    band = p.take(8 * (size_t)F0_BANDS * (size_t)(N + B));
    fe = p.take(8 * (size_t)(4 * F0_BANDS) * (size_t)(N + B));
    cand = p.take(8 * (size_t)F0_BANDS * (size_t)Ft);
    best = p.take(8 * (size_t)Ft);
    s1 = p.take(8 * (size_t)Ft);
    s2 = p.take(8 * (size_t)Ft);
    dio = p.take(8 * (size_t)Ft);
    cnt = p.take(4 * (size_t)(4 * F0_BANDS) * (size_t)B);
    neg = p.take(4 * (size_t)Ft);
    pos = p.take(4 * (size_t)Ft);
    bytes = p.off;
  }
};

}  // namespace svcb

using namespace svcb;

extern "C" {

size_t svcb_world_f0_workspace_bytes(int64_t total_samples, int32_t B) {
  if (total_samples < 0 || B < 1) return 0;
  return F0Plan(total_samples, B).bytes;
}

int svcb_world_f0_ragged(const double* x, const int64_t* offsets_host, int32_t B, double* out, void* ws, size_t ws_bytes,
                         svcb_stream stream) {
  static const char* who = "svcb_world_f0_ragged";
  if (!x || !out || !offsets_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, offsets_host, B, 1, 1, "samples", nullptr));
  const long long N = offsets_host[B] - offsets_host[0];
  const F0Plan plan(N, B);
  SVCB_TRY(check_workspace(ws, ws_bytes, plan.bytes, who));
  SVCB_TRY(f0_upload_taps());
  char* base = static_cast<char*>(ws);
  F0Ws w;
  w.mean = reinterpret_cast<double*>(base + plan.mean);
  w.ypad = reinterpret_cast<double*>(base + plan.ypad);
  w.ylc = reinterpret_cast<double*>(base + plan.ylc);
  w.band = reinterpret_cast<double*>(base + plan.band);
  w.fe = reinterpret_cast<double*>(base + plan.fe);
  w.cand = reinterpret_cast<double*>(base + plan.cand);
  w.best = reinterpret_cast<double*>(base + plan.best);
  w.s1 = reinterpret_cast<double*>(base + plan.s1);
  w.s2 = reinterpret_cast<double*>(base + plan.s2);
  w.dio = reinterpret_cast<double*>(base + plan.dio);
  w.cnt = reinterpret_cast<int*>(base + plan.cnt);
  w.neg = reinterpret_cast<int*>(base + plan.neg);
  w.pos = reinterpret_cast<int*>(base + plan.pos);
  w.in0 = offsets_host[0];
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return for_each_pass<F0_GROUP>(offsets_host, B, [](long long n) { return n / 160 + 1; },
                                 [&](const ItemPass<F0_GROUP>& it, int g0) -> int {
    w.g0 = g0;
    long long nmax = 0, fmax = 0, samples = it.in[it.n] - it.in[0], frames = it.out[it.n] - it.out[0];
    for (int i = 0; i < it.n; ++i) {
      nmax = std::max(nmax, it.in[i + 1] - it.in[i]);
      fmax = std::max(fmax, it.out[i + 1] - it.out[i]);
    }
    const unsigned items = (unsigned)it.n;
    auto tiles = [](long long len, int per) { return (unsigned)((len + per - 1) / per); };
    {
      KernelScope ks("f0_bands", s, 2.0 * (samples + items) * (F0_LC + 4.0 * (80 + 56 + 40 + 28 + 20 + 14 + 10 + 7)),
                     8.0 * samples * (1 + 2 + 2 + 2 * F0_BANDS));
      f0_mean_kernel<<<items, F0_T, 0, s>>>(x, it, w);
      SVCB_LAUNCH_CHECK("f0_mean");
      f0_center_kernel<<<dim3(tiles(nmax + 1 + 2 * F0_YPAD, F0_T), items), F0_T, 0, s>>>(x, it, w);
      SVCB_LAUNCH_CHECK("f0_center");
      f0_lowcut_kernel<<<dim3(tiles(nmax + 1 + 2 * F0_LPAD, F0_T), items), F0_T, 0, s>>>(it, w);
      SVCB_LAUNCH_CHECK("f0_lowcut");
      f0_band_kernel<<<dim3(tiles(nmax + 1, F0_T), items, F0_BANDS), F0_T, 0, s>>>(it, w);
      SVCB_LAUNCH_CHECK("f0_band");
    }
    {
      KernelScope ks("f0_events", s, 0.0, 8.0 * F0_BANDS * samples);
      f0_events_kernel<<<dim3(F0_BANDS, items), F0_T, 0, s>>>(it, w);
      SVCB_LAUNCH_CHECK("f0_events");
    }
    {
      KernelScope ks("f0_candidates", s, 0.0, 8.0 * F0_BANDS * frames);
      f0_candidates_kernel<<<dim3(tiles(fmax, 128), items), 128, 0, s>>>(it, w);
      SVCB_LAUNCH_CHECK("f0_candidates");
    }
    {
      KernelScope ks("f0_fix", s, 0.0, 8.0 * (F0_BANDS + 4) * frames);
      f0_fix_kernel<<<tiles(items, 32), 32, 0, s>>>(it, w);
      SVCB_LAUNCH_CHECK("f0_fix");
    }
    {
      KernelScope ks("f0_stonemask", s, 0.0, 16.0 * frames);
      f0_stonemask_kernel<<<dim3(tiles(fmax, F0_SM_WARPS), items), 32 * F0_SM_WARPS, 0, s>>>(x, out, it, w);
      SVCB_LAUNCH_CHECK("f0_stonemask");
    }
    return SVCB_OK;
  });
}

}  // extern "C"

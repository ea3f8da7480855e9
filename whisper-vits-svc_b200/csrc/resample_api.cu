// Resampling of raw recordings to the training rates (prepare/preprocess_a.py:10-14, librosa.load(path, sr) and the
// int16 normalisation that follows it) on the device.
//
//   resample     polyphase FIR of scipy.signal.resample_poly: y[j] = sum_k h[k] xup[(j + rm) down - k], where xup is
//                the input upsampled by `up` with zeros and h the pre-padded Kaiser low-pass; fp64 taps and
//                accumulation, one rounding to fp32 per output
//   pcm16_peak   per-item max|y| (exact: a block max, then atomicMax on the non-negative float's bit pattern)
//   pcm16        the reference's float32 steps y / m1 * 0.6 / m2 * 32767 * 0.6, truncated to int16
//
// Ragged batches: each pass of up to RS_GROUP items rides in the kernel parameters (ItemPass), and a CTA's tile of
// consecutive outputs may straddle items.  An output depends on its own item only and comes from the same
// instructions in any batch, so a ragged batch is bitwise equal to each item run alone.
#include <algorithm>
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int RS_THREADS = 256, RS_PER_THREAD = 4, RS_TILE = RS_THREADS * RS_PER_THREAD;   // outputs per CTA
constexpr int RS_GROUP = 128;                                 // items per pass
constexpr long long RS_X_CAP_MAX = 32768;                     // staged input floats per CTA, at most
constexpr size_t RS_SMEM_MAX = 200 * 1024;                    // dynamic shared memory: taps (if they fit) + input
constexpr int PK_THREADS = 256, PK_TILE = PK_THREADS * 16;    // normaliser: elements per CTA

struct RsFilter {
  const double* taps;   // pre-padded filter, n_taps long
  long long n_taps, rm, x_cap;   // rm = outputs removed at the front; x_cap = staged input floats available
  int up, down, taps_in_smem;
};

// Output jl of an item of n inputs: t = (jl + rm) down, and the inputs it reads, [lo, hi] with 0 <= k = t - i up < n_taps.
// lo is clamped to n, so in_off + lo is a lower bound of every later output's reads even when this one reads none.
__device__ __forceinline__ void rs_span(long long jl, long long n, const RsFilter& f, long long& t, long long& lo,
                                        long long& hi) {
  t = (jl + f.rm) * f.down;
  hi = min(t / f.up, n - 1);
  const long long a = t - (f.n_taps - 1);
  lo = min(a > 0 ? (a + f.up - 1) / f.up : 0ll, n);
}

// grid ceil(outputs / RS_TILE), RS_THREADS threads, dynamic shared memory [taps (doubles) if taps_in_smem][x_cap floats].
__global__ void __launch_bounds__(RS_THREADS)
resample_kernel(const float* __restrict__ x, float* __restrict__ y, ItemPass<RS_GROUP> it, RsFilter f) {
  extern __shared__ __align__(16) unsigned char rs_smem[];
  double* hs = reinterpret_cast<double*>(rs_smem);
  float* xs = reinterpret_cast<float*>(rs_smem + (f.taps_in_smem ? f.n_taps * (long long)sizeof(double) : 0));
  __shared__ long long s_lo, s_hi;
  __shared__ int s_b0;
  const int tid = threadIdx.x;
  const long long j0 = it.out[0] + (long long)blockIdx.x * RS_TILE;
  const long long jend = min(j0 + RS_TILE, it.out[it.n]);
  if (tid == 0) {   // the tile's items and the input span its outputs read
    long long t, lo, hi;
    int b = item_of(it.out, j0);
    s_b0 = b;
    rs_span(j0 - it.out[b], it.in[b + 1] - it.in[b], f, t, lo, hi);
    s_lo = it.in[b] + lo;
    b = item_of(it.out, jend - 1, b);
    rs_span(jend - 1 - it.out[b], it.in[b + 1] - it.in[b], f, t, lo, hi);
    s_hi = it.in[b] + hi + 1;
  }
  __syncthreads();
  const long long x_lo = s_lo, span = s_hi - s_lo;
  const bool staged = span <= f.x_cap;   // else the inputs are read through L1 / L2
  if (staged)
    for (long long i = tid; i < span; i += RS_THREADS) xs[i] = __ldg(x + x_lo + i);
  if (f.taps_in_smem)
    for (long long k = tid; k < f.n_taps; k += RS_THREADS) hs[k] = __ldg(f.taps + k);
  __syncthreads();
  const double* hp = f.taps_in_smem ? hs : f.taps;
  const float* xp = staged ? xs : x;
  int b = s_b0;
#pragma unroll 1
  for (int r = 0; r < RS_PER_THREAD; ++r) {
    const long long j = j0 + tid + (long long)r * RS_THREADS;
    if (j >= jend) break;
    b = item_of(it.out, j, b);
    long long t, lo, hi;
    rs_span(j - it.out[b], it.in[b + 1] - it.in[b], f, t, lo, hi);
    const int cnt = (int)max(hi - lo + 1, 0ll);
    const float* xq = xp + (it.in[b] - (staged ? x_lo : 0ll) + hi);   // input hi, read backwards
    const double* hq = hp + (t - hi * f.up);                             // its tap, read forwards by `up`
    double acc = 0.0;
    for (int m = 0; m < cnt; ++m) acc = fma(hq[(long long)m * f.up], (double)xq[-m], acc);
    y[j] = __double2float_rn(acc);
  }
}

// The normaliser's items are [in[b], in[b+1]) of both y and out; peak points at the pass's first item.
// grid ceil(elements / PK_TILE): each CTA reduces max|y| of every item its tile touches, one block reduction each.
__global__ void __launch_bounds__(PK_THREADS)
pcm16_peak_kernel(const float* __restrict__ y, unsigned int* __restrict__ peak_bits, ItemPass<RS_GROUP> it) {
  __shared__ int s_b0, s_b1;
  __shared__ float red[PK_THREADS / 32];
  const int tid = threadIdx.x;
  const long long e0 = it.in[0] + (long long)blockIdx.x * PK_TILE, e1 = min(e0 + PK_TILE, it.in[it.n]);
  if (tid == 0) {
    s_b0 = item_of(it.in, e0);
    s_b1 = item_of(it.in, e1 - 1, s_b0);
  }
  __syncthreads();
  for (int b = s_b0; b <= s_b1; ++b) {
    const long long lo = max(e0, it.in[b]), hi = min(e1, it.in[b + 1]);
    float m = 0.f;
    for (long long e = lo + tid; e < hi; e += PK_THREADS) m = fmaxf(m, fabsf(__ldg(y + e)));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((tid & 31) == 0) red[tid >> 5] = m;
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < PK_THREADS / 32; ++w) m = fmaxf(m, red[w]);
      atomicMax(peak_bits + b, __float_as_uint(m));   // m >= +0: its bits order as the values do
    }
    __syncthreads();
  }
}

// prepare/preprocess_a.py:12-14 in float32, IEEE division and no contraction (every product feeds no add):
// v = y / m1 * 0.6; v = v / m2 * 32767 * 0.6 with m2 = max(0.01, max|y / m1 * 0.6|); int16 by truncation.
// max|y / m1| is m1 / m1 = 1 exactly (division is monotone), so m2 = max(0.01, 1 * 0.6) = 0.6f.  Silent items
// (m1 = 0) give zeros; the host skips them.
__global__ void __launch_bounds__(PK_THREADS)
pcm16_kernel(const float* __restrict__ y, const float* __restrict__ peak, int16_t* __restrict__ out, ItemPass<RS_GROUP> it) {
  __shared__ int s_b0;
  const int tid = threadIdx.x;
  const long long e0 = it.in[0] + (long long)blockIdx.x * PK_TILE, e1 = min(e0 + PK_TILE, it.in[it.n]);
  if (tid == 0) s_b0 = item_of(it.in, e0);
  __syncthreads();
  int b = s_b0;
  for (long long e = e0 + tid; e < e1; e += PK_THREADS) {
    b = item_of(it.in, e, b);
    const float m1 = peak[b];
    int16_t v16 = 0;
    if (m1 > 0.f) {
      const float m2 = fmaxf(0.01f, __fmul_rn(__fdiv_rn(m1, m1), 0.6f));
      float v = __fmul_rn(__fdiv_rn(__ldg(y + e), m1), 0.6f);
      v = __fmul_rn(__fmul_rn(__fdiv_rn(v, m2), 32767.f), 0.6f);
      v16 = (int16_t)__float2int_rz(v);
    }
    out[e] = v16;
  }
}

}  // namespace svcb

using namespace svcb;

extern "C" {

int svcb_resample_ragged(const float* x, const int64_t* in_offsets_host, int32_t B, int32_t up, int32_t down,
                         const double* taps, int64_t n_taps, int64_t pre_remove, float* y, svcb_stream stream) {
  static const char* who = "svcb_resample_ragged";
  if (!x || !y || !taps || !in_offsets_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  if (up < 1 || down < 1 || n_taps < 1 || pre_remove < 0) {
    set_error(std::string(who) + ": need up, down, n_taps >= 1 and pre_remove >= 0; got up " + std::to_string(up) +
              ", down " + std::to_string(down) + ", n_taps " + std::to_string(n_taps) + ", pre_remove " +
              std::to_string(pre_remove));
    return SVCB_E_BAD_SHAPE;
  }
  SVCB_TRY(check_ragged(who, in_offsets_host, B, 1, 1, "samples", nullptr));
  RsFilter f;
  f.taps = taps; f.n_taps = n_taps; f.rm = pre_remove; f.up = up; f.down = down;
  // worst input span of a tile: T down / up for its outputs plus a filter's reach at each end (DESIGN.md §5)
  f.x_cap = std::min(((long long)RS_TILE * down + 2 * n_taps) / up + 8, RS_X_CAP_MAX);
  f.taps_in_smem = (size_t)n_taps * sizeof(double) + (size_t)f.x_cap * sizeof(float) <= RS_SMEM_MAX;
  const size_t smem = (f.taps_in_smem ? (size_t)n_taps * sizeof(double) : 0) + (size_t)f.x_cap * sizeof(float);
  SVCB_CUDA_CHECK(cudaFuncSetAttribute(resample_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const double taps_per_out = (double)((n_taps + up - 1) / up);
  const auto out_len = [=](long long n) { return (n * up + down - 1) / down; };   // ceil(n up / down)
  return for_each_pass<RS_GROUP>(in_offsets_host, B, out_len, [&](const ItemPass<RS_GROUP>& it, int) -> int {
    const long long n_out = it.out[it.n] - it.out[0], n_in = it.in[it.n] - it.in[0];
    KernelScope ks("resample", s, 2.0 * taps_per_out * (double)n_out,
                   4.0 * (double)(n_in + n_out) + 8.0 * (double)n_taps);
    resample_kernel<<<(unsigned)((n_out + RS_TILE - 1) / RS_TILE), RS_THREADS, smem, s>>>(x, y, it, f);
    SVCB_LAUNCH_CHECK("resample");
    return SVCB_OK;
  });
}

int svcb_pcm16_normalise_ragged(const float* y, const int64_t* offsets_host, int32_t B, int16_t* out, float* peak,
                                svcb_stream stream) {
  static const char* who = "svcb_pcm16_normalise_ragged";
  if (!y || !out || !peak || !offsets_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, offsets_host, B, 1, 1, "samples", nullptr));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  SVCB_CUDA_CHECK(cudaMemsetAsync(peak, 0, sizeof(float) * (size_t)B, s));
  return for_each_pass<RS_GROUP>(offsets_host, B, [](long long n) { return n; }, [&](const ItemPass<RS_GROUP>& it, int g0) -> int {
    const long long n = it.in[it.n] - it.in[0];
    const unsigned grid = (unsigned)((n + PK_TILE - 1) / PK_TILE);
    {
      KernelScope ks("pcm16_peak", s, 0.0, 4.0 * (double)n);
      pcm16_peak_kernel<<<grid, PK_THREADS, 0, s>>>(y, reinterpret_cast<unsigned int*>(peak + g0), it);
      SVCB_LAUNCH_CHECK("pcm16_peak");
    }
    KernelScope ks("pcm16", s, 0.0, 6.0 * (double)n);
    pcm16_kernel<<<grid, PK_THREADS, 0, s>>>(y, peak + g0, out, it);
    SVCB_LAUNCH_CHECK("pcm16");
    return SVCB_OK;
  });
}

}  // extern "C"

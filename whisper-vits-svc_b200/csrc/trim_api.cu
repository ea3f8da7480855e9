// Trimming silence out of raw recordings (prepare/preprocess_trim.py:trim_silence, the second VCTK cleaning step) on
// the device: the silence decision of pydub's detect_silence as split_on_silence calls it (min_silence_len = 200,
// silence_thresh = -45 dBFS, seek_step = 1) for every window of a ragged batch of 16-bit mono clips.
//
//   L = round(1000 n / rate)            the clip's length in ms (len(AudioSegment)); ms m is frame fs(m) = int(m * (rate / 1000.0))
//   window i = 0 .. L - 200             frames [fs(i), fs(i + 200)), zero past n (pydub pads a slice that runs off the end)
//   silent iff (unsigned) sqrt(S_i / N_i) <= 10^(-45 / 20) * 32768, S_i the window's sum of squares and
//   N_i = fs(i + 200) - fs(i) its frame count, padding included (audioop.rms)
//
// A window's frames are exactly those of the 200 ms intervals [fs(m), fs(m + 1)) it spans.  So a CTA takes a tile of
// windows of one item, forms the integer sum of squares of each 1 ms interval the tile reaches (one warp per interval),
// prefixes them in shared memory and takes each window as a difference.  S_i is an integer below 2^53 (at most 0.2 rate
// frames of at most 2^30 each, rate <= 192 kHz), as every partial sum of audioop's double accumulation is, so that
// accumulation is exact and equals S_i; (double) S_i / N_i and sqrt are correctly rounded here and in glibc.  The flags
// are therefore audioop's decisions bit for bit, and an item's flags do not depend on the batch.
#include <cmath>
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int TRIM_WIN = 200;                        // min_silence_len, ms
constexpr int TRIM_THREADS = 256, TRIM_WARPS = TRIM_THREADS / 32;
constexpr int TRIM_IV = 2048;                        // 1 ms intervals per CTA
constexpr int TRIM_TILE = TRIM_IV - TRIM_WIN + 1;    // windows per CTA: they reach TRIM_IV intervals
constexpr int TRIM_GROUP = 128;                      // items per pass
constexpr int TRIM_MAX_RATE = 192000;                // keeps every window's sum of squares below 2^53

struct TrimRates {
  int r[TRIM_GROUP];
};

// L - 199 windows (none below 200 ms), L = Python's round(1000 * (n / rate)): both operations are correctly rounded
// and rint rounds a tie to even, as round does
inline long long trim_windows(long long n, int rate) {
  const long long L = (long long)std::rint(1000.0 * ((double)n / (double)rate));
  return std::max(L - TRIM_WIN + 1, 0ll);
}

// grid (tiles of the pass's longest item, items of the pass), TRIM_THREADS threads.  Item b has n_b samples at it.in[b]
// and its windows' flags at it.out[b]; CTA (t, b) takes its windows t * TRIM_TILE .. + TRIM_TILE - 1.
__global__ void __launch_bounds__(TRIM_THREADS)
trim_kernel(const int16_t* __restrict__ x, uint8_t* __restrict__ flags, ItemPass<TRIM_GROUP> it, TrimRates rt,
            double thresh) {
  __shared__ unsigned long long pre[TRIM_IV + 1];   // pre[k]: sum of squares of the tile's first k intervals
  __shared__ unsigned long long wsum[TRIM_WARPS];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, b = blockIdx.y;
  const long long W = it.out[b + 1] - it.out[b], i0 = (long long)blockIdx.x * TRIM_TILE;
  if (i0 >= W) return;
  const int nw = (int)min((long long)TRIM_TILE, W - i0), M = nw + TRIM_WIN - 1;
  const long long n = it.in[b + 1] - it.in[b];
  const int16_t* xb = x + it.in[b];
  const double fr = (double)rt.r[b] / 1000.0;
  auto fs = [fr](long long m) { return (long long)((double)m * fr); };

  for (int k = warp; k < M; k += TRIM_WARPS) {
    const long long f1 = min(fs(i0 + k + 1), n);
    unsigned long long s = 0;
    for (long long f = fs(i0 + k) + lane; f < f1; f += 32) {
      const int v = __ldg(xb + f);
      s += (unsigned)(v * v);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) pre[k + 1] = s;
  }
  __syncthreads();
  // inclusive scan of pre[1 .. M]: thread t sums its run of c intervals, the runs' totals are scanned, then each
  // thread rewrites its run as prefixes
  const int c = (M + TRIM_THREADS - 1) / TRIM_THREADS, k0 = min(tid * c, M), k1 = min(k0 + c, M);
  unsigned long long own = 0;
  for (int k = k0; k < k1; ++k) own += pre[k + 1];
  unsigned long long inc = own;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const unsigned long long v = __shfl_up_sync(0xffffffffu, inc, o);
    if (lane >= o) inc += v;
  }
  if (lane == 31) wsum[warp] = inc;
  __syncthreads();
  unsigned long long run = inc - own;
  for (int w = 0; w < warp; ++w) run += wsum[w];
  for (int k = k0; k < k1; ++k) {
    run += pre[k + 1];
    pre[k + 1] = run;
  }
  if (tid == 0) pre[0] = 0;
  __syncthreads();
  uint8_t* fb = flags + it.out[b];
  for (int j = tid; j < nw; j += TRIM_THREADS) {
    const long long i = i0 + j, N = fs(i + TRIM_WIN) - fs(i);
    const unsigned long long S = pre[j + TRIM_WIN] - pre[j];
    const unsigned rms = N > 0 ? (unsigned)sqrt((double)S / (double)N) : 0u;   // audioop.rms of no frames is 0
    fb[i] = (double)rms <= thresh ? 1 : 0;
  }
}

}  // namespace svcb

using namespace svcb;

extern "C" {

int svcb_trim_silence_ragged(const int16_t* x, const int64_t* offsets_host, const int32_t* rates_host, int32_t B,
                             uint8_t* flags, svcb_stream stream) {
  static const char* who = "svcb_trim_silence_ragged";
  if (!x || !flags || !offsets_host || !rates_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, offsets_host, B, 1, 0, "samples", nullptr));
  for (int b = 0; b < B; ++b) {
    if (rates_host[b] < 1 || rates_host[b] > TRIM_MAX_RATE) {
      set_error(std::string(who) + ": item " + std::to_string(b) + " has rate " + std::to_string(rates_host[b]) +
                "; need 1.." + std::to_string(TRIM_MAX_RATE) + " (a 200 ms sum of squares must stay below 2^53)");
      return SVCB_E_BAD_SHAPE;
    }
  }
  const double thresh = std::pow(10.0, -45.0 / 20.0) * 32768.0;   // pydub: db_to_float(-45) * max_possible_amplitude
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  int item = 0;   // for_each_pass asks for the items' output lengths in order
  return for_each_pass<TRIM_GROUP>(offsets_host, B, [&](long long n) { return trim_windows(n, rates_host[item++]); },
                                   [&](const ItemPass<TRIM_GROUP>& it, int g0) -> int {
    TrimRates rt;
    long long tiles = 0;
    for (int i = 0; i < it.n; ++i) {
      rt.r[i] = rates_host[g0 + i];
      tiles = std::max(tiles, (it.out[i + 1] - it.out[i] + TRIM_TILE - 1) / TRIM_TILE);
    }
    if (tiles == 0) return SVCB_OK;   // every item is shorter than 200 ms
    KernelScope ks("trim", s, 2.0 * (double)(it.in[it.n] - it.in[0]),
                   2.0 * (double)(it.in[it.n] - it.in[0]) + (double)(it.out[it.n] - it.out[0]));
    trim_kernel<<<dim3((unsigned)tiles, (unsigned)it.n), TRIM_THREADS, 0, s>>>(x, flags, it, rt, thresh);
    SVCB_LAUNCH_CHECK("trim");
    return SVCB_OK;
  });
}

}  // extern "C"

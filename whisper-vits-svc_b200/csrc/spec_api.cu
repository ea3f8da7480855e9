// Linear spectrogram of the training data (vits/spectrogram.py:spectrogram_torch with n_fft 1024, hop 320, win 1024,
// center=False, as prepare/preprocess_spec.py calls it) on the device.
//
//   spec   reflect pad (1024 - 320) / 2 = 352 samples at each end, periodic-Hann frames (hop 320), 513-bin magnitude
//          sqrt(re^2 + im^2 + 1e-6) by a direct fp32 DFT; ragged batch in one launch per pass of up to SPEC_GROUP
//          items, each item's [513, T_b] block bin-major in the output
//
// A frame's values depend on its own samples only and are computed by the same instructions whatever the batch, so a
// ragged batch is bitwise equal to each item run alone.
#include <algorithm>
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int SPEC_NFFT = kDftN, SPEC_HOP = 320, SPEC_PAD = (SPEC_NFFT - SPEC_HOP) / 2, SPEC_BINS = SPEC_NFFT / 2 + 1;
constexpr int SPEC_FT = 8;        // frames per CTA
constexpr int SPEC_GROUP = 128;   // items per pass

struct SpecItems {   // one pass: n items, samples [s_off[b], s_off[b+1]) -> frames [f_off[b], f_off[b+1])
  int n;
  long long s_off[SPEC_GROUP + 1];
  long long f_off[SPEC_GROUP + 1];
};

// grid ceil(frames / SPEC_FT), 256 threads: SPEC_FT consecutive frames of the pass (they may straddle items).
// out: item b's frame t, bin k at 513 f_off[b] + k T_b + t (frame offsets count from the batch's first item).
__global__ void __launch_bounds__(kDftThreads)
spec_kernel(const float* __restrict__ wav, float* __restrict__ out, SpecItems it) {
  __shared__ float2 tw[SPEC_NFFT];
  __shared__ __align__(16) float xw[SPEC_FT][SPEC_NFFT];   // windowed frames
  // per frame of the CTA: its item's first sample and length N, the frame's first (padded) sample, its item's frame
  // count T and its output offset 513 f_off[b] + t (-1 past the pass's last frame)
  __shared__ long long fr_x[SPEC_FT], fr_n[SPEC_FT], fr_s0[SPEC_FT], fr_t[SPEC_FT], fr_o[SPEC_FT];
  const int tid = threadIdx.x;
  const long long f0 = it.f_off[0] + (long long)blockIdx.x * SPEC_FT, fend = it.f_off[it.n];
  dft1024_twiddles(tw, tid);
  if (tid < SPEC_FT) {
    const long long gf = f0 + tid;
    fr_n[tid] = 0;
    fr_o[tid] = -1;
    if (gf < fend) {
      int b = 0;
      while (it.f_off[b + 1] <= gf) ++b;
      const long long t = gf - it.f_off[b];
      fr_x[tid] = it.s_off[b];
      fr_n[tid] = it.s_off[b + 1] - it.s_off[b];
      fr_s0[tid] = t * SPEC_HOP - SPEC_PAD;
      fr_t[tid] = it.f_off[b + 1] - it.f_off[b];
      fr_o[tid] = SPEC_BINS * it.f_off[b] + t;
    }
  }
  __syncthreads();
  for (int i = tid; i < SPEC_FT * SPEC_NFFT; i += kDftThreads) {
    const int fr = i / SPEC_NFFT, n = i - fr * SPEC_NFFT;
    const long long N = fr_n[fr];
    float v = 0.f;
    if (N > 0) {
      long long s = fr_s0[fr] + n;   // reflect padding; N > 352 keeps one reflection in range
      if (s < 0) s = -s;
      if (s >= N) s = 2 * (N - 1) - s;
      v = __ldg(wav + fr_x[fr] + s) * (0.5f - 0.5f * cospif(2.f * (float)n / (float)SPEC_NFFT));   // periodic Hann
    }
    xw[fr][n] = v;
  }
  __syncthreads();
  float mg[2][SPEC_FT];
  dft1024_bins<SPEC_FT>(tw, xw, tid, mg, [](float re, float im) { return sqrtf(re * re + im * im + 1e-6f); });
  float nyq = 0.f;   // bin 512: imaginary part 0
  if (tid < SPEC_FT) {
    const float a = dft1024_nyquist(xw[tid]);
    nyq = sqrtf(a * a + 1e-6f);
  }
  __syncthreads();
  float* mag = &xw[0][0];   // [bin][frame]
#pragma unroll
  for (int f = 0; f < SPEC_FT; ++f) { mag[tid * SPEC_FT + f] = mg[0][f]; mag[(tid + 256) * SPEC_FT + f] = mg[1][f]; }
  if (tid < SPEC_FT) mag[(SPEC_BINS - 1) * SPEC_FT + tid] = nyq;
  __syncthreads();
  // consecutive threads -> consecutive frames of a bin: runs of up to SPEC_FT contiguous floats of an item's row
  for (int i = tid; i < SPEC_BINS * SPEC_FT; i += kDftThreads) {
    const int k = i / SPEC_FT, f = i - k * SPEC_FT;
    const long long ob = fr_o[f];
    if (ob >= 0) out[ob + (long long)k * fr_t[f]] = mag[i];
  }
}

}  // namespace svcb

using namespace svcb;

extern "C" {

int svcb_linear_spec_ragged(const float* audio, const int64_t* sample_offsets_host, int32_t B, float* out, void* scratch,
                            size_t scratch_bytes, svcb_stream stream) {
  (void)scratch; (void)scratch_bytes;
  if (!audio || !out || !sample_offsets_host || B <= 0) { set_error("svcb_linear_spec_ragged: bad argument"); return SVCB_E_BAD_SHAPE; }
  if (sample_offsets_host[0] < 0) { set_error("svcb_linear_spec_ragged: negative sample offset"); return SVCB_E_BAD_SHAPE; }
  for (int b = 0; b < B; ++b)
    if (sample_offsets_host[b + 1] - sample_offsets_host[b] <= SPEC_PAD) {
      set_error("svcb_linear_spec_ragged: item " + std::to_string(b) + " has " +
                std::to_string(sample_offsets_host[b + 1] - sample_offsets_host[b]) +
                " samples; the reflect padding of 352 needs more than 352");
      return SVCB_E_BAD_SHAPE;
    }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  long long frame = 0;
  for (int g0 = 0; g0 < B; g0 += SPEC_GROUP) {
    SpecItems it;
    it.n = std::min(SPEC_GROUP, B - g0);
    it.f_off[0] = frame;
    for (int i = 0; i <= it.n; ++i) it.s_off[i] = sample_offsets_host[g0 + i];
    for (int i = 0; i < it.n; ++i) it.f_off[i + 1] = it.f_off[i] + (it.s_off[i + 1] - it.s_off[i]) / SPEC_HOP;
    const long long F = it.f_off[it.n] - it.f_off[0];
    frame = it.f_off[it.n];
    KernelScope ks("spec", s, (double)F * 4.0 * SPEC_NFFT * SPEC_BINS,
                   4.0 * ((double)(it.s_off[it.n] - it.s_off[0]) + (double)SPEC_BINS * F));
    spec_kernel<<<(unsigned)((F + SPEC_FT - 1) / SPEC_FT), kDftThreads, 0, s>>>(audio, out, it);
    SVCB_LAUNCH_CHECK("spec");
  }
  return SVCB_OK;
}

}  // extern "C"

// Linear spectrogram of the training data (vits/spectrogram.py:spectrogram_torch with n_fft 1024, hop 320, win 1024,
// center=False, as prepare/preprocess_spec.py calls it) on the device.
//
//   spec   reflect pad (1024 - 320) / 2 = 352 samples at each end, periodic-Hann frames (hop 320), 513-bin magnitude
//          sqrt(re^2 + im^2 + 1e-6) by a direct fp32 DFT; ragged batch in one launch per pass of up to SPEC_GROUP
//          items, each item's [513, T_b] block bin-major in the output
//
// A frame's values depend on its own samples only and are computed by the same instructions whatever the batch, so a
// ragged batch is bitwise equal to each item run alone.
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int SPEC_NFFT = kDftN, SPEC_HOP = 320, SPEC_PAD = (SPEC_NFFT - SPEC_HOP) / 2, SPEC_BINS = SPEC_NFFT / 2 + 1;
constexpr int SPEC_FT = 8;        // frames per CTA
constexpr int SPEC_GROUP = 128;   // items per pass

// grid ceil(frames / SPEC_FT), 256 threads: SPEC_FT consecutive frames of the pass (they may straddle items).
// it: samples in, frames out.  out: item b's frame t, bin k at 513 out[b] + k T_b + t.
__global__ void __launch_bounds__(kDftThreads)
spec_kernel(const float* __restrict__ wav, float* __restrict__ out, ItemPass<SPEC_GROUP> it) {
  __shared__ float2 tw[SPEC_NFFT];
  __shared__ __align__(16) float xw[SPEC_FT][SPEC_NFFT];   // windowed frames
  // per frame of the CTA: its item's first sample and length N, the frame's first (padded) sample, its item's frame
  // count T and its output offset 513 out[b] + t (-1 past the pass's last frame)
  __shared__ long long fr_x[SPEC_FT], fr_n[SPEC_FT], fr_s0[SPEC_FT], fr_t[SPEC_FT], fr_o[SPEC_FT];
  const int tid = threadIdx.x;
  const long long f0 = it.out[0] + (long long)blockIdx.x * SPEC_FT, fend = it.out[it.n];
  dft1024_twiddles(tw, tid);
  if (tid < SPEC_FT) {
    const long long gf = f0 + tid;
    fr_n[tid] = 0;
    fr_o[tid] = -1;
    if (gf < fend) {
      const int b = item_of(it.out, gf);
      const long long t = gf - it.out[b];
      fr_x[tid] = it.in[b];
      fr_n[tid] = it.in[b + 1] - it.in[b];
      fr_s0[tid] = t * SPEC_HOP - SPEC_PAD;
      fr_t[tid] = it.out[b + 1] - it.out[b];
      fr_o[tid] = SPEC_BINS * it.out[b] + t;
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
  static const char* who = "svcb_linear_spec_ragged";
  if (!audio || !out || !sample_offsets_host) { set_error(std::string(who) + ": bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, sample_offsets_host, B, 1, SPEC_PAD + 1, "samples", "the reflect padding is 352 samples"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return for_each_pass<SPEC_GROUP>(sample_offsets_host, B, [](long long n) { return n / SPEC_HOP; },
                                   [&](const ItemPass<SPEC_GROUP>& it, int) -> int {
    const long long F = it.out[it.n] - it.out[0];
    KernelScope ks("spec", s, (double)F * 4.0 * SPEC_NFFT * SPEC_BINS,
                   4.0 * ((double)(it.in[it.n] - it.in[0]) + (double)SPEC_BINS * F));
    spec_kernel<<<(unsigned)((F + SPEC_FT - 1) / SPEC_FT), kDftThreads, 0, s>>>(audio, out, it);
    SVCB_LAUNCH_CHECK("spec");
    return SVCB_OK;
  });
}

}  // extern "C"

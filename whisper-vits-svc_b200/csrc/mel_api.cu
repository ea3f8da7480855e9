// Log-mel spectrogram of the trainer's validation pass (vits_extend/stft.py:TacotronSTFT.mel_spectrogram with
// n_fft 1024, hop 320, win 1024, center=False, as vits_extend/validation.py calls it) on the device.
//
//   mel   reflect pad 352 samples at each end of every row of a padded batch [B, L], periodic-Hann frames (hop 320),
//         513-bin magnitude sqrt(re^2 + im^2 + 1e-9) by a direct fp32 DFT, the mel projection mel_basis [n_mels, 513]
//         accumulated bin by bin in ascending order from each filter's first to its last non-zero bin, then
//         ln(max(x, 1e-5)); out [B, n_mels, L / 320]
//
// A frame's values depend on its own row's samples only and are computed by the same instructions whatever B and the
// row's position, so each item is bitwise that of a lone call.
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int MEL_NFFT = kDftN, MEL_HOP = 320, MEL_PAD = (MEL_NFFT - MEL_HOP) / 2, MEL_BINS = MEL_NFFT / 2 + 1;
constexpr int MEL_FT = 8;          // frames per CTA
constexpr int MEL_MAX_MELS = 128;  // mel bands the kernel supports
constexpr int MEL_LD = MEL_BINS + 3;

// T = L / 320.  grid (ceil(T / MEL_FT), B), 256 threads: frames MEL_FT blockIdx.x .. + MEL_FT of row blockIdx.y.
__global__ void __launch_bounds__(kDftThreads)
tacotron_mel_kernel(const float* __restrict__ audio, long long L, long long T, const float* __restrict__ fb, int n_mels,
                    float* __restrict__ out) {
  __shared__ float2 tw[MEL_NFFT];
  __shared__ __align__(16) float xw[MEL_FT][MEL_NFFT];   // windowed frames, then the magnitudes [MEL_FT][MEL_LD]
  __shared__ int lo[MEL_MAX_MELS], hi[MEL_MAX_MELS];     // each filter's non-zero bins [lo, hi)
  const int tid = threadIdx.x, b = blockIdx.y;
  const long long t0 = (long long)blockIdx.x * MEL_FT;
  const float* x = audio + (long long)b * L;
  dft1024_twiddles(tw, tid);
  for (int i = tid; i < MEL_FT * MEL_NFFT; i += kDftThreads) {
    const int fr = i / MEL_NFFT, n = i - fr * MEL_NFFT;
    const long long t = t0 + fr;
    float v = 0.f;
    if (t < T) {
      long long s = t * MEL_HOP - MEL_PAD + n;   // reflect padding; L > 352 keeps one reflection in range
      if (s < 0) s = -s;
      if (s >= L) s = 2 * (L - 1) - s;
      v = __ldg(x + s) * (0.5f - 0.5f * cospif(2.f * (float)n / (float)MEL_NFFT));   // periodic Hann
    }
    xw[fr][n] = v;
  }
  __syncthreads();
  float mg[2][MEL_FT];
  dft1024_bins<MEL_FT>(tw, xw, tid, mg, [](float re, float im) { return sqrtf(re * re + im * im + 1e-9f); });
  float nyq = 0.f;   // bin 512: imaginary part 0
  if (tid < MEL_FT) {
    const float a = dft1024_nyquist(xw[tid]);
    nyq = sqrtf(a * a + 1e-9f);
  }
  __syncthreads();
  float* mag = &xw[0][0];
#pragma unroll
  for (int f = 0; f < MEL_FT; ++f) { mag[f * MEL_LD + tid] = mg[0][f]; mag[f * MEL_LD + tid + 256] = mg[1][f]; }
  if (tid < MEL_FT) mag[tid * MEL_LD + 512] = nyq;
  for (int m = tid; m < n_mels; m += kDftThreads) {
    const float* fm = fb + (long long)m * MEL_BINS;
    int a = 0, e = MEL_BINS;
    while (a < MEL_BINS && __ldg(fm + a) == 0.f) ++a;
    while (e > a && __ldg(fm + e - 1) == 0.f) --e;
    lo[m] = a;
    hi[m] = e;
  }
  __syncthreads();
  // consecutive threads -> consecutive frames of a band: runs of up to MEL_FT contiguous floats of a row of out
  for (int i = tid; i < MEL_FT * n_mels; i += kDftThreads) {
    const int m = i / MEL_FT, f = i - m * MEL_FT;
    const long long t = t0 + f;
    if (t >= T) continue;
    const float* fm = fb + (long long)m * MEL_BINS;
    const float* mf = mag + f * MEL_LD;
    float a = 0.f;
    for (int k = lo[m]; k < hi[m]; ++k) a = fmaf(__ldg(fm + k), mf[k], a);
    out[((long long)b * n_mels + m) * T + t] = logf(fmaxf(a, 1e-5f));
  }
}

}  // namespace svcb

using namespace svcb;

extern "C" {

int svcb_tacotron_mel(const float* audio, int32_t B, int64_t L, const float* mel_basis, int32_t n_mels, float* mel,
                      svcb_stream stream) {
  static const char* who = "svcb_tacotron_mel";
  if (!audio || !mel_basis || !mel) { set_error(std::string(who) + ": bad argument"); return SVCB_E_BAD_SHAPE; }
  if (B <= 0 || B > 65535) {
    set_error(std::string(who) + ": B = " + std::to_string(B) + "; need 1..65535");
    return SVCB_E_BAD_SHAPE;
  }
  if (L <= MEL_PAD) {
    set_error(std::string(who) + ": L = " + std::to_string(L) + " samples; the reflect padding needs more than 352");
    return SVCB_E_BAD_SHAPE;
  }
  if (n_mels < 1 || n_mels > MEL_MAX_MELS) {
    set_error(std::string(who) + ": n_mels = " + std::to_string(n_mels) + "; the kernel supports 1..128");
    return SVCB_E_UNSUPPORTED;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const long long T = L / MEL_HOP;
  const double F = (double)B * T;
  KernelScope ks("tacotron_mel", s, F * 4.0 * MEL_NFFT * MEL_BINS + F * 2.0 * n_mels * MEL_BINS,
                 4.0 * ((double)B * L + (double)n_mels * MEL_BINS + (double)n_mels * F));
  tacotron_mel_kernel<<<dim3((unsigned)((T + MEL_FT - 1) / MEL_FT), (unsigned)B), kDftThreads, 0, s>>>(audio, L, T,
                                                                                                      mel_basis, n_mels, mel);
  SVCB_LAUNCH_CHECK("tacotron_mel");
  return SVCB_OK;
}

}  // extern "C"

// Log-mel front end of the PPG extractor on the device (SURVEY.md §8f row 1).
//
// Replaces whisper.audio.log_mel_spectrogram (whisper/audio.py:68-100) for a batch of equal-length
// chunks: Hann-windowed STFT (n_fft 400, hop 160, centre = reflect padding of 200 samples, the last
// frame dropped), squared magnitude, mel projection, log10 of the 1e-10 clamp, per-chunk `max - 8`
// floor, (x + 4) / 4, and the extractor's additive mel noise (whisper/inference.py:46,58) in the
// same pass.  Three launches: max reset, power+mel+log (with a per-chunk atomic max), finalize.
// Ragged batches (lens != null): item b is its first lens[b] samples (F_b = lens[b] / 160 frames), reflect-padded
// at its own end, floored at the max over its own frames; its frames >= F_b are written as exact zeros, which is
// the zero padding the encoder's conv1 expects there.  Every frame is computed as a lone run of the item computes it.
//
// The 400-point DFT is evaluated directly in fp32 against a 400-entry twiddle table in shared
// memory (index k*n mod 400 advanced incrementally): 2 x 400 x 201 MACs per frame = 15 GFLOP for
// 16 x 30 s, well under a millisecond of FMA time — an FFT would not pay for its shuffles here.
#include <cstdint>

#include "common.cuh"

namespace svcb {

constexpr int LM_NFFT = 400, LM_HOP = 160, LM_BINS = 201, LM_FT = 8;  // frames per CTA

__device__ __forceinline__ unsigned lm_order(float f) {  // float -> uint with the same ordering
  const unsigned u = __float_as_uint(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float lm_unorder(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

__global__ void logmel_reset_kernel(unsigned* mx, int B) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < B) mx[i] = 0u;  // below every ordered float
}

// grid (ceil(F / LM_FT), B), 256 threads.  out[b][m][f] = log10(max(mel power, 1e-10)).
__global__ void __launch_bounds__(256)
logmel_power_kernel(const float* __restrict__ audio, const float* __restrict__ filt, float* __restrict__ out,
                    unsigned* __restrict__ mx, int N, int F, int n_mels, const int* __restrict__ lens) {
  __shared__ float tw_c[LM_NFFT], tw_s[LM_NFFT];
  __shared__ float xw[LM_FT][LM_NFFT];
  __shared__ float pw[LM_FT][LM_BINS + 3];
  __shared__ float red[8];
  const int tid = threadIdx.x, b = blockIdx.y, f0 = blockIdx.x * LM_FT;
  const float* ab = audio + (long long)b * N;
  const int Nb = lens ? __ldg(lens + b) : N, Fb = Nb / LM_HOP;
  for (int n = tid; n < LM_NFFT; n += 256) {
    float s, c;
    sincospif(2.f * (float)n / (float)LM_NFFT, &s, &c);
    tw_c[n] = c; tw_s[n] = s;
  }
  for (int i = tid; i < LM_FT * LM_NFFT; i += 256) {
    const int fr = i / LM_NFFT, n = i - fr * LM_NFFT;
    const int f = f0 + fr;
    float v = 0.f;
    if (f < Fb) {
      int t = f * LM_HOP + n - LM_NFFT / 2;           // centre=True: reflect padding (torch.stft)
      if (t < 0) t = -t;
      if (t >= Nb) t = 2 * (Nb - 1) - t;
      t = min(max(t, 0), Nb - 1);
      // periodic Hann window (torch.hann_window): 0.5 - 0.5 cos(2 pi n / 400)
      v = __ldg(ab + t) * (0.5f - 0.5f * cospif(2.f * (float)n / (float)LM_NFFT));
    }
    xw[fr][n] = v;
  }
  __syncthreads();
  for (int i = tid; i < LM_FT * LM_BINS; i += 256) {
    const int fr = i / LM_BINS, k = i - fr * LM_BINS;
    float re = 0.f, im = 0.f;
    int idx = 0;
#pragma unroll 8
    for (int n = 0; n < LM_NFFT; ++n) {
      const float x = xw[fr][n];
      re = fmaf(x, tw_c[idx], re);
      im = fmaf(x, tw_s[idx], im);
      idx += k;
      if (idx >= LM_NFFT) idx -= LM_NFFT;
    }
    pw[fr][k] = re * re + im * im;
  }
  __syncthreads();
  float lmax = -1e30f;
  for (int i = tid; i < LM_FT * n_mels; i += 256) {
    const int m = i / LM_FT, fr = i - m * LM_FT;   // consecutive threads -> consecutive frames (stores)
    const int f = f0 + fr;
    if (f >= F) continue;
    if (f >= Fb) { out[((long long)b * n_mels + m) * F + f] = 0.f; continue; }
    const float* fm = filt + (long long)m * LM_BINS;
    float a = 0.f;
    for (int k = 0; k < LM_BINS; ++k) a = fmaf(__ldg(fm + k), pw[fr][k], a);
    const float lg = log10f(fmaxf(a, 1e-10f));
    out[((long long)b * n_mels + m) * F + f] = lg;
    lmax = fmaxf(lmax, lg);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) lmax = fmaxf(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
  if ((tid & 31) == 0) red[tid >> 5] = lmax;
  __syncthreads();
  if (tid == 0) {
    float v = red[0];
    for (int w = 1; w < 8; ++w) v = fmaxf(v, red[w]);
    if (v > -1e29f) atomicMax(mx + b, lm_order(v));
  }
}

__global__ void __launch_bounds__(256)
logmel_finalize_kernel(float* __restrict__ out, const unsigned* __restrict__ mx, const float* __restrict__ noise,
                       float gain, long long per_item, int F, const int* __restrict__ lens) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  const int b = blockIdx.y;
  if (i >= per_item) return;
  const long long off = (long long)b * per_item + i;
  if (lens && (int)(i % F) >= __ldg(lens + b) / LM_HOP) { out[off] = 0.f; return; }   // past the item's frames
  const float floor_v = lm_unorder(mx[b]) - 8.0f;
  float v = (fmaxf(out[off], floor_v) + 4.0f) / 4.0f;
  if (noise) v = fmaf(__ldg(noise + off), gain, v);
  out[off] = v;
}

int launch_log_mel(const float* audio, const float* filt, const float* noise, float gain, float* out,
                   unsigned* scratch, int B, int N, int n_mels, cudaStream_t s, const int* lens) {
  const int F = N / LM_HOP;
  if (B <= 0 || F <= 0) return SVCB_OK;
  if (N < LM_NFFT / 2 + 1) { set_error("log_mel: chunk shorter than the reflect padding"); return SVCB_E_BAD_SHAPE; }
  {
    KernelScope ks("logmel_reset", s, 0.0, 4.0 * B);
    logmel_reset_kernel<<<(B + 255) / 256, 256, 0, s>>>(scratch, B);
    SVCB_LAUNCH_CHECK("logmel_reset");
  }
  {
    dim3 grid((F + LM_FT - 1) / LM_FT, B);
    KernelScope ks("logmel_power", s, (double)B * F * (4.0 * LM_NFFT * LM_BINS + 2.0 * LM_BINS * n_mels),
                   4.0 * B * ((double)N + (double)n_mels * F));
    logmel_power_kernel<<<grid, 256, 0, s>>>(audio, filt, out, scratch, N, F, n_mels, lens);
    SVCB_LAUNCH_CHECK("logmel_power");
  }
  {
    const long long per_item = (long long)n_mels * F;
    dim3 grid((unsigned)((per_item + 255) / 256), B);
    KernelScope ks("logmel_finalize", s, 0.0, (noise ? 12.0 : 8.0) * B * (double)per_item);
    logmel_finalize_kernel<<<grid, 256, 0, s>>>(out, scratch, noise, gain, per_item, F, lens);
    SVCB_LAUNCH_CHECK("logmel_finalize");
  }
  return SVCB_OK;
}

}  // namespace svcb

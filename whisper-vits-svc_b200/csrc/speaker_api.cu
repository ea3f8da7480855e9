// LSTM speaker encoder (speaker/models/lstm.py, LSTMSpeakerEncoder with projection: 3 x LSTM(768) -> Linear(768, 256))
// and its mel front end (speaker/utils/audio.py AudioProcessor.melspectrogram) on the device.
//
//   spk_mel         pre-emphasis, reflect-centred periodic-Hann frames (n_fft 1024, hop 256), 513-bin magnitude by a
//                   direct fp32 DFT, 80-band mel, 20 log10 - ref, symmetric clipped normalisation; ragged batch in one pass
//   spk_gather0     compute_embedding's 10 windows of min(250, T) frames per item (offsets int(linspace(0, T - L, 10)))
//                   as fp32 rows m = t * Mp + r, r = item * 10 + window; then ivf_pack's [x_hi | x_lo | x_hi] image
//   gemm_tc         per layer G = X . W_ih^T + (b_ih + b_hh) over every (step, window) row, and the 768 -> 256
//                   projection (every step of layers 0 and 1), both bf16x3 by K-tripling (csrc/whisper_gemm.cu,
//                   epilogue 2 without residual)
//   spk_lstm_rec    the recurrence: one cooperative launch per layer, 128 CTAs x 6 hidden units (N = 24 gate columns),
//                   W_hh slice (bf16 hi / lo) resident in shared memory, h_{t-1} streamed by bulk copies, grid barrier
//                   between steps
//   spk_gather_last the last layer's h at each window's own last step, so its projection runs over 10 rows per item
//   spk_finish      L2-normalise each window's last-step projection and average the 10 windows of each item
// Timing (svcb_timing): spk_pack, spk_gemm_ih and spk_gemm_proj bracket launch_ivf_pack / launch_gemm_tc, which book
// the same launch again under their own names (ivf_pack, whisper_gemm_tc); a sum over the report counts those twice.
//
// Rows of every item are computed by the same instructions whatever the batch, so a ragged batch is bitwise equal to
// each item run alone.  A window shorter than the batch's longest runs on past its own end (the LSTM is causal); its
// embedding is taken at its own last step.
#include <cooperative_groups.h>
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdint>
#include <memory>
#include <type_traits>

#include "common.cuh"
#include "tc.cuh"

namespace cg = cooperative_groups;

namespace svcb {

constexpr int SPK_NFFT = 1024, SPK_HOP = 256, SPK_BINS = 513, SPK_MELS = 80, SPK_FT = 8;   // frames per mel CTA
constexpr int SPK_H = 768, SPK_P = 256, SPK_G4 = 4 * SPK_H, SPK_LAYERS = 3;
constexpr int SPK_WIN = 250, SPK_NWIN = 10;
constexpr int SPK_CTAS = 128, SPK_UPC = SPK_H / SPK_CTAS, SPK_NC = 4 * SPK_UPC;   // 6 units, 24 gate columns per CTA
constexpr int SPK_HK = 3 * SPK_H;            // K of the h image [h_hi | h_lo | h_hi] (the projection's A operand)
constexpr int SPK_REC_KT = 2 * SPK_H / 64;   // k-tiles the recurrence reads: [h_hi | h_lo]
constexpr int SPK_GROUP = 64;                // items per pass of svcb_speaker_embed / svcb_speaker_mel
constexpr int SPK_MAXMP = (SPK_GROUP * SPK_NWIN + 127) / 128 * 128;
constexpr int SPK_K0 = 128;                  // layer 0's K (80 mels) padded to whole 64-wide k-tiles
constexpr int REC_STAGES = 4, REC_LD = 28, REC_THREADS = 288;
constexpr uint32_t REC_W_BYTES = 2u * (SPK_H / 8) * SPK_NC * 16;   // W_hh hi + lo, [k/8][24][8] each: 73728
constexpr uint32_t REC_A_BYTES = 128u * 64 * 2;                    // one 128-row k-tile of the h image
constexpr size_t REC_SMEM = REC_W_BYTES + REC_STAGES * REC_A_BYTES + 2 * 64 * REC_LD * 4 + SPK_MAXMP * SPK_UPC * 4;

struct SpkMelItems {   // one pass: n items, samples [s_off[b], s_off[b+1]) -> mel rows [f_off[b], f_off[b+1])
  int n;
  long long s_off[SPK_GROUP + 1];
  long long f_off[SPK_GROUP + 1];
};
struct SpkItems {      // one pass: n items, mel rows [f_off[b], f_off[b+1])
  int n;
  long long f_off[SPK_GROUP + 1];
};

// element offset of (m, k) in a gemm_tc tile image with KT k-tiles per 128-row tile (csrc/whisper_gemm.cu)
__host__ __device__ inline size_t spk_img_off(size_t m, int k, int KT) {
  return ((m >> 7) * KT + (k >> 6)) * (128 * 64) + (size_t)((k & 63) >> 3) * (128 * 8) + (m & 127) * 8 + (k & 7);
}

// compute_embedding (lstm.py:86-92): int(np.linspace(0, S, 10)[w]) with numpy's float64 arithmetic (step = S / 9,
// y = w * step, the last point set to S exactly)
__device__ __forceinline__ long long spk_win_offset(long long S, int w) {
  if (w == SPK_NWIN - 1) return S;
  return (long long)((double)w * ((double)S / (double)(SPK_NWIN - 1)));
}

__device__ __forceinline__ void fence_proxy_async_global() { asm volatile("fence.proxy.async.global;" ::: "memory"); }

// ----------------------------------------------------------------------------------------------------------- mel
// grid ceil(frames / SPK_FT), 256 threads: SPK_FT consecutive frames of the pass (they may straddle items).
// audio = {preemphasis, ref_level_db, min_level_db, max_norm}
__global__ void __launch_bounds__(256)
spk_mel_kernel(const float* __restrict__ wav, const float* __restrict__ fb, const float* __restrict__ audio,
               float* __restrict__ out, SpkMelItems it) {
  __shared__ float2 tw[SPK_NFFT];
  __shared__ __align__(16) float xw[SPK_FT][SPK_NFFT];   // windowed frames, then the magnitudes [SPK_FT][SPK_BINS + 3]
  const int tid = threadIdx.x;
  const long long f0 = it.f_off[0] + (long long)blockIdx.x * SPK_FT, fend = it.f_off[it.n];
  const float pre = __ldg(audio);
  for (int n = tid; n < SPK_NFFT; n += 256) {
    float s, c;
    sincospif(2.f * (float)n / (float)SPK_NFFT, &s, &c);
    tw[n] = make_float2(c, s);
  }
  for (int i = tid; i < SPK_FT * SPK_NFFT; i += 256) {
    const int fr = i / SPK_NFFT, n = i - fr * SPK_NFFT;
    const long long gf = f0 + fr;
    float v = 0.f;
    if (gf < fend) {
      int b = 0;
      while (it.f_off[b + 1] <= gf) ++b;
      const long long N = it.s_off[b + 1] - it.s_off[b];
      const float* x = wav + it.s_off[b];
      long long s = (gf - it.f_off[b]) * SPK_HOP + n - SPK_NFFT / 2;   // center=True, reflect padding
      if (s < 0) s = -s;
      if (s >= N) s = 2 * (N - 1) - s;
      // lfilter([1, -pre], [1]) with x[-1] = 0, applied before the padding
      const float y = __ldg(x + s) - pre * (s > 0 ? __ldg(x + s - 1) : 0.f);
      v = y * (0.5f - 0.5f * cospif(2.f * (float)n / (float)SPK_NFFT));   // periodic Hann
    }
    xw[fr][n] = v;
  }
  __syncthreads();
  // bins tid and tid + 256 for all SPK_FT frames: one twiddle load feeds 2 x SPK_FT FMAs; twiddle index k n mod 1024
  float mg[2][SPK_FT];
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int k = tid + 256 * h;
    float re[SPK_FT], im[SPK_FT];
#pragma unroll
    for (int f = 0; f < SPK_FT; ++f) { re[f] = 0.f; im[f] = 0.f; }
#pragma unroll 2
    for (int n = 0; n < SPK_NFFT; n += 4) {
      const float2 t0 = tw[(k * n) & (SPK_NFFT - 1)], t1 = tw[(k * (n + 1)) & (SPK_NFFT - 1)];
      const float2 t2 = tw[(k * (n + 2)) & (SPK_NFFT - 1)], t3 = tw[(k * (n + 3)) & (SPK_NFFT - 1)];
#pragma unroll
      for (int f = 0; f < SPK_FT; ++f) {
        const float4 x = *reinterpret_cast<const float4*>(&xw[f][n]);
        re[f] = fmaf(x.x, t0.x, re[f]); im[f] = fmaf(x.x, t0.y, im[f]);
        re[f] = fmaf(x.y, t1.x, re[f]); im[f] = fmaf(x.y, t1.y, im[f]);
        re[f] = fmaf(x.z, t2.x, re[f]); im[f] = fmaf(x.z, t2.y, im[f]);
        re[f] = fmaf(x.w, t3.x, re[f]); im[f] = fmaf(x.w, t3.y, im[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < SPK_FT; ++f) mg[h][f] = sqrtf(re[f] * re[f] + im[f] * im[f]);
  }
  float nyq = 0.f;   // bin 512: the alternating sum
  if (tid < SPK_FT) {
    for (int n = 0; n < SPK_NFFT; n += 2) nyq += xw[tid][n] - xw[tid][n + 1];
    nyq = fabsf(nyq);
  }
  __syncthreads();
  float* mag = &xw[0][0];
  constexpr int MLD = SPK_BINS + 3;
#pragma unroll
  for (int f = 0; f < SPK_FT; ++f) { mag[f * MLD + tid] = mg[0][f]; mag[f * MLD + tid + 256] = mg[1][f]; }
  if (tid < SPK_FT) mag[tid * MLD + 512] = nyq;
  __syncthreads();
  const float ref = __ldg(audio + 1), mn = __ldg(audio + 2), mx = __ldg(audio + 3);
  for (int i = tid; i < SPK_FT * SPK_MELS; i += 256) {
    const int fr = i / SPK_MELS, m = i - fr * SPK_MELS;   // consecutive threads -> consecutive mels (stores)
    const long long gf = f0 + fr;
    if (gf >= fend) continue;
    const float* fm = fb + m * SPK_BINS;
    float a = 0.f;
    for (int k = 0; k < SPK_BINS; ++k) a = fmaf(__ldg(fm + k), mag[fr * MLD + k], a);
    float S = 20.f * log10f(fmaxf(1e-5f, a)) - ref;      // _amp_to_db (audio.py:480-489), normalize (:378-386)
    S = (S - mn) / (-mn);
    S = (2.f * mx) * S - mx;
    out[gf * SPK_MELS + m] = fminf(fmaxf(S, -mx), mx);
  }
}

// --------------------------------------------------------------------------------------------- windows -> rows
// x[m][0..128) for m = t * Mp + r: the mel frame of window r at step t (zero past the window's end, for k >= 80 and
// for pad rows r >= 10 n)
__global__ void __launch_bounds__(256)
spk_gather0_kernel(const float* __restrict__ mel, float* __restrict__ x, SpkItems it, int Mp, size_t R) {
  const size_t idx = (size_t)blockIdx.x * 256 + threadIdx.x;
  if (idx >= R * (SPK_K0 / 4)) return;
  const size_t m = idx / (SPK_K0 / 4);
  const int q = (int)(idx - m * (SPK_K0 / 4));
  const int t = (int)(m / Mp), r = (int)(m - (size_t)t * Mp);
  float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
  if (r < SPK_NWIN * it.n && q < SPK_MELS / 4) {
    const int b = r / SPK_NWIN, w = r - b * SPK_NWIN;
    const long long T = it.f_off[b + 1] - it.f_off[b], L = T < SPK_WIN ? T : SPK_WIN;
    if (t < L) v = __ldg(reinterpret_cast<const float4*>(mel + (it.f_off[b] + spk_win_offset(T - L, w) + t) * SPK_MELS) + q);
  }
  reinterpret_cast<float4*>(x + m * SPK_K0)[q] = v;
}

// ------------------------------------------------------------------------------------------------- recurrence
// 128 CTAs (cooperative launch), CTA c owns hidden units 6c .. 6c+5 with their 4 gates: gate column n = 4 u + gate of
// the CTA's 24 (pack order: speaker_infer.py:pack_speaker).  Per step t:
//   producer thread   bulk-copies the 128-row k-tiles of h_{t-1} = [h_hi | h_lo] (24 per row tile) through a ring
//   2 warpgroups      64 rows each: acc = h_hi W_hi + h_hi W_lo + h_lo W_hi (wgmma m64n24k16, W_hh resident),
//                     + G[t] (input product and both biases), gate math in fp32, c in shared memory,
//                     h_t -> the h image (next step's operand and the projection's A operand)
// then fence.proxy.async (generic h stores before other SMs' bulk reads) and a grid barrier.
__global__ void __launch_bounds__(REC_THREADS, 1)
spk_lstm_rec_kernel(const __nv_bfloat16* __restrict__ whh, const float* __restrict__ G, __nv_bfloat16* himg, int Mp, int Lw) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar_full[REC_STAGES], bar_empty[REC_STAGES], bar_w;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, warp = tid >> 5, cta = blockIdx.x, nrt = Mp / 128;
  uint8_t* ring = smem + REC_W_BYTES;
  float* strips = reinterpret_cast<float*>(ring + REC_STAGES * REC_A_BYTES);
  float* cst = strips + 2 * 64 * REC_LD;   // c [Mp][6]
  constexpr int KT = SPK_HK / 64;
  if (tid == 0) {
    for (int s = 0; s < REC_STAGES; ++s) { tc::mbar_init(&bar_full[s], 1); tc::mbar_init(&bar_empty[s], 2); }
    tc::mbar_init(&bar_w, 1);
    tc::fence_barrier_init();
  }
  for (int i = tid; i < Mp * SPK_UPC; i += REC_THREADS) cst[i] = 0.f;
  __syncthreads();
  if (tid == 0) {
    tc::mbar_arrive_expect_tx(&bar_w, REC_W_BYTES);
    tc::bulk_g2s(smem, reinterpret_cast<const uint8_t*>(whh) + (size_t)cta * REC_W_BYTES, REC_W_BYTES, &bar_w);
  }
  // the warpgroups wait for W_hh whatever the step count: no CTA may exit with the copy still in flight (Lw == 1)
  if (warp < 8) tc::mbar_wait(&bar_w, 0);
  int kc = 0;   // k-tile counter (ring position), advanced identically by the producer and the warpgroups
  for (int t = 0; t < Lw; ++t) {
    if (warp == 8) {
      if (t > 0 && (tid & 31) == 0) {
        fence_proxy_async_global();
        const size_t m0 = (size_t)(t - 1) * Mp;
        for (int rt = 0; rt < nrt; ++rt)
          for (int kt = 0; kt < SPK_REC_KT; ++kt, ++kc) {
            const int st = kc % REC_STAGES;
            if (kc >= REC_STAGES) tc::mbar_wait(&bar_empty[st], (uint32_t)(((kc / REC_STAGES) - 1) & 1));
            tc::mbar_arrive_expect_tx(&bar_full[st], REC_A_BYTES);
            tc::bulk_g2s(ring + st * REC_A_BYTES, himg + spk_img_off(m0 + rt * 128, kt * 64, KT), REC_A_BYTES, &bar_full[st]);
          }
      }
    } else {
      const int wg = warp >> 2, tt = tid & 127;
      float* strip = strips + wg * 64 * REC_LD;
      const uint32_t w0 = tc::smem_u32(smem), w_lo = w0 + REC_W_BYTES / 2;
      for (int rt = 0; rt < nrt; ++rt) {
        float acc[12];
#pragma unroll
        for (int i = 0; i < 12; ++i) acc[i] = 0.f;
        if (t > 0) {
          // k-tile kt of [h_hi | h_lo]: h_hi . (W_hi, W_lo) for the first half, h_lo . W_hi for the second
          auto ktile = [&](int kt, auto lo_too) {
            const int st = kc % REC_STAGES;
            tc::mbar_wait(&bar_full[st], (uint32_t)((kc / REC_STAGES) & 1));
            const uint32_t a0 = tc::smem_u32(ring + st * REC_A_BYTES) + (uint32_t)wg * 64u * 16u;
            const int kb = decltype(lo_too)::value ? kt : kt - SPK_REC_KT / 2;   // k-tile inside the segment
            tc::wg_fence();
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
              const uint64_t ad = tc::smem_desc(a0 + kk * 4096u, 2048u);
              const uint32_t wo = (uint32_t)(kb * 8 + kk * 2) * (SPK_NC * 16u);
              tc::Wg<24, 0>::ss(acc, ad, tc::smem_desc(w0 + wo, SPK_NC * 16u), 1u);
              if constexpr (decltype(lo_too)::value) tc::Wg<24, 0>::ss(acc, ad, tc::smem_desc(w_lo + wo, SPK_NC * 16u), 1u);
            }
            tc::wg_commit();
            tc::wg_wait<1>();
            if (kt > 0 && tt == 0) tc::mbar_arrive(&bar_empty[(kc - 1) % REC_STAGES]);
            ++kc;
          };
          for (int kt = 0; kt < SPK_REC_KT / 2; ++kt) ktile(kt, std::true_type{});
          for (int kt = SPK_REC_KT / 2; kt < SPK_REC_KT; ++kt) ktile(kt, std::false_type{});
          tc::wg_wait<0>();
          tc::wg_hold(acc);
          if (tt == 0) tc::mbar_arrive(&bar_empty[(kc - 1) % REC_STAGES]);
        }
        tc::named_sync(1 + wg, 128);   // the previous row tile's strip has been read
        tc::acc_to_smem<24>(acc, strip, REC_LD, 0, 3);
        tc::named_sync(1 + wg, 128);
        for (int i = tt; i < 64 * (SPK_UPC / 2); i += 128) {   // (row, unit pair)
          const int rl = i / (SPK_UPC / 2), p = i - rl * (SPK_UPC / 2);
          const int row = rt * 128 + wg * 64 + rl;
          const float4* gp = reinterpret_cast<const float4*>(G + ((size_t)t * Mp + row) * SPK_G4 + cta * SPK_NC + 8 * p);
          const float4 ga = __ldg(gp), gb = __ldg(gp + 1);
          const float* sp = strip + rl * REC_LD + 8 * p;
          const float z[8] = {sp[0] + ga.x, sp[1] + ga.y, sp[2] + ga.z, sp[3] + ga.w,
                              sp[4] + gb.x, sp[5] + gb.y, sp[6] + gb.z, sp[7] + gb.w};
          float h[2];
#pragma unroll
          for (int u = 0; u < 2; ++u) {   // gates i, f, g, o (nn.LSTM order)
            const float ig = 1.f / (1.f + expf(-z[4 * u])), fg = 1.f / (1.f + expf(-z[4 * u + 1]));
            const float gg = tanhf(z[4 * u + 2]), og = 1.f / (1.f + expf(-z[4 * u + 3]));
            float& c = cst[row * SPK_UPC + 2 * p + u];
            c = fg * c + ig * gg;
            h[u] = og * tanhf(c);
          }
          __nv_bfloat162 hi = __floats2bfloat162_rn(h[0], h[1]);
          const float2 hif = __bfloat1622float2(hi);
          __nv_bfloat162 lo = __floats2bfloat162_rn(h[0] - hif.x, h[1] - hif.y);
          const size_t m = (size_t)t * Mp + row;
          const int k = cta * SPK_UPC + 2 * p;
          *reinterpret_cast<__nv_bfloat162*>(himg + spk_img_off(m, k, KT)) = hi;
          *reinterpret_cast<__nv_bfloat162*>(himg + spk_img_off(m, SPK_H + k, KT)) = lo;
          *reinterpret_cast<__nv_bfloat162*>(himg + spk_img_off(m, 2 * SPK_H + k, KT)) = hi;
        }
      }
    }
    fence_proxy_async_global();
    grid.sync();
  }
}

// ------------------------------------------------------------------------------------------------------ finish
// The last layer's h at each window's own last step: row r of a [Mp][2304] h image (pad rows: step Lw - 1), so the last
// projection runs over Mp rows instead of Lw x Mp.  Thread = one 16-byte octet.
__global__ void __launch_bounds__(256)
spk_gather_last_kernel(const __nv_bfloat16* __restrict__ himg, __nv_bfloat16* __restrict__ last, SpkItems it, int Mp, int Lw) {
  constexpr int KT = SPK_HK / 64, NO = SPK_HK / 8;
  const int idx = blockIdx.x * 256 + threadIdx.x;
  if (idx >= Mp * NO) return;
  const int o = idx / Mp, r = idx - o * Mp;   // consecutive threads -> consecutive rows: contiguous in the tile image
  long long t = Lw - 1;
  if (r < SPK_NWIN * it.n) {
    const int b = r / SPK_NWIN;
    const long long T = it.f_off[b + 1] - it.f_off[b];
    t = (T < SPK_WIN ? T : SPK_WIN) - 1;
  }
  *reinterpret_cast<uint4*>(last + spk_img_off(r, 8 * o, KT)) =
      __ldg(reinterpret_cast<const uint4*>(himg + spk_img_off((size_t)t * Mp + r, 8 * o, KT)));
}

// one CTA per item, thread = embedding dim: F.normalize(d[:, -1]) per window (lstm.py:69-74), then the mean of the 10.
// proj: the last layer's projection of the gathered last steps, [Mp][256]
__global__ void __launch_bounds__(256)
spk_finish_kernel(const float* __restrict__ proj, float* __restrict__ out, float* __restrict__ wout, SpkItems it) {
  __shared__ float red[8];
  const int b = blockIdx.x, j = threadIdx.x, lane = j & 31, warp = j >> 5;
  float acc = 0.f;
  for (int w = 0; w < SPK_NWIN; ++w) {
    const int r = b * SPK_NWIN + w;
    const float v = __ldg(proj + (size_t)r * SPK_P + j);
    float s = v * v;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) red[warp] = s;
    __syncthreads();
    float tot = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) tot += red[i];
    __syncthreads();
    const float e = v / fmaxf(sqrtf(tot), 1e-12f);
    if (wout) wout[(size_t)r * SPK_P + j] = e;
    acc += e;
  }
  out[(size_t)b * SPK_P + j] = acc / (float)SPK_NWIN;
}

static size_t align256s(size_t x) { return (x + 255) & ~(size_t)255; }

struct SpkLayout {
  size_t img, G, himg, proj, last, total;
};
// R = Lw * Mp rows; the layer-0 rows (R x 128 fp32) live in the projection buffer
static SpkLayout spk_layout(size_t R, int Mp) {
  SpkLayout L;
  size_t off = 0;
  L.img = off; off = align256s(off + R * 3 * SPK_P * 2);
  L.G = off; off = align256s(off + R * SPK_G4 * 4);
  L.himg = off; off = align256s(off + R * SPK_HK * 2);
  L.proj = off; off = align256s(off + R * SPK_P * 4);
  L.last = off; off = align256s(off + (size_t)Mp * SPK_HK * 2);
  L.total = off;
  return L;
}
static int spk_mp(int nb) { return (nb * SPK_NWIN + 127) / 128 * 128; }

static DevSmemCache g_rec_smem;

}  // namespace svcb

using namespace svcb;

struct svcb_speaker {
  const float* fb = nullptr;      // mel basis [80][513]
  const float* audio = nullptr;   // {preemphasis, ref_level_db, min_level_db, max_norm}
  struct Layer {
    const void* wih = nullptr;    // bf16 tile image [3072][3 Kin] = [W_hi | W_hi | W_lo], rows in gate-column order
    const float* b = nullptr;     // b_ih + b_hh [3072], same order
    const void* whh = nullptr;    // bf16 [128 CTAs][hi, lo][96][24][8]
    const void* wproj = nullptr;  // bf16 tile image [256][2304]
  } L[SPK_LAYERS];
};

extern "C" {

int svcb_speaker_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                        svcb_speaker** out) {
  if (!dev_blob || !table_host || !out) { set_error("svcb_speaker_create: bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_blob_device(dev_blob));
  // the recurrence's grid barrier needs all 128 CTAs resident at once (one per SM)
  int dev = 0, coop = 0, per_sm = 0;
  SVCB_CUDA_CHECK(cudaGetDevice(&dev));
  SVCB_CUDA_CHECK(cudaDeviceGetAttribute(&coop, cudaDevAttrCooperativeLaunch, dev));
  SVCB_CUDA_CHECK(ensure_dyn_smem(spk_lstm_rec_kernel, REC_SMEM, g_rec_smem));
  SVCB_CUDA_CHECK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, spk_lstm_rec_kernel, REC_THREADS, REC_SMEM));
  if (!coop || per_sm * device_sm_count() < SPK_CTAS) {
    set_error("svcb_speaker_create: the LSTM recurrence needs a cooperative launch of 128 co-resident CTAs");
    return SVCB_E_UNSUPPORTED;
  }
  BlobTensors t;
  SVCB_TRY(t.read(dev_blob, blob_bytes, table_host, n_entries));
  auto sp = std::make_unique<svcb_speaker>();
  sp->fb = t.get("spk.mel_fb", (uint64_t)SPK_MELS * SPK_BINS);
  sp->audio = t.get("spk.audio", 4);
  for (int l = 0; l < SPK_LAYERS; ++l) {
    const std::string p = "spk.l" + std::to_string(l);
    const uint64_t kin = l == 0 ? SPK_K0 : SPK_P;
    sp->L[l].wih = t.get(p + ".wih", (uint64_t)SPK_G4 * 3 * kin / 2);
    sp->L[l].b = t.get(p + ".b", SPK_G4);
    sp->L[l].whh = t.get(p + ".whh", (uint64_t)SPK_CTAS * REC_W_BYTES / 4);
    sp->L[l].wproj = t.get(p + ".wproj", (uint64_t)SPK_P * SPK_HK / 2);
  }
  SVCB_TRY(t.status("speaker blob"));
  *out = sp.release();
  return SVCB_OK;
}

void svcb_speaker_destroy(svcb_speaker* sp) { delete sp; }

int32_t svcb_speaker_frames(int64_t n_samples) { return n_samples < 0 ? 0 : (int32_t)(1 + n_samples / SPK_HOP); }

size_t svcb_speaker_workspace_bytes(const svcb_speaker* sp, int32_t B, int64_t total_samples) {
  if (!sp || B <= 0 || total_samples <= 0) return 0;
  const int Lw = std::min<int64_t>(SPK_WIN, svcb_speaker_frames(total_samples));
  const int Mp = spk_mp(std::min(B, SPK_GROUP));
  return spk_layout((size_t)Lw * Mp, Mp).total;
}

int svcb_speaker_mel(const svcb_speaker* sp, const float* wav, const int64_t* sample_offsets_host, int32_t B, float* mel_out,
                     void* ws, size_t ws_bytes, svcb_stream stream) {
  (void)ws; (void)ws_bytes;
  if (!sp || !wav || !mel_out || !sample_offsets_host || B < 0) { set_error("svcb_speaker_mel: bad argument"); return SVCB_E_BAD_SHAPE; }
  for (int b = 0; b < B; ++b)
    if (sample_offsets_host[b] < 0 || sample_offsets_host[b + 1] - sample_offsets_host[b] <= SPK_NFFT / 2) {
      set_error("svcb_speaker_mel: item " + std::to_string(b) + " has " +
                std::to_string(sample_offsets_host[b + 1] - sample_offsets_host[b]) +
                " samples; the reflect-padded STFT needs more than 512");
      return SVCB_E_BAD_SHAPE;
    }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  long long frame = 0;
  for (int g0 = 0; g0 < B; g0 += SPK_GROUP) {
    SpkMelItems it;
    it.n = std::min(SPK_GROUP, B - g0);
    it.f_off[0] = frame;
    for (int i = 0; i <= it.n; ++i) it.s_off[i] = sample_offsets_host[g0 + i];
    for (int i = 0; i < it.n; ++i) it.f_off[i + 1] = it.f_off[i] + svcb_speaker_frames(it.s_off[i + 1] - it.s_off[i]);
    const long long F = it.f_off[it.n] - it.f_off[0];
    frame = it.f_off[it.n];
    KernelScope ks("spk_mel", s, (double)F * (4.0 * SPK_NFFT * SPK_BINS + 2.0 * SPK_BINS * SPK_MELS),
                   4.0 * ((double)(it.s_off[it.n] - it.s_off[0]) + (double)SPK_MELS * F));
    spk_mel_kernel<<<(unsigned)((F + SPK_FT - 1) / SPK_FT), 256, 0, s>>>(wav, sp->fb, sp->audio, mel_out, it);
    SVCB_LAUNCH_CHECK("spk_mel");
  }
  return SVCB_OK;
}

int svcb_speaker_embed(const svcb_speaker* sp, const float* mel, const int64_t* frame_offsets_host, int32_t B, float* out,
                       float* window_out, void* ws, size_t ws_bytes, svcb_stream stream) {
  if (!sp || !mel || !out || !frame_offsets_host || B < 0) { set_error("svcb_speaker_embed: bad argument"); return SVCB_E_BAD_SHAPE; }
  if ((uintptr_t)mel & 15) { set_error("svcb_speaker_embed: mel must be 16-byte aligned"); return SVCB_E_BAD_ALIGN; }
  for (int b = 0; b < B; ++b)
    if (frame_offsets_host[b] < 0 || frame_offsets_host[b + 1] <= frame_offsets_host[b]) {
      set_error("svcb_speaker_embed: item " + std::to_string(b) + " has no mel frames");
      return SVCB_E_BAD_SHAPE;
    }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(ws);
  for (int g0 = 0; g0 < B; g0 += SPK_GROUP) {
    SpkItems it;
    it.n = std::min(SPK_GROUP, B - g0);
    int Lw = 0;
    for (int i = 0; i <= it.n; ++i) it.f_off[i] = frame_offsets_host[g0 + i];
    for (int i = 0; i < it.n; ++i) Lw = std::max<int>(Lw, (int)std::min<long long>(SPK_WIN, it.f_off[i + 1] - it.f_off[i]));
    const int Mp = spk_mp(it.n), rows = SPK_NWIN * it.n;
    const size_t R = (size_t)Lw * Mp;
    const SpkLayout L = spk_layout(R, Mp);
    if (!ws || ((uintptr_t)ws & 255) || ws_bytes < L.total) { set_error("speaker workspace too small or misaligned"); return SVCB_E_WORKSPACE; }
    void* img = base + L.img;
    float* G = reinterpret_cast<float*>(base + L.G);
    __nv_bfloat16* himg = reinterpret_cast<__nv_bfloat16*>(base + L.himg);
    float* proj = reinterpret_cast<float*>(base + L.proj);
    __nv_bfloat16* last = reinterpret_cast<__nv_bfloat16*>(base + L.last);
    const double steps = (double)rows * Lw;   // algorithmic (window, step) pairs
    {
      KernelScope ks("spk_gather0", s, 0.0, 4.0 * steps * SPK_MELS + 4.0 * R * SPK_K0);
      spk_gather0_kernel<<<(unsigned)((R * (SPK_K0 / 4) + 255) / 256), 256, 0, s>>>(mel, proj, it, Mp, R);
      SVCB_LAUNCH_CHECK("spk_gather0");
    }
    for (int l = 0; l < SPK_LAYERS; ++l) {
      const int kin = l == 0 ? SPK_K0 : SPK_P, kin_alg = l == 0 ? SPK_MELS : SPK_P;
      {
        KernelScope ks("spk_pack", s, 0.0, 4.0 * R * kin + 6.0 * R * kin);
        SVCB_TRY(launch_ivf_pack(proj, img, (int)R, kin, s));
      }
      {
        KernelScope ks("spk_gemm_ih", s, 2.0 * steps * kin_alg * SPK_G4, 6.0 * R * kin + 6.0 * SPK_G4 * kin + 4.0 * R * SPK_G4);
        SVCB_TRY(launch_gemm_tc(img, sp->L[l].wih, sp->L[l].b, G, nullptr, (int)R, SPK_G4, 3 * kin, EPI_RESID_F32, s));
      }
      {
        KernelScope ks("spk_lstm_rec", s, 2.0 * steps * SPK_H * SPK_G4,
                       (double)SPK_CTAS * REC_W_BYTES + 4.0 * R * SPK_G4 + 6.0 * R * SPK_H);
        const __nv_bfloat16* whh = static_cast<const __nv_bfloat16*>(sp->L[l].whh);
        const float* Gc = G;
        int mp = Mp, lw = Lw;
        void* args[] = {(void*)&whh, (void*)&Gc, (void*)&himg, (void*)&mp, (void*)&lw};
        SVCB_CUDA_CHECK(ensure_dyn_smem(spk_lstm_rec_kernel, REC_SMEM, g_rec_smem));
        SVCB_CUDA_CHECK(cudaLaunchCooperativeKernel((const void*)spk_lstm_rec_kernel, dim3(SPK_CTAS), dim3(REC_THREADS), args,
                                                    REC_SMEM, s));
        SVCB_LAUNCH_CHECK("spk_lstm_rec");
      }
      if (l + 1 < SPK_LAYERS) {   // every step feeds the next layer
        KernelScope ks("spk_gemm_proj", s, 2.0 * steps * SPK_H * SPK_P, 6.0 * R * SPK_H + 6.0 * SPK_P * SPK_H + 4.0 * R * SPK_P);
        SVCB_TRY(launch_gemm_tc(himg, sp->L[l].wproj, nullptr, proj, nullptr, (int)R, SPK_P, SPK_HK, EPI_RESID_F32, s));
      } else {                    // the embedding reads each window's last step only
        {
          KernelScope ks("spk_gather_last", s, 0.0, 4.0 * Mp * SPK_HK);
          spk_gather_last_kernel<<<(Mp * (SPK_HK / 8) + 255) / 256, 256, 0, s>>>(himg, last, it, Mp, Lw);
          SVCB_LAUNCH_CHECK("spk_gather_last");
        }
        KernelScope ks("spk_gemm_proj", s, 2.0 * rows * SPK_H * SPK_P, 6.0 * Mp * SPK_H + 6.0 * SPK_P * SPK_H + 4.0 * Mp * SPK_P);
        SVCB_TRY(launch_gemm_tc(last, sp->L[l].wproj, nullptr, proj, nullptr, Mp, SPK_P, SPK_HK, EPI_RESID_F32, s));
      }
    }
    {
      KernelScope ks("spk_finish", s, 0.0, 4.0 * rows * SPK_P * (window_out ? 2.0 : 1.0) + 4.0 * it.n * SPK_P);
      spk_finish_kernel<<<it.n, 256, 0, s>>>(proj, out + (size_t)g0 * SPK_P, window_out ? window_out + (size_t)g0 * SPK_NWIN * SPK_P : nullptr,
                                             it);
      SVCB_LAUNCH_CHECK("spk_finish");
    }
  }
  return SVCB_OK;
}

}  // extern "C"

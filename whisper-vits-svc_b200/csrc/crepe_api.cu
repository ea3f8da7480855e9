// CREPE pitch extractor (crepe/model.py, crepe/core.py, crepe/decode.py) on the device, for a ragged batch of 16 kHz
// recordings.  From the framing on the batch is flat: frame rows are independent, so nothing is padded per item until
// the decoder.
//
//   crepe_frame      one CTA per frame: gather 1024 samples around f * hop from the zero-padded item (+ 0.001 * noise),
//                    subtract the mean, divide by max(1e-10, unbiased std) -> frames [F, 1024] fp32
//   full capacity, bf16 operands on wgmma, fp32 accumulation, frames in chunks sized from the workspace:
//   crepe_conv1_tc   Toeplitz GEMM straight off the 1532-sample padded frame (K = 512, stride 4): even and odd output
//                    positions are two GEMMs over the frame and its copy shifted by 4 samples (row q of either is the
//                    16-byte-aligned window at 8 q), whose max is the pool; a CTA keeps its 128 x 512 weight tile in
//                    shared memory across frames
//   crepe_conv_tc    conv2 .. conv6 as implicit GEMMs: the input is an "image" [Cin/8][R][8] per group of G frames with
//                    row (p + 31) * G + g for padded position p of frame g, so that tap j of the 64-tap window is the
//                    operand descriptor advanced by j * G rows and a 64-row tile is P * G = 64 valid outputs whatever
//                    the layer (G = 1, 1, 2, 4, 8); bulk copies fetch an image's channel chunk once per 64 taps and the
//                    weight stages (32 KB) through a three-stage mbarrier ring
//                    epilogue, in registers: + bias, ReLU, BN scale / shift (eval), max over the position pair (a lane
//                    shuffle, or the fragment's other half when G = 8), bf16 into the next layer's image
//   tiny capacity:   crepe_tiny, one CTA per frame, all six layers in fp32 on CUDA cores out of shared memory
//   crepe_classify   features [F, 4 * C6] (position, channel) x W^T + b, sigmoid, bins outside [39, 299) = -inf
//   crepe_decode     one CTA per (item, segment of <= 512 frames): fp32 softmax, dense 360-state Viterbi in fp64 (first
//                    maximum on ties, log(x + FLT_MIN) as librosa takes them), back-pointers in the workspace, back-track,
//                    bins -> cents + dither -> Hz, periodicity = probs[t][bin]
#include <cfloat>
#include <cmath>
#include <memory>
#include <string>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

constexpr int CR_WIN = 1024, CR_BINS = 360, CR_TAPS = 64, CR_PADL = 31;
constexpr int CR_BIN_LO = 39, CR_BIN_HI = 299;   // frequency_to_bins(50), frequency_to_bins(1000, ceil)
constexpr int CR_SEG_MAX = 512;
constexpr int CR_GROUP = 128;                    // items per pass
constexpr int CR_CHUNK_MAX = 4096, CR_CHUNK_ALIGN = 16;   // frames per chunk: two units of G = 8 per conv6 CTA

__host__ __device__ constexpr int cr_rows(int G, int UM) { return (64 * UM + 63 * G + 7) / 8 * 8; }

// ------------------------------------------------------------------------------------------------------- framing
__global__ void __launch_bounds__(256)
crepe_frame_kernel(const float* __restrict__ wav, const float* __restrict__ noise, ItemPass<CR_GROUP> it, long long f0, int hop,
                   float* __restrict__ frames) {
  __shared__ double red[8];
  __shared__ float stat;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long gf = f0 + blockIdx.x;
  const int b = item_of(it.out, gf);
  const long long s0 = it.in[b], n = it.in[b + 1] - s0, c = (gf - it.out[b]) * hop - CR_WIN / 2;
  float x[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const long long s = c + tid + 256 * k;
    float v = 0.f;
    if (s >= 0 && s < n) {
      v = __ldg(wav + s0 + s);
      if (noise) v = __fadd_rn(v, __fmul_rn(__ldg(noise + s0 + s), 0.001f));
    }
    x[k] = v;
  }
  auto block_sum = [&](double a) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
    __syncthreads();
    if (lane == 0) red[warp] = a;
    __syncthreads();
    double t = 0.0;
    for (int w = 0; w < 8; ++w) t += red[w];
    return t;
  };
  const float mean = (float)(block_sum((double)x[0] + x[1] + x[2] + x[3]) / CR_WIN);
  double q = 0.0;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    x[k] -= mean;
    q += (double)x[k] * x[k];
  }
  const double ss = block_sum(q), sc = block_sum((double)x[0] + x[1] + x[2] + x[3]);
  if (tid == 0) stat = fmaxf(1e-10f, (float)sqrt(fmax(ss - sc * sc / CR_WIN, 0.0) / (CR_WIN - 1)));
  __syncthreads();
#pragma unroll
  for (int k = 0; k < 4; ++k) frames[(size_t)blockIdx.x * CR_WIN + tid + 256 * k] = x[k] / stat;
}

// ------------------------------------------------------------------------------------------------- epilogue pieces
struct CrepeEpi {
  const float *bias, *scale, *shift;   // [Cout]
  __nv_bfloat16* img;                  // the next layer's images, or null for the last layer
  float* feat;                         // last layer: [frames][Pq * Cout] in (position, channel) order
  int Cout, Gn, Rn, Pq;                // next image: frames per group, rows; pooled positions per frame
};
__device__ __forceinline__ void crepe_store2(const CrepeEpi& E, long long frame, int q, int col, float v0, float v1) {
  if (E.img) {
    const long long un = frame / E.Gn;
    const int row = (q + CR_PADL) * E.Gn + (int)(frame - un * E.Gn);
    __nv_bfloat16* p = E.img + ((size_t)un * E.Cout + (col & ~7)) * E.Rn + (size_t)row * 8 + (col & 7);
    *reinterpret_cast<__nv_bfloat162*>(p) = __floats2bfloat162_rn(v0, v1);
  } else {
    *reinterpret_cast<float2*>(E.feat + ((size_t)frame * E.Pq + q) * E.Cout + col) = make_float2(v0, v1);
  }
}

// ------------------------------------------------------------------------------------------------- conv1 (full)
constexpr int C1_K = 512, C1_XLEN = 1536, C1_PAD = 254;
constexpr size_t C1_SMEM = (size_t)128 * C1_K * 2 + 2 * C1_XLEN * 2 + 16;
// grid (Cout / 128, frame lanes), 256 threads: warpgroup w owns pooled positions 64 w .. 64 w + 63 of each frame
__global__ void __launch_bounds__(256, 1)
crepe_conv1_tc_kernel(const float* __restrict__ frames, const __nv_bfloat16* __restrict__ wimg, CrepeEpi E, int nframes) {
  extern __shared__ __align__(128) uint8_t smem[];
  __nv_bfloat16* Bs = reinterpret_cast<__nv_bfloat16*>(smem);   // [64 k-octets][128][8]
  __nv_bfloat16* xe = Bs + 128 * C1_K;                          // the padded frame
  __nv_bfloat16* xo = xe + C1_XLEN;                             // ... shifted left by 4 samples
  uint64_t* bar = reinterpret_cast<uint64_t*>(xo + C1_XLEN);
  const int tid = threadIdx.x, wg = tid >> 7, l = tid & 31, w = (tid & 127) >> 5;
  if (tid == 0) {
    tc::mbar_init(bar, 1);
    tc::fence_barrier_init();
  }
  for (int i = tid; i < 2 * C1_XLEN; i += 256) xe[i] = __float2bfloat16(0.f);
  __syncthreads();
  if (tid == 0) {
    tc::mbar_arrive_expect_tx(bar, 128 * C1_K * 2);
    const uint8_t* src = reinterpret_cast<const uint8_t*>(wimg) + (size_t)blockIdx.x * 128 * C1_K * 2;
    for (int c = 0; c < 4; ++c) tc::bulk_g2s(smem + c * 32768, src + c * 32768, 32768, bar);
  }
  tc::mbar_wait(bar, 0);
  const int n0 = blockIdx.x * 128;
  const uint32_t b_addr = tc::smem_u32(Bs);
  for (int f = blockIdx.y; f < nframes; f += gridDim.y) {
    for (int i = tid; i < CR_WIN; i += 256) {
      const __nv_bfloat16 v = __float2bfloat16(__ldg(frames + (size_t)f * CR_WIN + i));
      xe[C1_PAD + i] = v;
      xo[C1_PAD - 4 + i] = v;
    }
    tc::fence_proxy_async_smem();
    __syncthreads();
    float de[64], dd[64];
    // A row q, K chunk c = the 16 bytes at sample 8 (q + c): rows and K chunks both advance by 16 bytes
    const uint32_t ae = tc::smem_u32(xe) + wg * 64 * 16, ao = tc::smem_u32(xo) + wg * 64 * 16;
    tc::wg_fence();
#pragma unroll 4
    for (int s = 0; s < C1_K / 16; ++s) {
      const uint64_t db = tc::smem_desc(b_addr + 2 * s * 2048, 2048);
      tc::Wg<128, 0>::ss(de, tc::smem_desc(ae + 32 * s, 16), db, s ? 1u : 0u);
      tc::Wg<128, 0>::ss(dd, tc::smem_desc(ao + 32 * s, 16), db, s ? 1u : 0u);
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_hold(de);
    tc::wg_hold(dd);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int col = n0 + 8 * i + 2 * (l & 3);
      const float b0 = __ldg(E.bias + col), b1 = __ldg(E.bias + col + 1), s0 = __ldg(E.scale + col), s1 = __ldg(E.scale + col + 1);
      const float h0 = __ldg(E.shift + col), h1 = __ldg(E.shift + col + 1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int q = 64 * wg + 16 * w + (l >> 2) + 8 * h;
        const float v0 = fmaxf(fmaf(fmaxf(de[4 * i + 2 * h] + b0, 0.f), s0, h0), fmaf(fmaxf(dd[4 * i + 2 * h] + b0, 0.f), s0, h0));
        const float v1 = fmaxf(fmaf(fmaxf(de[4 * i + 2 * h + 1] + b1, 0.f), s1, h1), fmaf(fmaxf(dd[4 * i + 2 * h + 1] + b1, 0.f), s1, h1));
        crepe_store2(E, f, q, col, v0, v1);
      }
    }
    __syncthreads();   // the frame buffers are rewritten next
  }
}

// ------------------------------------------------------------------------------------------------- conv2 .. conv6 (full)
constexpr int CV_STAGES = 3, CV_BSTAGE = 32768;
template <int G, int UM, int CK>
constexpr size_t cv_smem() { return (size_t)CV_STAGES * CV_BSTAGE + 2 * 2 * (size_t)CK * cr_rows(G, UM) * 2 + 64; }

// grid (units / 2, Cout / 128), 256 threads: warpgroup w owns unit 2 * blockIdx.x + w (a group of G frames; UM m64 tiles)
template <int CIN, int G, int UM, int CK>
__global__ void __launch_bounds__(256, 1)
crepe_conv_tc_kernel(const __nv_bfloat16* __restrict__ img, const __nv_bfloat16* __restrict__ wimg, CrepeEpi E) {
  constexpr int R = cr_rows(G, UM), TG = 128 / CK, NCC = CIN / CK, NTG = CR_TAPS / TG, NIT = NCC * NTG;
  constexpr uint32_t A_UNIT = CK * R * 2;
  extern __shared__ __align__(128) uint8_t smem[];
  uint8_t* Bs = smem;                                    // [stage][TG taps][CK / 8][128][8]
  uint8_t* As = smem + CV_STAGES * CV_BSTAGE;            // [2][unit of the CTA][CK / 8][R][8]
  uint64_t* full = reinterpret_cast<uint64_t*>(As + 4 * A_UNIT);
  const int tid = threadIdx.x, wg = tid >> 7, l = tid & 31, w = (tid & 127) >> 5;
  const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(wimg) + (size_t)blockIdx.y * NIT * CV_BSTAGE;
  const uint8_t* asrc = reinterpret_cast<const uint8_t*>(img) + (size_t)blockIdx.x * 2 * CIN * R * 2;
  auto issue = [&](int it) {
    const int s = it % CV_STAGES, cc = it / NTG;
    const bool first = it % NTG == 0;
    tc::mbar_arrive_expect_tx(full + s, CV_BSTAGE + (first ? 2 * A_UNIT : 0u));
    tc::bulk_g2s(Bs + s * CV_BSTAGE, wsrc + (size_t)it * CV_BSTAGE, CV_BSTAGE, full + s);
    if (first)
      for (int u = 0; u < 2; ++u)
        tc::bulk_g2s(As + ((cc & 1) * 2 + u) * A_UNIT, asrc + ((size_t)u * CIN + (size_t)cc * CK) * R * 2, A_UNIT, full + s);
  };
  if (tid == 0) {
    for (int s = 0; s < CV_STAGES; ++s) tc::mbar_init(full + s, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();
  if (tid == 0) {
    issue(0);
    issue(1);
  }
  float d[UM][64];
  for (int it = 0; it < NIT; ++it) {
    // stage (it + 2) % 3 was read by iteration it - 1, which every thread has left; the image buffer it may refill
    // was last read NTG >= 8 iterations earlier
    if (tid == 0 && it + 2 < NIT) issue(it + 2);
    const int s = it % CV_STAGES, cc = it / NTG, tg = it % NTG;
    tc::mbar_wait(full + s, (it / CV_STAGES) & 1);
    const uint32_t a0 = tc::smem_u32(As + ((cc & 1) * 2 + wg) * A_UNIT), b0 = tc::smem_u32(Bs + s * CV_BSTAGE);
    tc::wg_fence();
#pragma unroll
    for (int t = 0; t < TG; ++t) {
#pragma unroll
      for (int k = 0; k < CK / 16; ++k) {
        const uint64_t db = tc::smem_desc(b0 + (t * (CK / 8) + 2 * k) * 2048, 2048);
#pragma unroll
        for (int mt = 0; mt < UM; ++mt)
          tc::Wg<128, 0>::ss(d[mt], tc::smem_desc(a0 + 2 * k * (R * 16) + (mt * 64 + (tg * TG + t) * G) * 16, R * 16), db,
                             (it | t | k) ? 1u : 0u);
      }
    }
    tc::wg_commit();
    tc::wg_wait<0>();
    __syncthreads();
  }
  const long long unit = (long long)blockIdx.x * 2 + wg;
  const int n0 = blockIdx.y * 128;
#pragma unroll
  for (int mt = 0; mt < UM; ++mt) {
    tc::wg_hold(d[mt]);
#pragma unroll
    for (int i = 0; i < 16; ++i) {
      const int col = n0 + 8 * i + 2 * (l & 3);
      const float b0 = __ldg(E.bias + col), b1 = __ldg(E.bias + col + 1), s0 = __ldg(E.scale + col), s1 = __ldg(E.scale + col + 1);
      const float h0 = __ldg(E.shift + col), h1 = __ldg(E.shift + col + 1);
      float v[4];
#pragma unroll
      for (int e = 0; e < 4; ++e)
        v[e] = fmaf(fmaxf(d[mt][4 * i + e] + ((e & 1) ? b1 : b0), 0.f), (e & 1) ? s1 : s0, (e & 1) ? h1 : h0);
      // tile row m = 16 w + l / 4 + 8 h is position m / G of frame m % G: the pool partner is row m + G
      if (G == 8) {
        const int m = 16 * w + (l >> 2);
        crepe_store2(E, unit * G + (m & 7), (mt * 64 + m) / (2 * G), col, fmaxf(v[0], v[2]), fmaxf(v[1], v[3]));
      } else {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const float p0 = fmaxf(v[2 * h], __shfl_xor_sync(0xffffffffu, v[2 * h], 4 * G));
          const float p1 = fmaxf(v[2 * h + 1], __shfl_xor_sync(0xffffffffu, v[2 * h + 1], 4 * G));
          const int m = mt * 64 + 16 * w + (l >> 2) + 8 * h;
          if (((m / G) & 1) == 0) crepe_store2(E, unit * G + (m % G), m / (2 * G), col, p0, p1);
        }
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------- tiny capacity
struct CrepeTinyLayer {
  const float *w, *bias, *scale, *shift;   // w [Cout][Cin][taps]
};
struct CrepeTinyParams {
  CrepeTinyLayer L[6];
};
constexpr int TN_C[7] = {1, 128, 16, 16, 16, 32, 64};
constexpr int TN_BUF0 = 128 * (128 + 63), TN_BUF1 = 2048;
constexpr size_t TN_SMEM = sizeof(float) * (TN_BUF0 + TN_BUF1);

// out[co][31 + q] = max over the position pair of BN(ReLU(conv)); in rows are inW wide with the padding in place
template <int TAPS, int STRIDE>
__device__ void crepe_tiny_layer(const float* in, int cin, int inW, const CrepeTinyLayer& L, int cout, int P, float* out,
                                 float* feat) {
  const int Pq = P / 2, outW = Pq + CR_TAPS - 1;
  if (!feat) {
    for (int i = threadIdx.x; i < cout * outW; i += blockDim.x) out[i] = 0.f;
    __syncthreads();
  }
  for (int idx = threadIdx.x; idx < cout * Pq; idx += blockDim.x) {
    const int co = idx / Pq, q = idx - co * Pq;
    float a0 = __ldg(L.bias + co), a1 = a0;
    for (int ci = 0; ci < cin; ++ci) {
      const float* xp = in + ci * inW + 2 * q * STRIDE;
      const float* wp = L.w + ((size_t)co * cin + ci) * TAPS;
#pragma unroll 8
      for (int j = 0; j < TAPS; ++j) {
        const float wv = __ldg(wp + j);
        a0 = fmaf(wv, xp[j], a0);
        a1 = fmaf(wv, xp[j + STRIDE], a1);
      }
    }
    const float sc = __ldg(L.scale + co), sh = __ldg(L.shift + co);
    const float v = fmaxf(fmaf(fmaxf(a0, 0.f), sc, sh), fmaf(fmaxf(a1, 0.f), sc, sh));
    if (feat) feat[q * cout + co] = v;
    else out[co * outW + CR_PADL + q] = v;
  }
  __syncthreads();
}

__global__ void __launch_bounds__(256)
crepe_tiny_kernel(const float* __restrict__ frames, CrepeTinyParams P, float* __restrict__ feat) {
  extern __shared__ __align__(16) float tsm[];
  float* b0 = tsm;
  float* b1 = tsm + TN_BUF0;
  for (int i = threadIdx.x; i < C1_XLEN; i += 256) {
    const int s = i - C1_PAD;
    b1[i] = s >= 0 && s < CR_WIN ? __ldg(frames + (size_t)blockIdx.x * CR_WIN + s) : 0.f;
  }
  __syncthreads();
  crepe_tiny_layer<512, 4>(b1, 1, C1_XLEN, P.L[0], 128, 256, b0, nullptr);   // channels: TN_C
  crepe_tiny_layer<64, 1>(b0, 128, 191, P.L[1], 16, 128, b1, nullptr);
  crepe_tiny_layer<64, 1>(b1, 16, 127, P.L[2], 16, 64, b0, nullptr);
  crepe_tiny_layer<64, 1>(b0, 16, 95, P.L[3], 16, 32, b1, nullptr);
  crepe_tiny_layer<64, 1>(b1, 16, 79, P.L[4], 32, 16, b0, nullptr);
  crepe_tiny_layer<64, 1>(b0, 32, 71, P.L[5], 64, 8, nullptr, feat + (size_t)blockIdx.x * 256);
}

// ------------------------------------------------------------------------------------------------- classifier
constexpr int CL_FR = 8;
// grid ceil(F / 8), 384 threads; wt [IN][360], thread = bin
__global__ void __launch_bounds__(384)
crepe_classify_kernel(const float* __restrict__ feat, const float* __restrict__ wt, const float* __restrict__ bias, int IN,
                      int nframes, float* __restrict__ probs) {
  extern __shared__ __align__(16) float fs[];   // [8][IN]
  const int f0 = blockIdx.x * CL_FR, n = threadIdx.x;
  for (int i = threadIdx.x; i < CL_FR * IN; i += 384) fs[i] = f0 + i / IN < nframes ? __ldg(feat + (size_t)f0 * IN + i) : 0.f;
  __syncthreads();
  if (n >= CR_BINS) return;
  float acc[CL_FR];
#pragma unroll
  for (int f = 0; f < CL_FR; ++f) acc[f] = 0.f;
  for (int k = 0; k < IN; ++k) {
    const float wv = __ldg(wt + (size_t)k * CR_BINS + n);
#pragma unroll
    for (int f = 0; f < CL_FR; ++f) acc[f] = fmaf(wv, fs[f * IN + k], acc[f]);
  }
  const float b = __ldg(bias + n);
  const bool in_band = n >= CR_BIN_LO && n < CR_BIN_HI;
#pragma unroll
  for (int f = 0; f < CL_FR; ++f)
    if (f0 + f < nframes) probs[(size_t)(f0 + f) * CR_BINS + n] = in_band ? 1.f / (1.f + expf(-(acc[f] + b))) : -INFINITY;
}

// ------------------------------------------------------------------------------------------------- decoder
constexpr int DC_BAND = 23;   // transition[i][j] > 0 for |i - j| < 12
constexpr size_t DC_SMEM = sizeof(double) * (CR_BINS * DC_BAND + 2 * CR_BINS) + sizeof(float) * 2 * CR_SEG_MAX + sizeof(short) * CR_SEG_MAX;
// one CTA per segment; it.in: frame offsets, it.out: segment offsets
__global__ void __launch_bounds__(384)
crepe_decode_kernel(const float* __restrict__ probs, const float* __restrict__ dither, ItemPass<CR_GROUP> it, long long seg0,
                    int segment, unsigned short* __restrict__ ptr, int* __restrict__ bins_out, float* __restrict__ pitch_out,
                    float* __restrict__ period_out) {
  extern __shared__ __align__(16) uint8_t dsm[];
  double* band = reinterpret_cast<double*>(dsm);   // [360][23]: log(transition[i][i + d - 11] + tiny)
  double* val = band + CR_BINS * DC_BAND;          // [2][360]
  float* smax = reinterpret_cast<float*>(val + 2 * CR_BINS);
  float* ssum = smax + CR_SEG_MAX;
  short* state = reinterpret_cast<short*>(ssum + CR_SEG_MAX);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long sg = seg0 + blockIdx.x;
  const int b = item_of(it.out, sg);
  const long long t0 = it.in[b] + (sg - it.out[b]) * segment;
  const int T = (int)min((long long)segment, it.in[b + 1] - t0);
  const float* x = probs + t0 * CR_BINS;
  unsigned short* bp = ptr + t0 * CR_BINS;
  const double tiny = (double)FLT_MIN, ltiny = log(tiny);

  for (int i = tid; i < CR_BINS; i += 384) {
    int rowsum = 0;
    for (int j = max(0, i - 11); j <= min(CR_BINS - 1, i + 11); ++j) rowsum += 12 - abs(i - j);
    for (int dd = 0; dd < DC_BAND; ++dd) band[i * DC_BAND + dd] = log((double)(12 - abs(dd - 11)) / (double)rowsum + tiny);
  }
  for (int t = warp; t < T; t += 12) {   // softmax statistics of each frame (fp32, as torch takes them)
    float m = -INFINITY;
    for (int j = lane; j < CR_BINS; j += 32) m = fmaxf(m, x[(size_t)t * CR_BINS + j]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
    float s = 0.f;
    for (int j = lane; j < CR_BINS; j += 32) s += expf(x[(size_t)t * CR_BINS + j] - m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) { smax[t] = m; ssum[t] = s; }
  }
  __syncthreads();
  const int j = tid;
  auto logp = [&](int t) { return log((double)(expf(x[(size_t)t * CR_BINS + j] - smax[t]) / ssum[t]) + tiny); };
  if (j < CR_BINS) val[j] = logp(0) + log(1.0 / CR_BINS + tiny);
  __syncthreads();
  for (int t = 1; t < T; ++t) {
    const double* vp = val + ((t - 1) & 1) * CR_BINS;
    if (j < CR_BINS) {
      double best = -INFINITY;
      int arg = 0;
      for (int i = 0; i < CR_BINS; ++i) {
        const unsigned dd = (unsigned)(j - i + 11);
        const double c = vp[i] + (dd < (unsigned)DC_BAND ? band[i * DC_BAND + dd] : ltiny);
        if (c > best) { best = c; arg = i; }
      }
      bp[(size_t)t * CR_BINS + j] = (unsigned short)arg;
      val[(t & 1) * CR_BINS + j] = logp(t) + best;
    }
    __syncthreads();
  }
  if (tid == 0) {
    const double* vp = val + ((T - 1) & 1) * CR_BINS;
    int arg = 0;
    for (int i = 1; i < CR_BINS; ++i)
      if (vp[i] > vp[arg]) arg = i;
    state[T - 1] = (short)arg;
    for (int t = T - 2; t >= 0; --t) {
      arg = bp[(size_t)(t + 1) * CR_BINS + arg];
      state[t] = (short)arg;
    }
  }
  __syncthreads();
  for (int t = tid; t < T; t += 384) {
    const int bin = state[t];
    bins_out[t0 + t] = bin;
    // crepe/convert.py: cents = 20 bin + 1997.379...; + dither; 10 * 2^(cents / 1200), all fp32
    float cents = __fadd_rn(__fmul_rn(20.f, (float)bin), 1997.3794084376191f);
    if (dither) cents = __fadd_rn(cents, __ldg(dither + t0 + t));
    pitch_out[t0 + t] = 10.f * exp2f(cents / 1200.f);
    if (period_out) period_out[t0 + t] = x[(size_t)t * CR_BINS + bin];
  }
}

static DevSmemCache g_c1, g_cv[5], g_tiny, g_cls, g_dec;

// geometry of the full-capacity images: the input of conv L + 2
struct CrepeGeom { int cin, cout, G, UM, R; };
constexpr CrepeGeom CR_FULL[5] = {{1024, 128, 1, 2, cr_rows(1, 2)}, {128, 128, 1, 1, cr_rows(1, 1)}, {128, 128, 2, 1, cr_rows(2, 1)},
                                  {128, 256, 4, 1, cr_rows(4, 1)}, {256, 512, 8, 1, cr_rows(8, 1)}};
inline size_t cr_image_bytes(int L, int frames) { return (size_t)(frames / CR_FULL[L].G) * CR_FULL[L].cin * CR_FULL[L].R * 2; }

}  // namespace svcb

using namespace svcb;

struct svcb_crepe {
  int capacity = 0;   // 0 full, 1 tiny
  int feat = 0;       // classifier inputs
  const float *bias[6], *scale[6], *shift[6];
  const __nv_bfloat16* wimg[6];   // full
  CrepeTinyParams tiny;
  const float *cls_wt, *cls_b;
};

struct CrepeWs {
  size_t frames, feat, img[5], total;
  CrepeWs(int capacity, int chunk, int feat_dim) {
    WsPlan p;
    frames = p.take((size_t)chunk * CR_WIN * 4);
    feat = p.take((size_t)chunk * feat_dim * 4);
    for (int L = 0; L < 5; ++L) img[L] = capacity == 0 ? p.take(cr_image_bytes(L, chunk)) : 0;
    total = p.off;
  }
};
static int crepe_chunk(int64_t total_frames) {
  const int64_t c = std::min<int64_t>(CR_CHUNK_MAX, (total_frames + CR_CHUNK_ALIGN - 1) / CR_CHUNK_ALIGN * CR_CHUNK_ALIGN);
  return (int)std::max<int64_t>(c, CR_CHUNK_ALIGN);
}

template <int L, int CIN, int G, int UM, int CK>
static int crepe_launch_conv(const svcb_crepe* m, const uint8_t* ws, const CrepeWs& W, int chunk, float* feat, cudaStream_t s) {
  auto kern = crepe_conv_tc_kernel<CIN, G, UM, CK>;
  SVCB_CUDA_CHECK(ensure_dyn_smem(kern, cv_smem<G, UM, CK>(), g_cv[L]));
  const CrepeGeom& g = CR_FULL[L];
  CrepeEpi E{m->bias[L + 1], m->scale[L + 1], m->shift[L + 1], nullptr, nullptr, g.cout, 1, 0, 64 * UM / G / 2};
  if (L < 4) {
    E.img = reinterpret_cast<__nv_bfloat16*>(const_cast<uint8_t*>(ws) + W.img[L + 1]);
    E.Gn = CR_FULL[L + 1].G;
    E.Rn = CR_FULL[L + 1].R;
  } else {
    E.feat = feat;
  }
  static const char* names[5] = {"crepe_conv2", "crepe_conv3", "crepe_conv4", "crepe_conv5", "crepe_conv6"};
  KernelScope ks(names[L], s, 2.0 * chunk * (64.0 * UM / G) * g.cout * CR_TAPS * CIN,
                 (double)cr_image_bytes(L, chunk) + 2.0 * g.cout * CR_TAPS * CIN);
  kern<<<dim3(chunk / G / 2, g.cout / 128), 256, cv_smem<G, UM, CK>(), s>>>(
      reinterpret_cast<const __nv_bfloat16*>(ws + W.img[L]), m->wimg[L + 1], E);
  SVCB_LAUNCH_CHECK(names[L]);
  return SVCB_OK;
}

static int crepe_frame_pass(const float* wav, const float* noise, const ItemPass<CR_GROUP>& it, long long f0, int n, int hop,
                            float* frames, cudaStream_t s) {
  KernelScope ks("crepe_frame", s, 0.0, (double)n * CR_WIN * 8.0);
  crepe_frame_kernel<<<n, 256, 0, s>>>(wav, noise, it, f0, hop, frames);
  SVCB_LAUNCH_CHECK("crepe_frame");
  return SVCB_OK;
}

static int crepe_check_hop(const char* who, int32_t hop) {
  if (hop >= 1 && hop <= CR_WIN) return SVCB_OK;
  set_error(std::string(who) + ": hop " + std::to_string(hop) + " is outside 1..1024");
  return SVCB_E_BAD_SHAPE;
}

extern "C" {

int svcb_crepe_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                      int32_t capacity, svcb_crepe** out) {
  if (!dev_blob || !table_host || !out) { set_error("svcb_crepe_create: bad argument"); return SVCB_E_BAD_SHAPE; }
  if (capacity != 0 && capacity != 1) { set_error("svcb_crepe_create: capacity must be 0 (full) or 1 (tiny)"); return SVCB_E_UNSUPPORTED; }
  SVCB_TRY(check_blob_device(dev_blob));
  BlobTensors t;
  SVCB_TRY(t.read(dev_blob, blob_bytes, table_host, n_entries));
  auto m = std::make_unique<svcb_crepe>();
  m->capacity = capacity;
  static const int full_c[7] = {1, 1024, 128, 128, 128, 256, 512};
  const int* C = capacity == 0 ? full_c : TN_C;
  m->feat = 4 * C[6];
  for (int L = 0; L < 6; ++L) {
    const std::string p = "crepe.conv" + std::to_string(L + 1);
    const uint64_t wn = (uint64_t)C[L + 1] * C[L] * (L == 0 ? C1_K : CR_TAPS);
    m->bias[L] = t.get(p + ".bias", C[L + 1]);
    m->scale[L] = t.get(p + ".scale", C[L + 1]);
    m->shift[L] = t.get(p + ".shift", C[L + 1]);
    if (capacity == 0) {
      m->wimg[L] = reinterpret_cast<const __nv_bfloat16*>(t.get(p + ".wimg", wn / 2));
    } else {
      m->tiny.L[L] = {t.get(p + ".w", wn), m->bias[L], m->scale[L], m->shift[L]};
    }
  }
  m->cls_wt = t.get("crepe.cls.wt", (uint64_t)m->feat * CR_BINS);
  m->cls_b = t.get("crepe.cls.bias", CR_BINS);
  SVCB_TRY(t.status("crepe blob"));
  *out = m.release();
  return SVCB_OK;
}

void svcb_crepe_destroy(svcb_crepe* m) { delete m; }

int64_t svcb_crepe_frames(int64_t n_samples, int32_t hop) { return n_samples < 0 || hop < 1 ? 0 : 1 + n_samples / hop; }

size_t svcb_crepe_workspace_bytes(const svcb_crepe* m, int64_t total_frames) {
  if (!m || total_frames <= 0) return 0;
  return CrepeWs(m->capacity, crepe_chunk(total_frames), m->feat).total;
}

int svcb_crepe_frame(const float* wav, const int64_t* sample_offsets_host, int32_t B, int32_t hop, const float* noise,
                     float* frames_out, svcb_stream stream) {
  if (!sample_offsets_host || !frames_out) { set_error("svcb_crepe_frame: bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(crepe_check_hop("svcb_crepe_frame", hop));
  SVCB_TRY(check_ragged("svcb_crepe_frame", sample_offsets_host, B, 1, 0, "samples", nullptr));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return for_each_pass<CR_GROUP>(sample_offsets_host, B, [&](long long n) { return 1 + n / hop; },
                                 [&](const ItemPass<CR_GROUP>& it, int) -> int {
    for (long long f = it.out[0]; f < it.out[it.n]; f += 65536) {
      const int n = (int)std::min<long long>(65536, it.out[it.n] - f);
      SVCB_TRY(crepe_frame_pass(wav, noise, it, f, n, hop, frames_out + (size_t)f * CR_WIN, s));
    }
    return SVCB_OK;
  });
}

int svcb_crepe_probs(const svcb_crepe* m, const float* wav, const int64_t* sample_offsets_host, int32_t B, int32_t hop,
                     const float* noise, float* probs_out, void* ws, size_t ws_bytes, svcb_stream stream) {
  if (!m || !sample_offsets_host || !probs_out) { set_error("svcb_crepe_probs: bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(crepe_check_hop("svcb_crepe_probs", hop));
  SVCB_TRY(check_ragged("svcb_crepe_probs", sample_offsets_host, B, 1, 0, "samples", nullptr));
  long long total = 0;
  for (int b = 0; b < B; ++b) total += 1 + (sample_offsets_host[b + 1] - sample_offsets_host[b]) / hop;
  const int chunk = crepe_chunk(total);
  const CrepeWs W(m->capacity, chunk, m->feat);
  SVCB_TRY(check_workspace(ws, ws_bytes, W.total, "crepe"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  uint8_t* w8 = static_cast<uint8_t*>(ws);
  float* frames = reinterpret_cast<float*>(w8 + W.frames);
  float* feat = reinterpret_cast<float*>(w8 + W.feat);
  const size_t cls_smem = (size_t)CL_FR * m->feat * sizeof(float);
  SVCB_CUDA_CHECK(ensure_dyn_smem(crepe_classify_kernel, cls_smem, g_cls));
  if (m->capacity == 0) {
    SVCB_CUDA_CHECK(ensure_dyn_smem(crepe_conv1_tc_kernel, C1_SMEM, g_c1));
    // the padding rows of the images are never written: zero them once, every chunk leaves them so
    SVCB_CUDA_CHECK(cudaMemsetAsync(w8 + W.img[0], 0, W.total - W.img[0], s));
  } else {
    SVCB_CUDA_CHECK(ensure_dyn_smem(crepe_tiny_kernel, TN_SMEM, g_tiny));
  }
  const int sms = std::max(device_sm_count(), 8);
  return for_each_pass<CR_GROUP>(sample_offsets_host, B, [&](long long n) { return 1 + n / hop; },
                                 [&](const ItemPass<CR_GROUP>& it, int) -> int {
    for (long long f = it.out[0]; f < it.out[it.n]; f += chunk) {
      const int n = (int)std::min<long long>(chunk, it.out[it.n] - f);
      const int np = (n + CR_CHUNK_ALIGN - 1) / CR_CHUNK_ALIGN * CR_CHUNK_ALIGN;   // whole conv6 CTAs; the rest is discarded
      SVCB_TRY(crepe_frame_pass(wav, noise, it, f, n, hop, frames, s));
      if (m->capacity == 0) {
        {
          CrepeEpi E{m->bias[0], m->scale[0], m->shift[0], reinterpret_cast<__nv_bfloat16*>(w8 + W.img[0]), nullptr, 1024, 1,
                     CR_FULL[0].R, 128};
          KernelScope ks("crepe_conv1", s, 2.0 * n * 256 * 1024 * C1_K, (double)n * (CR_WIN * 4.0 + 128 * 1024 * 2.0));
          crepe_conv1_tc_kernel<<<dim3(8, std::min(n, std::max(sms / 8, 1))), 256, C1_SMEM, s>>>(frames, m->wimg[0], E, n);
          SVCB_LAUNCH_CHECK("crepe_conv1");
        }
        SVCB_TRY((crepe_launch_conv<0, 1024, 1, 2, 64>(m, w8, W, np, feat, s)));
        SVCB_TRY((crepe_launch_conv<1, 128, 1, 1, 64>(m, w8, W, np, feat, s)));
        SVCB_TRY((crepe_launch_conv<2, 128, 2, 1, 64>(m, w8, W, np, feat, s)));
        SVCB_TRY((crepe_launch_conv<3, 128, 4, 1, 32>(m, w8, W, np, feat, s)));
        SVCB_TRY((crepe_launch_conv<4, 256, 8, 1, 16>(m, w8, W, np, feat, s)));
      } else {
        KernelScope ks("crepe_tiny", s, 2.0 * n * 36.2e6, (double)n * CR_WIN * 4.0);
        crepe_tiny_kernel<<<n, 256, TN_SMEM, s>>>(frames, m->tiny, feat);
        SVCB_LAUNCH_CHECK("crepe_tiny");
      }
      KernelScope ks("crepe_classify", s, 2.0 * n * m->feat * CR_BINS, (double)n * (m->feat + CR_BINS) * 4.0);
      crepe_classify_kernel<<<(n + CL_FR - 1) / CL_FR, 384, cls_smem, s>>>(feat, m->cls_wt, m->cls_b, m->feat, n,
                                                                            probs_out + (size_t)f * CR_BINS);
      SVCB_LAUNCH_CHECK("crepe_classify");
    }
    return SVCB_OK;
  });
}

size_t svcb_crepe_decode_workspace_bytes(int64_t total_frames) {
  return total_frames <= 0 ? 0 : align256((size_t)total_frames * CR_BINS * sizeof(unsigned short));
}

int svcb_crepe_decode(const float* probs, const int64_t* frame_offsets_host, int32_t B, int32_t segment, const float* dither,
                      int32_t* bins_out, float* pitch_out, float* periodicity_out, void* ws, size_t ws_bytes,
                      svcb_stream stream) {
  if (!probs || !frame_offsets_host || !bins_out || !pitch_out) { set_error("svcb_crepe_decode: bad argument"); return SVCB_E_BAD_SHAPE; }
  if (segment < 1 || segment > CR_SEG_MAX) {
    set_error("svcb_crepe_decode: segment " + std::to_string(segment) + " is outside 1..512");
    return SVCB_E_BAD_SHAPE;
  }
  SVCB_TRY(check_ragged("svcb_crepe_decode", frame_offsets_host, B, 1, 1, "frames", nullptr));
  SVCB_TRY(check_workspace(ws, ws_bytes, svcb_crepe_decode_workspace_bytes(frame_offsets_host[B]), "crepe decode"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  SVCB_CUDA_CHECK(ensure_dyn_smem(crepe_decode_kernel, DC_SMEM, g_dec));
  return for_each_pass<CR_GROUP>(frame_offsets_host, B, [&](long long n) { return (n + segment - 1) / segment; },
                                 [&](const ItemPass<CR_GROUP>& it, int) -> int {
    const long long nseg = it.out[it.n] - it.out[0];
    KernelScope ks("crepe_decode", s, 0.0, (double)(it.in[it.n] - it.in[0]) * CR_BINS * 6.0, (double)(it.in[it.n] - it.in[0]) * CR_BINS * CR_BINS);
    crepe_decode_kernel<<<(unsigned)nseg, 384, DC_SMEM, s>>>(probs, dither, it, it.out[0], segment,
                                                             static_cast<unsigned short*>(ws), bins_out, pitch_out,
                                                             periodicity_out);
    SVCB_LAUNCH_CHECK("crepe_decode");
    return SVCB_OK;
  });
}

}  // extern "C"

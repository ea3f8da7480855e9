// Silero VAD (vad/assets/silero_vad.jit, the 16 kHz branch `_model`) on the device: one speech probability per
// 512-sample window of 16 kHz audio, for a ragged batch of recordings.
//
//   vad_front  one CTA per VAD_WPC consecutive windows of a pass (they may straddle items), all fp32:
//              reflect-pad each window by 96 to 704 samples (local to the window), STFT as the 258 x 256 conv basis at
//              stride 64 (8 frames; FFMA, the basis read k-major from L2 as float4), magnitude, the adaptive
//              normalisation (log1p(mag 2^20), the bin mean per frame, reflect pad 3, 7-tap filter, the frame mean),
//              first_layer and the encoder (BatchNorm as eval scale and shift) down to one 64-d vector, then layer 0's
//              input product W_ih0 x + b_ih0 + b_hh0 -> G [window][256]; the 64-d vector is an optional tap
//   vad_rec    one CTA per item, the whole chain of its windows: W_hh0, W_ih1 and W_hh1 (192 KB, k-major) resident in
//              shared memory, h broadcast through shared memory, fp32 gate math with expf / tanhf, then ReLU, the
//              64 -> 1 conv and the sigmoid fused into each step
//
// Every window's front end and every item's chain run the same instructions whatever the batch, so an item's
// probabilities are bitwise equal to the item run alone.
#include <algorithm>
#include <cstdint>
#include <memory>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int VAD_WIN = 512, VAD_PAD = 96, VAD_PW = VAD_WIN + 2 * VAD_PAD;   // 704 padded samples per window
constexpr int VAD_NFFT = 256, VAD_HOP = 64, VAD_NF = 8, VAD_BINS = 129, VAD_FEAT = 2 * VAD_BINS;
constexpr int VAD_H = 64, VAD_G = 4 * VAD_H;
constexpr int VAD_WPC = 4;        // windows per front-end CTA (2 x 16 frames per thread)
constexpr int VAD_GROUP = 128;    // items per pass
constexpr int VAD_BUF = 128;      // floats per window of an encoder buffer (the widest is 16 x 8 = 32 x 4)
constexpr size_t VAD_FRONT_SMEM = sizeof(float) * (VAD_WPC * VAD_PW + VAD_WPC * VAD_FEAT * VAD_NF + 3 * VAD_WPC * VAD_BUF + VAD_WPC * 8);
constexpr size_t VAD_REC_SMEM = sizeof(float) * (3 * VAD_H * VAD_G + 2 * VAD_H + VAD_G);

struct VadWeights {
  const float* basis4;   // [2 (re, im)][64 k-quads][128 bins][4]: bins 0 .. 127
  const float* nyq;      // [2][256]: bin 128
  const float* filt;     // [7]
  const float *fl_dw_w, *fl_dw_b, *fl_pw_w, *fl_pw_b, *fl_pj_w, *fl_pj_b;   // first_layer: [258][5], [16][258] x 2
  const float *e0_w, *e0_b, *bn0;                                           // encoder.0 [16][16], BN {scale, shift}
  const float *b1_dw_w, *b1_dw_b, *b1_pw_w, *b1_pw_b, *b1_pj_w, *b1_pj_b;   // encoder.3.0: 16 -> 32
  const float *e4_w, *e4_b, *bn4;                                           // encoder.4 [32][32]
  const float *b2_dw_w, *b2_dw_b, *b2_pw_w, *b2_pw_b;                       // encoder.7.0: 32 -> 32, identity residual
  const float *e8_w, *e8_b, *bn8;                                           // encoder.8 [32][32]
  const float *b3_dw_w, *b3_dw_b, *b3_pw_w, *b3_pw_b, *b3_pj_w, *b3_pj_b;   // encoder.11.0: 32 -> 64
  const float *e12_w, *e12_b, *bn12;                                        // encoder.12 [64][64]
  const float *wih0t, *b0;                                                  // W_ih0^T [64][256], b_ih0 + b_hh0
};

// y[w][co][t] = act(bn(b[co] + sum_ci W[co][ci] x[w][ci][t s]) + res[w][co][t]) for the CTA's windows (1 x 1 conv;
// BatchNorm after the conv, the residual after the bias, as each caller's module orders them)
__device__ void vad_conv1x1(const float* x, int xws, int Cin, int Tin, int s, const float* __restrict__ W,
                            const float* __restrict__ b, float* y, int Cout, int Tout, const float* res,
                            const float* __restrict__ bn, bool relu) {
  for (int i = threadIdx.x; i < VAD_WPC * Cout * Tout; i += blockDim.x) {
    const int w = i / (Cout * Tout), co = (i / Tout) % Cout, t = i % Tout;
    const float* xp = x + w * xws + t * s;
    const float* wp = W + co * Cin;
    float acc = __ldg(b + co);
    for (int ci = 0; ci < Cin; ++ci) acc = fmaf(__ldg(wp + ci), xp[ci * Tin], acc);
    if (res) acc += res[i];
    if (bn) acc = fmaf(acc, __ldg(bn + co), __ldg(bn + Cout + co));
    y[i] = relu ? fmaxf(acc, 0.f) : acc;
  }
}

// depthwise conv k5, zero pad 2, with bias, then ReLU: y[w][c][t] (y may alias x: each thread owns whole rows)
template <int T>
__device__ void vad_dw(const float* x, int xws, int C, const float* __restrict__ wk, const float* __restrict__ bk, float* y) {
  for (int i = threadIdx.x; i < VAD_WPC * C; i += blockDim.x) {
    const int w = i / C, c = i - w * C;
    const float* xp = x + w * xws + c * T;
    float v[T], o[T];
#pragma unroll
    for (int t = 0; t < T; ++t) v[t] = xp[t];
#pragma unroll
    for (int t = 0; t < T; ++t) {
      float acc = __ldg(bk + c);
#pragma unroll
      for (int j = 0; j < 5; ++j)
        if (t + j - 2 >= 0 && t + j - 2 < T) acc = fmaf(__ldg(wk + c * 5 + j), v[t + j - 2], acc);
      o[t] = fmaxf(acc, 0.f);
    }
    float* yp = y + w * xws + c * T;
#pragma unroll
    for (int t = 0; t < T; ++t) yp[t] = o[t];
  }
}

// ----------------------------------------------------------------------------------------------------- front end
// grid ceil(windows of the pass / VAD_WPC), 256 threads; it: samples in, windows out
__global__ void __launch_bounds__(256)
vad_front_kernel(const float* __restrict__ wav, VadWeights P, ItemPass<VAD_GROUP> it, float* __restrict__ G,
                 float* __restrict__ feat_out) {
  extern __shared__ __align__(16) float sm[];
  float* xw = sm;                                       // [VAD_WPC][704]
  float* fe = xw + VAD_WPC * VAD_PW;                    // [VAD_WPC][258][8]: magnitude, then the normalised log
  float* bA = fe + VAD_WPC * VAD_FEAT * VAD_NF;         // encoder buffers [VAD_WPC][VAD_BUF]
  float* bB = bA + VAD_WPC * VAD_BUF;
  float* bR = bB + VAD_WPC * VAD_BUF;
  float* fm = bR + VAD_WPC * VAD_BUF;                   // [VAD_WPC][8] bin means of each frame
  const int tid = threadIdx.x;
  const long long w_first = it.out[0] + (long long)blockIdx.x * VAD_WPC, w_end = it.out[it.n];

  for (int i = tid; i < VAD_WPC * VAD_PW; i += 256) {
    const int w = i / VAD_PW, p = i - w * VAD_PW;
    const long long gw = w_first + w;
    float v = 0.f;
    if (gw < w_end) {
      const int b = item_of(it.out, gw);
      const long long s0 = it.in[b] + (gw - it.out[b]) * VAD_WIN, n = it.in[b + 1] - s0;   // n >= 1
      int s = p - VAD_PAD;                              // reflect inside the zero-padded 512-sample window
      if (s < 0) s = -s;
      if (s >= VAD_WIN) s = 2 * (VAD_WIN - 1) - s;
      if (s < n) v = __ldg(wav + s0 + s);
    }
    xw[i] = v;
  }
  __syncthreads();

  {  // STFT, bins 0 .. 127: thread = (bin, half of the CTA's 32 frames)
    const int bin = tid & 127, half = tid >> 7;
    float re[2 * VAD_NF], im[2 * VAD_NF];
#pragma unroll
    for (int f = 0; f < 2 * VAD_NF; ++f) { re[f] = 0.f; im[f] = 0.f; }
    const float4* br = reinterpret_cast<const float4*>(P.basis4) + bin;
    const float4* bi = br + (VAD_NFFT / 4) * 128;
    const float* x0 = xw + 2 * half * VAD_PW;
#pragma unroll 2
    for (int kq = 0; kq < VAD_NFFT / 4; ++kq) {
      const float4 r = __ldg(br + kq * 128), m = __ldg(bi + kq * 128);
#pragma unroll
      for (int f = 0; f < 2 * VAD_NF; ++f) {
        const float4 x = *reinterpret_cast<const float4*>(x0 + (f >> 3) * VAD_PW + (f & 7) * VAD_HOP + 4 * kq);
        re[f] = fmaf(r.x, x.x, re[f]); im[f] = fmaf(m.x, x.x, im[f]);
        re[f] = fmaf(r.y, x.y, re[f]); im[f] = fmaf(m.y, x.y, im[f]);
        re[f] = fmaf(r.z, x.z, re[f]); im[f] = fmaf(m.z, x.z, im[f]);
        re[f] = fmaf(r.w, x.w, re[f]); im[f] = fmaf(m.w, x.w, im[f]);
      }
    }
#pragma unroll
    for (int f = 0; f < 2 * VAD_NF; ++f) {
      const int w = 2 * half + (f >> 3);
      fe[(w * VAD_FEAT + bin) * VAD_NF + (f & 7)] = __fsqrt_rn(__fadd_rn(__fmul_rn(re[f], re[f]), __fmul_rn(im[f], im[f])));
    }
  }
  {  // bin 128: 64 dot products (32 frames x re / im), 4 threads each
    const int d = tid >> 2, q = tid & 3, f = d >> 1, ri = d & 1;
    const float* bp = P.nyq + ri * VAD_NFFT + q * 64;
    const float* xp = xw + (f >> 3) * VAD_PW + (f & 7) * VAD_HOP + q * 64;
    float acc = 0.f;
    for (int k = 0; k < 64; ++k) acc = fmaf(__ldg(bp + k), xp[k], acc);
    acc += __shfl_xor_sync(0xffffffffu, acc, 1);
    acc += __shfl_xor_sync(0xffffffffu, acc, 2);
    const float other = __shfl_xor_sync(0xffffffffu, acc, 4);   // the same frame's other part
    if (q == 0 && ri == 0)
      fe[((f >> 3) * VAD_FEAT + 128) * VAD_NF + (f & 7)] = __fsqrt_rn(__fadd_rn(__fmul_rn(acc, acc), __fmul_rn(other, other)));
  }
  __syncthreads();

  // adaptive normalisation: s = log1p(mag 2^20); the mean over bins per frame; reflect pad 3; 7-tap filter; frame mean
  for (int i = tid; i < VAD_WPC * VAD_BINS * VAD_NF; i += 256) {
    const int w = i / (VAD_BINS * VAD_NF), r = i - w * (VAD_BINS * VAD_NF);
    fe[w * VAD_FEAT * VAD_NF + VAD_BINS * VAD_NF + r] = log1pf(fe[w * VAD_FEAT * VAD_NF + r] * 1048576.f);
  }
  __syncthreads();
  {
    const int warp = tid >> 5, lane = tid & 31;
    for (int p = warp; p < VAD_WPC * VAD_NF; p += 8) {
      const int w = p >> 3, f = p & 7;
      const float* sp = fe + (w * VAD_FEAT + VAD_BINS) * VAD_NF + f;
      float a = 0.f;
      for (int c = lane; c < VAD_BINS; c += 32) a += sp[c * VAD_NF];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) a += __shfl_xor_sync(0xffffffffu, a, o);
      if (lane == 0) fm[p] = a / (float)VAD_BINS;
    }
  }
  __syncthreads();
  if (tid < VAD_WPC) {
    const float* m = fm + tid * VAD_NF;
    float mp[VAD_NF + 6];
#pragma unroll
    for (int i = 0; i < 3; ++i) { mp[i] = m[3 - i]; mp[VAD_NF + 3 + i] = m[VAD_NF - 2 - i]; }
#pragma unroll
    for (int i = 0; i < VAD_NF; ++i) mp[3 + i] = m[i];
    float tot = 0.f;
#pragma unroll
    for (int f = 0; f < VAD_NF; ++f) {
      float a = 0.f;
#pragma unroll
      for (int j = 0; j < 7; ++j) a = fmaf(__ldg(P.filt + j), mp[f + j], a);
      tot += a;
    }
    bA[tid] = tot / (float)VAD_NF;
  }
  __syncthreads();
  for (int i = tid; i < VAD_WPC * VAD_BINS * VAD_NF; i += 256) {
    const int w = i / (VAD_BINS * VAD_NF), r = i - w * (VAD_BINS * VAD_NF);
    fe[w * VAD_FEAT * VAD_NF + VAD_BINS * VAD_NF + r] -= bA[w];
  }
  __syncthreads();

  constexpr int FW = VAD_FEAT * VAD_NF;
  // first_layer: proj (258 -> 16) of the features, the depthwise conv in place, pointwise (258 -> 16) + proj, ReLU
  vad_conv1x1(fe, FW, VAD_FEAT, VAD_NF, 1, P.fl_pj_w, P.fl_pj_b, bR, 16, VAD_NF, nullptr, nullptr, false);
  __syncthreads();
  vad_dw<VAD_NF>(fe, FW, VAD_FEAT, P.fl_dw_w, P.fl_dw_b, fe);
  __syncthreads();
  vad_conv1x1(fe, FW, VAD_FEAT, VAD_NF, 1, P.fl_pw_w, P.fl_pw_b, bA, 16, VAD_NF, bR, nullptr, true);
  __syncthreads();
  // encoder: frames 8 -> 4 -> 2 -> 1
  vad_conv1x1(bA, 16 * 8, 16, 8, 2, P.e0_w, P.e0_b, bB, 16, 4, nullptr, P.bn0, true);               // [16][4]
  __syncthreads();
  vad_conv1x1(bB, 16 * 4, 16, 4, 1, P.b1_pj_w, P.b1_pj_b, bR, 32, 4, nullptr, nullptr, false);
  vad_dw<4>(bB, 16 * 4, 16, P.b1_dw_w, P.b1_dw_b, bA);
  __syncthreads();
  vad_conv1x1(bA, 16 * 4, 16, 4, 1, P.b1_pw_w, P.b1_pw_b, bB, 32, 4, bR, nullptr, true);            // [32][4]
  __syncthreads();
  vad_conv1x1(bB, 32 * 4, 32, 4, 2, P.e4_w, P.e4_b, bR, 32, 2, nullptr, P.bn4, true);               // [32][2]
  __syncthreads();
  vad_dw<2>(bR, 32 * 2, 32, P.b2_dw_w, P.b2_dw_b, bA);
  __syncthreads();
  vad_conv1x1(bA, 32 * 2, 32, 2, 1, P.b2_pw_w, P.b2_pw_b, bB, 32, 2, bR, nullptr, true);            // identity residual
  __syncthreads();
  vad_conv1x1(bB, 32 * 2, 32, 2, 2, P.e8_w, P.e8_b, bA, 32, 1, nullptr, P.bn8, true);               // [32][1]
  __syncthreads();
  vad_conv1x1(bA, 32, 32, 1, 1, P.b3_pj_w, P.b3_pj_b, bR, 64, 1, nullptr, nullptr, false);
  vad_dw<1>(bA, 32, 32, P.b3_dw_w, P.b3_dw_b, bB);
  __syncthreads();
  vad_conv1x1(bB, 32, 32, 1, 1, P.b3_pw_w, P.b3_pw_b, bA, 64, 1, bR, nullptr, true);                // [64][1]
  __syncthreads();
  vad_conv1x1(bA, 64, 64, 1, 1, P.e12_w, P.e12_b, bB, 64, 1, nullptr, P.bn12, true);                // [64]
  __syncthreads();

  // layer 0's input product, thread = gate row
  {
    float acc[VAD_WPC];
    const float bj = __ldg(P.b0 + tid);
#pragma unroll
    for (int w = 0; w < VAD_WPC; ++w) acc[w] = bj;
    for (int k = 0; k < VAD_H; ++k) {
      const float wk = __ldg(P.wih0t + k * VAD_G + tid);
#pragma unroll
      for (int w = 0; w < VAD_WPC; ++w) acc[w] = fmaf(wk, bB[w * VAD_H + k], acc[w]);
    }
#pragma unroll
    for (int w = 0; w < VAD_WPC; ++w)
      if (w_first + w < w_end) G[(w_first + w) * VAD_G + tid] = acc[w];
  }
  if (feat_out)
    for (int i = tid; i < VAD_WPC * VAD_H; i += 256)
      if (w_first + i / VAD_H < w_end) feat_out[w_first * VAD_H + i] = bB[i];
}

// ---------------------------------------------------------------------------------------------------- recurrence
// one CTA per item of the pass, 256 threads, thread j = gate row j (i, f, g, o blocks of 64); units u < 64 keep c
// of both layers in registers.  wrec = [W_hh0^T | W_ih1^T | W_hh1^T], each [64][256].
__global__ void __launch_bounds__(256, 1)
vad_rec_kernel(const float* __restrict__ wrec, const float* __restrict__ b1, const float* __restrict__ wdec,
               const float* __restrict__ G, float* __restrict__ probs, ItemPass<VAD_GROUP> it) {
  extern __shared__ __align__(16) float sm[];
  float* W = sm;                       // [3][64][256]
  float* h0 = W + 3 * VAD_H * VAD_G;   // [64]
  float* h1 = h0 + VAD_H;              // [64]
  float* gt = h1 + VAD_H;              // [256]
  const int j = threadIdx.x, lane = j & 31;
  const long long w0 = it.out[blockIdx.x], nw = it.out[blockIdx.x + 1] - w0;
  if (nw <= 0) return;
  for (int i = j; i < 3 * VAD_H * VAD_G / 4; i += 256)
    reinterpret_cast<float4*>(W)[i] = __ldg(reinterpret_cast<const float4*>(wrec) + i);
  if (j < VAD_H) { h0[j] = 0.f; h1[j] = 0.f; }
  const float bj = __ldg(b1 + j);
  const float wd0 = __ldg(wdec + lane), wd1 = __ldg(wdec + 32 + lane), bd = __ldg(wdec + VAD_H);
  float c0 = 0.f, c1 = 0.f;
  float g = __ldg(G + w0 * VAD_G + j);
  __syncthreads();
  const float* W0 = W;
  const float* W1 = W + VAD_H * VAD_G;
  const float* W2 = W + 2 * VAD_H * VAD_G;
  auto cell = [&](float& c, float* h) {   // gates i, f, g, o (nn.LSTM order) of unit j
    const float ig = 1.f / (1.f + expf(-gt[j])), fg = 1.f / (1.f + expf(-gt[VAD_H + j]));
    const float gg = tanhf(gt[2 * VAD_H + j]), og = 1.f / (1.f + expf(-gt[3 * VAD_H + j]));
    c = fg * c + ig * gg;
    h[j] = og * tanhf(c);
  };
  for (long long t = 0; t < nw; ++t) {
    float acc = g;
    if (t + 1 < nw) g = __ldg(G + (w0 + t + 1) * VAD_G + j);   // the next step's input product, in flight meanwhile
#pragma unroll 4
    for (int k = 0; k < VAD_H; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h0 + k);
      acc = fmaf(W0[(k + 0) * VAD_G + j], hv.x, acc);
      acc = fmaf(W0[(k + 1) * VAD_G + j], hv.y, acc);
      acc = fmaf(W0[(k + 2) * VAD_G + j], hv.z, acc);
      acc = fmaf(W0[(k + 3) * VAD_G + j], hv.w, acc);
    }
    gt[j] = acc;
    __syncthreads();
    if (j < VAD_H) cell(c0, h0);
    __syncthreads();
    acc = bj;
#pragma unroll 4
    for (int k = 0; k < VAD_H; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h0 + k);
      acc = fmaf(W1[(k + 0) * VAD_G + j], hv.x, acc);
      acc = fmaf(W1[(k + 1) * VAD_G + j], hv.y, acc);
      acc = fmaf(W1[(k + 2) * VAD_G + j], hv.z, acc);
      acc = fmaf(W1[(k + 3) * VAD_G + j], hv.w, acc);
    }
#pragma unroll 4
    for (int k = 0; k < VAD_H; k += 4) {
      const float4 hv = *reinterpret_cast<const float4*>(h1 + k);
      acc = fmaf(W2[(k + 0) * VAD_G + j], hv.x, acc);
      acc = fmaf(W2[(k + 1) * VAD_G + j], hv.y, acc);
      acc = fmaf(W2[(k + 2) * VAD_G + j], hv.z, acc);
      acc = fmaf(W2[(k + 3) * VAD_G + j], hv.w, acc);
    }
    gt[j] = acc;
    __syncthreads();
    if (j < VAD_H) cell(c1, h1);
    __syncthreads();
    if (j < 32) {      // decoder: ReLU, conv 64 -> 1 with bias, sigmoid (the others run ahead into the next step)
      float v = fmaxf(h1[lane], 0.f) * wd0 + fmaxf(h1[32 + lane], 0.f) * wd1;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) probs[w0 + t] = 1.f / (1.f + expf(-(v + bd)));
    }
  }
}

static DevSmemCache g_front_smem, g_rec_smem_v;

}  // namespace svcb

using namespace svcb;

struct svcb_vad {
  VadWeights P;
  const float* wrec = nullptr;   // [3][64][256]
  const float* b1 = nullptr;     // b_ih1 + b_hh1 [256]
  const float* wdec = nullptr;   // decoder conv [64] then its bias
};

extern "C" {

int svcb_vad_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                    svcb_vad** out) {
  if (!dev_blob || !table_host || !out) { set_error("svcb_vad_create: bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_blob_device(dev_blob));
  SVCB_CUDA_CHECK(ensure_dyn_smem(vad_front_kernel, VAD_FRONT_SMEM, g_front_smem));
  SVCB_CUDA_CHECK(ensure_dyn_smem(vad_rec_kernel, VAD_REC_SMEM, g_rec_smem_v));
  BlobTensors t;
  SVCB_TRY(t.read(dev_blob, blob_bytes, table_host, n_entries));
  auto v = std::make_unique<svcb_vad>();
  VadWeights& P = v->P;
  P.basis4 = t.get("vad.basis4", 2 * VAD_NFFT * 128);
  P.nyq = t.get("vad.nyq", 2 * VAD_NFFT);
  P.filt = t.get("vad.filt", 7);
  auto block = [&](const std::string& p, int cin, int cout, bool proj, const float** dw_w, const float** dw_b,
                   const float** pw_w, const float** pw_b, const float** pj_w, const float** pj_b) {
    *dw_w = t.get(p + ".dw_w", (uint64_t)cin * 5);
    *dw_b = t.get(p + ".dw_b", cin);
    *pw_w = t.get(p + ".pw_w", (uint64_t)cout * cin);
    *pw_b = t.get(p + ".pw_b", cout);
    if (proj) {
      *pj_w = t.get(p + ".pj_w", (uint64_t)cout * cin);
      *pj_b = t.get(p + ".pj_b", cout);
    }
  };
  const float* unused[2];
  block("vad.fl", VAD_FEAT, 16, true, &P.fl_dw_w, &P.fl_dw_b, &P.fl_pw_w, &P.fl_pw_b, &P.fl_pj_w, &P.fl_pj_b);
  block("vad.b1", 16, 32, true, &P.b1_dw_w, &P.b1_dw_b, &P.b1_pw_w, &P.b1_pw_b, &P.b1_pj_w, &P.b1_pj_b);
  block("vad.b2", 32, 32, false, &P.b2_dw_w, &P.b2_dw_b, &P.b2_pw_w, &P.b2_pw_b, &unused[0], &unused[1]);
  block("vad.b3", 32, 64, true, &P.b3_dw_w, &P.b3_dw_b, &P.b3_pw_w, &P.b3_pw_b, &P.b3_pj_w, &P.b3_pj_b);
  auto conv = [&](const std::string& p, int c, const float** w, const float** b, const float** bn) {
    *w = t.get(p + ".w", (uint64_t)c * c);
    *b = t.get(p + ".b", c);
    *bn = t.get(p + ".bn", 2 * c);
  };
  conv("vad.e0", 16, &P.e0_w, &P.e0_b, &P.bn0);
  conv("vad.e4", 32, &P.e4_w, &P.e4_b, &P.bn4);
  conv("vad.e8", 32, &P.e8_w, &P.e8_b, &P.bn8);
  conv("vad.e12", 64, &P.e12_w, &P.e12_b, &P.bn12);
  P.wih0t = t.get("vad.wih0t", VAD_H * VAD_G);
  P.b0 = t.get("vad.b0", VAD_G);
  v->wrec = t.get("vad.wrec", 3 * VAD_H * VAD_G);
  v->b1 = t.get("vad.b1sum", VAD_G);
  v->wdec = t.get("vad.dec", VAD_H + 1);
  SVCB_TRY(t.status("vad blob"));
  *out = v.release();
  return SVCB_OK;
}

void svcb_vad_destroy(svcb_vad* v) { delete v; }

int64_t svcb_vad_windows(int64_t n_samples) { return n_samples <= 0 ? 0 : (n_samples + VAD_WIN - 1) / VAD_WIN; }

size_t svcb_vad_workspace_bytes(const svcb_vad* v, int32_t B, int64_t total_windows) {
  if (!v || B <= 0 || total_windows <= 0) return 0;
  return align256((size_t)total_windows * VAD_G * sizeof(float));
}

int svcb_vad_probs(const svcb_vad* v, const float* wav, const int64_t* sample_offsets_host, int32_t B, float* probs_out,
                   float* feat_out, void* ws, size_t ws_bytes, svcb_stream stream) {
  if (!v || !sample_offsets_host) { set_error("svcb_vad_probs: bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged("svcb_vad_probs", sample_offsets_host, B, 0, 0, "samples", nullptr));
  long long total = 0;
  for (int b = 0; b < B; ++b) total += svcb_vad_windows(sample_offsets_host[b + 1] - sample_offsets_host[b]);
  if (total == 0) return SVCB_OK;
  if (!wav || !probs_out) { set_error("svcb_vad_probs: bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_workspace(ws, ws_bytes, svcb_vad_workspace_bytes(v, B, total), "vad"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  float* G = static_cast<float*>(ws);
  SVCB_CUDA_CHECK(ensure_dyn_smem(vad_front_kernel, VAD_FRONT_SMEM, g_front_smem));
  SVCB_CUDA_CHECK(ensure_dyn_smem(vad_rec_kernel, VAD_REC_SMEM, g_rec_smem_v));
  return for_each_pass<VAD_GROUP>(sample_offsets_host, B, svcb_vad_windows, [&](const ItemPass<VAD_GROUP>& it, int) -> int {
    const long long W = it.out[it.n] - it.out[0];
    if (W == 0) return SVCB_OK;
    {
      KernelScope ks("vad_front", s, (double)W * VAD_NF * (2.0 * VAD_FEAT * VAD_NFFT + 4.0 * 16 * VAD_FEAT + 2.0 * VAD_G * VAD_H),
                     (double)W * 4.0 * (VAD_WIN + VAD_G + (feat_out ? VAD_H : 0)));
      vad_front_kernel<<<(unsigned)((W + VAD_WPC - 1) / VAD_WPC), 256, VAD_FRONT_SMEM, s>>>(wav, v->P, it, G, feat_out);
      SVCB_LAUNCH_CHECK("vad_front");
    }
    {
      KernelScope ks("vad_rec", s, (double)W * 2.0 * VAD_G * 3 * VAD_H, (double)W * 4.0 * (VAD_G + 1) + it.n * 4.0 * 3 * VAD_H * VAD_G);
      vad_rec_kernel<<<it.n, 256, VAD_REC_SMEM, s>>>(v->wrec, v->b1, v->wdec, G, probs_out, it);
      SVCB_LAUNCH_CHECK("vad_rec");
    }
    return SVCB_OK;
  });
}

}  // extern "C"

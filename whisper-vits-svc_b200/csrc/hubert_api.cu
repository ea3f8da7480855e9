// HuBERT-Soft content encoder (the `vec` input of the SVC model, 256-d at 50 frames/s) — SURVEY.md §8f-2.
//
// Replaces HubertSoft.units (hubert/hubert_model.py:64-72 -> encode :39-48):
//   pad 40 + 40 -> FeatureExtractor (:75-95: Conv1d(1,512,10,5) -> GroupNorm(512,512) -> GELU, six stride-2 convs + GELU)
//   -> FeatureProjection (:98-109: LayerNorm(512) -> Linear(512,768)) -> x + GELU(pos_conv(x)[..., :-1]) (:112-128:
//   Conv1d(768,768,128, pad 64, groups 16), weight_norm folded by the packer) -> LayerNorm(768) -> 12 x
//   nn.TransformerEncoderLayer(768, 12, 3072, gelu, post-LN) (:131-153) -> Linear(768,256).
// The transformer runs on the PPG extractor's kernels: wgmma GEMMs over bf16 tile images (whisper_gemm.cu), the
// wgmma attention with P fed from registers (whisper_attn_tc.cu: 12 heads of 64, scores / 8), `ln_rows` writing the
// normalised rows both as the next GEMM's A image and as the fp32 residual stream (post-LN).
// Convolutional stem (97 GFLOP per 20 s chunk): conv0 (one input channel, 10 taps) + GroupNorm + GELU in fp32 as two
// passes over the audio (statistics, then normalise-and-pack) that write conv1's im2col tile image directly; the six
// stride-2 convs as wgmma GEMMs over such images — every GEMM's epilogue (6) applies GELU and scatters straight into the NEXT
// conv's image, the last one writes the fp32 time-major rows LayerNorm reads.  flags bit 0 selects the all-fp32 stem
// (`conv1d`, the last conv writing time-major rows through its output strides) for parity work.
// Positional conv (Conv1d(768, 768, 128, groups 16): 9.4 GFLOP per 1000 frames): per group an im2col tile image
// (K = 128 taps x 48 channels) times a [256 (48 used), K] weight image, epilogue 7 = GELU + residual into the group's 48
// columns of the 768-wide rows; flags bit 1 selects the fp32 CUDA-core form (32 `conv1d` launches, 16 ms per 16 x 20 s).
// Ragged batches (svcb_hubert_units_ragged): item b is its first n_b samples, T_b = svcb_hubert_frames(n_b).  Samples past
// n_b read as conv0's zero padding, the GroupNorm statistics cover the item's own conv0 frames, the positional conv
// reads rows past T_b as zeros and attention masks keys past T_b; the stride-2 stem convs are valid convolutions,
// whose first T_b frames never read later ones.  Everything else is row-local, so an item's rows are the bits a lone
// run computes, and the rows past T_b stay finite (attention reads them as V rows times P = 0).
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"

namespace svcb {
constexpr int HB_C = 512, HB_D = 768, HB_H = 12, HB_FF = 3072, HB_OUT = 256, HB_PK = 128, HB_PG = 16, HB_PHALF = 24;
static const int kHbKernels[6] = {3, 3, 3, 3, 2, 2};

struct HLayer {
  const float *wqkv, *bqkv, *wo, *bo, *w1, *b1, *w2, *b2, *ln1g, *ln1b, *ln2g, *ln2b;
};

// GroupNorm(512, 512) = per-(item, channel) normalisation over time, affine, then GELU; in place on [rows][T]
__global__ void __launch_bounds__(256)
groupnorm_gelu_rows_kernel(float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, int C,
                           int T, float eps) {
  __shared__ float red[8];
  const int row = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  float* xr = x + (size_t)row * T;
  auto block_sum = [&](float v) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    __syncthreads();
    if (lane == 0) red[warp] = v;
    __syncthreads();
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += red[i];
    return s;
  };
  float s = 0.f;
  for (int t = tid; t < T; t += 256) s += xr[t];
  const float mean = block_sum(s) / (float)T;
  float q = 0.f;
  for (int t = tid; t < T; t += 256) { const float d = xr[t] - mean; q += d * d; }
  const float rstd = rsqrtf(block_sum(q) / (float)T + eps);
  const float g = __ldg(gamma + row % C) * rstd, b = __ldg(beta + row % C);
  for (int t = tid; t < T; t += 256) {
    const float v = (xr[t] - mean) * g + b;
    xr[t] = 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
  }
}

// ---- conv0 + GroupNorm + GELU + the first im2col image in two passes over the AUDIO instead of three over the 2.1 GB
// conv0 output (conv1d 3.3 + GroupNorm 1.5 + im2col 2.5 ms per 16 x 20 s): conv0 has one input channel and 10 taps, so
// recomputing it costs less than storing it.
// pass 1: mean / rstd of every (item, channel) row of y[b, c, t] = sum_j w[c][j] wav[b][5 t + j - 40].  One CTA = (item,
// octet of channels): a thread loads its 10-sample window once and feeds 8 channels (one channel per CTA was bound by
// load issue: 10 LDG per FMA chain, 1.8 ms per 16 x 20 s).
__global__ void __launch_bounds__(256)
hubert_conv0_stats_kernel(const float* __restrict__ wav, const float* __restrict__ w0, float2* __restrict__ stats, int N,
                          int T0, float eps, const int* __restrict__ lens) {
  __shared__ double red[16][8];
  __shared__ float ws[10][8];
  const int oc = blockIdx.x, b = blockIdx.y, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid < 80) ws[tid >> 3][tid & 7] = __ldg(w0 + (tid >> 3) * HB_C + oc * 8 + (tid & 7));   // packed [1][10][512]
  __syncthreads();
  const float* xb = wav + (size_t)b * N;
  const int Nb = lens ? __ldg(lens + b) : N, T0b = lens ? (Nb + 80 - 10) / 5 + 1 : T0;   // the item's own samples and frames
  double s[8], q[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) { s[e] = 0.0; q[e] = 0.0; }
  for (int t = tid; t < T0b; t += 256) {
    const int i0 = 5 * t - 40;
    float x[10];
#pragma unroll
    for (int j = 0; j < 10; ++j) {
      const int i = i0 + j;
      x[j] = (i >= 0 && i < Nb) ? __ldg(xb + i) : 0.f;
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float y = 0.f;
#pragma unroll
      for (int j = 0; j < 10; ++j) y = fmaf(ws[j][e], x[j], y);
      s[e] += y; q[e] += (double)y * y;
    }
  }
#pragma unroll
  for (int e = 0; e < 8; ++e) {
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) { s[e] += __shfl_xor_sync(0xffffffffu, s[e], off); q[e] += __shfl_xor_sync(0xffffffffu, q[e], off); }
    if (lane == 0) { red[e][warp] = s[e]; red[8 + e][warp] = q[e]; }
  }
  __syncthreads();
  if (tid < 8) {
    double S = 0.0, Q = 0.0;
    for (int i = 0; i < 8; ++i) { S += red[tid][i]; Q += red[8 + tid][i]; }
    const int nf = lens ? (__ldg(lens + b) + 80 - 10) / 5 + 1 : T0;
    const double mean = S / nf, var = Q / nf - mean * mean;
    stats[(size_t)b * HB_C + oc * 8 + tid] = make_float2((float)mean, (float)(1.0 / sqrt((var > 0.0 ? var : 0.0) + (double)eps)));
  }
}

// pass 2: thread = (item, frame t, octet of channels): conv0 again, GroupNorm + GELU, and the bf16 octet stored where
// conv1's im2col image wants frame t: A1[b * T1 + t2][j * 512 + c] = h0[b][c][2 t2 + j]  (tile image of whisper_gemm.cu)
__global__ void __launch_bounds__(128)
hubert_conv0_pack_kernel(const float* __restrict__ wav, const float* __restrict__ w0, const float2* __restrict__ stats,
                         const float* __restrict__ gamma, const float* __restrict__ beta, __nv_bfloat16* __restrict__ img,
                         int N, int T0, int T1, const int* __restrict__ lens) {
  __shared__ float ws[10][8];
  __shared__ float2 aff[8];   // y -> y * aff.x + aff.y  (normalisation and affine folded)
  const int oc = blockIdx.y, b = blockIdx.z, tid = threadIdx.x;
  if (tid < 80) ws[tid >> 3][tid & 7] = __ldg(w0 + (tid >> 3) * HB_C + oc * 8 + (tid & 7));
  if (tid < 8) {
    const int c = oc * 8 + tid;
    const float2 st = stats[(size_t)b * HB_C + c];
    const float g = __ldg(gamma + c) * st.y;
    aff[tid] = make_float2(g, __ldg(beta + c) - st.x * g);
  }
  __syncthreads();
  const int t = blockIdx.x * 128 + tid;
  if (t >= T0) return;
  const float* xb = wav + (size_t)b * N;
  const int Nb = lens ? __ldg(lens + b) : N;
  float x[10];
#pragma unroll
  for (int j = 0; j < 10; ++j) {
    const int i = 5 * t - 40 + j;
    x[j] = (i >= 0 && i < Nb) ? __ldg(xb + i) : 0.f;
  }
  __align__(16) __nv_bfloat16 hv[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    float y = 0.f;
#pragma unroll
    for (int j = 0; j < 10; ++j) y = fmaf(ws[j][e], x[j], y);
    const float v = fmaf(y, aff[e].x, aff[e].y);
    hv[e] = __float2bfloat16_rn(0.5f * v * (1.f + erff(v * 0.70710678118654752440f)));
  }
  const uint4 pk = *reinterpret_cast<const uint4*>(hv);
  constexpr int KT = 3 * HB_C / 64;
  auto put = [&](int t2, int j) {
    if (t2 >= 0 && t2 < T1) {
      const int m = b * T1 + t2, k = j * HB_C + oc * 8;
      *reinterpret_cast<uint4*>(img + ((size_t)(m >> 7) * KT + (k >> 6)) * 8192 + (size_t)((k & 63) >> 3) * 1024 + (size_t)(m & 127) * 8) = pk;
    }
  };
  if (t & 1) put((t - 1) >> 1, 1);
  else { put(t >> 1, 0); put((t >> 1) - 1, 2); }
}

struct HLayout {
  int T[7];            // frames after conv0 .. conv6
  int M;
  size_t bufa, bufb, imgb, stats, posimg, rows, a512, x, y, a, qkv, att, mid, lens, total;   // bufb doubles as the first im2col image
};
static HLayout hubert_layout(int B, int n_samples) {
  HLayout L;
  L.T[0] = (n_samples + 80 - 10) / 5 + 1;
  for (int i = 1; i <= 6; ++i) L.T[i] = L.T[i - 1] >= kHbKernels[i - 1] ? (L.T[i - 1] - kHbKernels[i - 1]) / 2 + 1 : 0;
  const int T = L.T[6];
  L.M = B * T;
  const size_t Mp = ((size_t)L.M + 127) / 128 * 128;
  WsPlan P;
  L.bufa = P.take((size_t)B * HB_C * L.T[0] * 4);
  {  // fp32 stem: ping-pong activations [B, 512, T1]; tensor-core stem: im2col images [ceil(B T_i / 128) * 128][taps * 512] bf16
    const size_t m1 = ((size_t)B * (L.T[1] > 0 ? L.T[1] : 1) + 127) / 128 * 128, m2 = ((size_t)B * (L.T[2] > 0 ? L.T[2] : 1) + 127) / 128 * 128;
    L.bufb = P.take(std::max((size_t)B * HB_C * (L.T[1] > 0 ? L.T[1] : 1) * 4, m1 * 3 * HB_C * 2));
    L.imgb = P.take(m2 * 3 * HB_C * 2);
  }
  L.stats = P.take((size_t)B * HB_C * sizeof(float2));
  L.posimg = P.take(Mp * (size_t)HB_PK * (HB_D / HB_PG) * 2);   // one group's im2col image, K = 128 * 48
  L.rows = P.take((size_t)(L.M > 0 ? L.M : 1) * HB_C * 4);
  L.a512 = P.take(Mp * HB_C * 2);
  L.x = P.take((size_t)(L.M > 0 ? L.M : 1) * HB_D * 4);
  L.y = P.take((size_t)(L.M > 0 ? L.M : 1) * HB_D * 4);
  L.a = P.take(Mp * HB_D * 2);
  L.qkv = P.take((size_t)B * qkv_heads_tp(T > 0 ? T : 1) * 3 * HB_D * 2);
  L.att = P.take(Mp * HB_D * 2);
  L.mid = P.take(Mp * HB_FF * 2);
  L.lens = P.take(ragged_lens_bytes(B));
  L.total = P.off + 4096;
  return L;
}

}  // namespace svcb

using namespace svcb;

struct svcb_hubert {
  int n_layer = 0;
  const float *conv0_w, *gn_g, *gn_b, *conv_w[6], *conv_wimg[6], *fp_lng, *fp_lnb, *fp_w, *fp_b, *pos_w[HB_PG][2], *pos_b, *pos_wimg[HB_PG], *pos_bimg[HB_PG], *norm_g, *norm_b,
      *proj_w, *proj_b;
  std::vector<HLayer> layers;
};

extern "C" {

int svcb_hubert_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                       int32_t n_layer, svcb_hubert** out) {
  if (!dev_blob || !table_host || !out || n_layer < 1 || n_layer > 64) { set_error("svcb_hubert_create: bad argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_blob_device(dev_blob));
  BlobTensors t;
  SVCB_TRY(t.read(dev_blob, blob_bytes, table_host, n_entries));
  auto h = std::make_unique<svcb_hubert>();
  h->n_layer = n_layer;
  const uint64_t C = HB_C, D = HB_D, FF = HB_FF;
  h->conv0_w = t.get("fe.conv0.w", 10 * C);
  h->gn_g = t.get("fe.gn.g", C); h->gn_b = t.get("fe.gn.b", C);
  for (int i = 0; i < 6; ++i) {
    h->conv_w[i] = t.get("fe.conv" + std::to_string(i + 1) + ".w", C * kHbKernels[i] * C);
    h->conv_wimg[i] = t.get("fe.conv" + std::to_string(i + 1) + ".wimg", C * kHbKernels[i] * C / 2);
  }
  h->fp_lng = t.get("fp.ln.g", C); h->fp_lnb = t.get("fp.ln.b", C);
  h->fp_w = t.get("fp.w", D * C / 2); h->fp_b = t.get("fp.b", D);
  for (int g = 0; g < HB_PG; ++g)
    for (int hf = 0; hf < 2; ++hf)
      h->pos_w[g][hf] = t.get("pos." + std::to_string(g) + "." + std::to_string(hf) + ".w", (uint64_t)(D / HB_PG) * HB_PK * HB_PHALF);
  for (int g = 0; g < HB_PG; ++g) {
    h->pos_wimg[g] = t.get("pos." + std::to_string(g) + ".wimg", (uint64_t)256 * HB_PK * (D / HB_PG) / 2);
    h->pos_bimg[g] = t.get("pos." + std::to_string(g) + ".bimg", 256);
  }
  h->pos_b = t.get("pos.b", D);
  h->norm_g = t.get("norm.g", D); h->norm_b = t.get("norm.b", D);
  h->layers.resize(n_layer);
  for (int i = 0; i < n_layer; ++i) {
    const std::string p = "L" + std::to_string(i);
    HLayer& l = h->layers[i];
    l.wqkv = t.get(p + ".wqkv", 3 * D * D / 2); l.bqkv = t.get(p + ".bqkv", 3 * D);
    l.wo = t.get(p + ".wo", D * D / 2); l.bo = t.get(p + ".bo", D);
    l.w1 = t.get(p + ".w1", FF * D / 2); l.b1 = t.get(p + ".b1", FF);
    l.w2 = t.get(p + ".w2", FF * D / 2); l.b2 = t.get(p + ".b2", D);
    l.ln1g = t.get(p + ".ln1.g", D); l.ln1b = t.get(p + ".ln1.b", D);
    l.ln2g = t.get(p + ".ln2.g", D); l.ln2b = t.get(p + ".ln2.b", D);
  }
  h->proj_w = t.get("proj.w", (uint64_t)HB_OUT * D / 2); h->proj_b = t.get("proj.b", HB_OUT);
  SVCB_TRY(t.status("hubert blob"));
  *out = h.release();
  return SVCB_OK;
}

void svcb_hubert_destroy(svcb_hubert* h) { delete h; }

int32_t svcb_hubert_frames(int32_t n_samples) { return n_samples > 0 ? hubert_layout(1, n_samples).T[6] : 0; }

size_t svcb_hubert_workspace_bytes(const svcb_hubert* h, int32_t B, int32_t n_samples) {
  if (!h || B <= 0 || n_samples <= 0) return 0;
  return hubert_layout(B, n_samples).total;
}

}  // extern "C"

// lens_host: null, or per-item sample counts of a ragged batch (flags 0 only)
static int hubert_units(const svcb_hubert* h, const float* wav, float* out, int32_t B, int32_t n_samples, void* ws,
                        size_t ws_bytes, float* const* taps, int32_t flags, const int32_t* lens_host, cudaStream_t s) {
  if (!h || !wav || !out || B <= 0 || n_samples <= 0) { set_error("svcb_hubert_units: bad argument"); return SVCB_E_BAD_SHAPE; }
  const HLayout L = hubert_layout(B, n_samples);
  const int T = L.T[6], M = L.M;
  if (T < 1) { set_error("svcb_hubert_units: audio shorter than one frame"); return SVCB_E_BAD_SHAPE; }
  RaggedLens ragged;   // samples, frames
  SVCB_TRY(ragged.validate(lens_host, B, n_samples, [](int n) { return hubert_layout(1, n).T[6]; }, "svcb_hubert_units_ragged",
                         "samples"));
  SVCB_TRY(check_workspace(ws, ws_bytes, L.total, "hubert"));
  char* base = static_cast<char*>(ws);
  SVCB_TRY(ragged.stage(base + L.lens, s));
  float* bufa = reinterpret_cast<float*>(base + L.bufa);
  float* bufb = reinterpret_cast<float*>(base + L.bufb);
  float* rows = reinterpret_cast<float*>(base + L.rows);
  float* x = reinterpret_cast<float*>(base + L.x);
  float* y = reinterpret_cast<float*>(base + L.y);
  void* a512 = base + L.a512; void* a = base + L.a; void* qkv = base + L.qkv; void* att = base + L.att; void* mid = base + L.mid;
  auto tap = [&](int i, const float* src, size_t n) -> int {
    if (taps && taps[i]) SVCB_CUDA_CHECK(cudaMemcpyAsync(taps[i], src, n * sizeof(float), cudaMemcpyDeviceToDevice, s));
    return SVCB_OK;
  };
  if (flags & 1) {  // conv0 over the zero-padded audio (pad 40 + 40, hubert_model.py:70) -> [B, 512, T0]
    ConvParams p;
    p.x = wav; p.sxb = n_samples; p.sxc = n_samples; p.sxt = 1;
    p.w = h->conv0_w; p.cout_pad = HB_C; p.bias = nullptr;
    p.y = bufa; p.syb = (long long)HB_C * L.T[0]; p.syc = L.T[0]; p.syt = 1;
    p.B = B; p.Cin = 1; p.Cout = HB_C; p.Tin = n_samples; p.K = 10; p.stride = 5; p.pad = 40; p.nq = L.T[0];
    SVCB_TRY(launch_conv1d(p, s));
  }
  if (flags & 1) {
    KernelScope ks("groupnorm_gelu_rows", s, 0.0, 16.0 * B * HB_C * (double)L.T[0]);
    groupnorm_gelu_rows_kernel<<<B * HB_C, 256, 0, s>>>(bufa, h->gn_g, h->gn_b, HB_C, L.T[0], 1e-5f);
    SVCB_LAUNCH_CHECK("groupnorm_gelu_rows");
  }
  if (!(flags & 1)) {
    // conv1 .. conv6 + GELU on the tensor cores: A_i[b * T_i + t][j * 512 + ci] = h_{i-1}[b][ci][2 t + j]
    void* img[2] = {base + L.bufb, base + L.imgb};
    {  // conv0 + GroupNorm + GELU straight into conv1's image (two passes over the audio, see the kernels)
      float2* stats = reinterpret_cast<float2*>(base + L.stats);
      {
        KernelScope ks("hubert_conv0_stats", s, 20.0 * B * HB_C * (double)L.T[0], 4.0 * B * (double)n_samples);
        hubert_conv0_stats_kernel<<<dim3(HB_C / 8, B), 256, 0, s>>>(wav, h->conv0_w, stats, n_samples, L.T[0], 1e-5f, ragged.lens);
        SVCB_LAUNCH_CHECK("hubert_conv0_stats");
      }
      {
        KernelScope ks("hubert_conv0_pack", s, 20.0 * B * HB_C * (double)L.T[0], 4.0 * B * (double)n_samples + 2.0 * B * 3 * HB_C * (double)L.T[1]);
        hubert_conv0_pack_kernel<<<dim3((L.T[0] + 127) / 128, HB_C / 8, B), 128, 0, s>>>(
            wav, h->conv0_w, stats, h->gn_g, h->gn_b, static_cast<__nv_bfloat16*>(img[0]), n_samples, L.T[0], L.T[1], ragged.lens);
        SVCB_LAUNCH_CHECK("hubert_conv0_pack");
      }
    }
    for (int i = 1; i <= 6; ++i) {
      const int K = kHbKernels[i - 1] * HB_C, Mi = B * L.T[i];
      if (i < 6)   // GELU, scattered into conv_{i+1}'s image
        SVCB_TRY(launch_gemm_tc(img[(i - 1) & 1], h->conv_wimg[i - 1], nullptr, img[i & 1], nullptr, Mi, HB_C, K, EPI_GELU_VALID_S2_IMG, s, L.T[i], kHbKernels[i]));
      else         // GELU -> fp32 rows [B * T, 512]
        SVCB_TRY(launch_gemm_tc(img[(i - 1) & 1], h->conv_wimg[i - 1], nullptr, rows, nullptr, Mi, HB_C, K, EPI_GELU_ADD_F32, s));
    }
  }
  const float* cur = bufa;
  for (int i = 1; i <= 6 && (flags & 1); ++i) {   // fp32 stem: conv1 .. conv6 + GELU; the last one writes time-major rows
    float* dst = i == 6 ? rows : (cur == bufa ? bufb : bufa);
    ConvParams p;
    p.x = cur; p.sxb = (long long)HB_C * L.T[i - 1]; p.sxc = L.T[i - 1]; p.sxt = 1;
    p.w = h->conv_w[i - 1]; p.cout_pad = HB_C; p.bias = nullptr;
    p.y = dst;
    if (i == 6) { p.syb = (long long)T * HB_C; p.syc = 1; p.syt = HB_C; }
    else { p.syb = (long long)HB_C * L.T[i]; p.syc = L.T[i]; p.syt = 1; }
    p.B = B; p.Cin = HB_C; p.Cout = HB_C; p.Tin = L.T[i - 1]; p.K = kHbKernels[i - 1]; p.stride = 2; p.pad = 0; p.nq = L.T[i];
    p.act = ACT_GELU;
    SVCB_TRY(launch_conv1d(p, s));
    cur = dst;
  }
  SVCB_TRY(tap(0, rows, (size_t)M * HB_C));
  // FeatureProjection: LayerNorm(512) -> Linear(512, 768)
  SVCB_TRY(launch_ln_rows(rows, h->fp_lng, h->fp_lnb, a512, M, HB_C, true, s));
  SVCB_TRY(launch_gemm_tc(a512, h->fp_w, h->fp_b, x, nullptr, M, HB_D, HB_C, EPI_RESID_F32, s));
  SVCB_TRY(tap(1, x, (size_t)M * HB_D));
  // y = x + GELU(pos_conv(x)[..., :-1]): 16 groups of 48 channels, 128 taps, two 24-channel halves per group
  for (int g = 0; g < HB_PG && !(flags & 2); ++g) {   // tensor cores: per group an im2col image (K = 128 x 48) x [256 (48 used), K]
    const int cg = HB_D / HB_PG, c0 = g * cg;
    SVCB_TRY(launch_im2col_rows_image(x, base + L.posimg, B, T, HB_D, c0, cg, HB_PK, HB_PK / 2, s, ragged.out_lens));
    SVCB_TRY(launch_gemm_tc(base + L.posimg, h->pos_wimg[g], h->pos_bimg[g], y + c0, x + c0, M, 256, HB_PK * cg, EPI_GELU_ADD_F32_LD, s, cg, HB_D));
  }
  for (int g = 0; g < HB_PG && (flags & 2); ++g)       // flags bit 1: fp32 on the CUDA cores
    for (int hf = 0; hf < 2; ++hf) {
      const int ci0 = g * (HB_D / HB_PG), co0 = ci0 + hf * HB_PHALF;
      ConvParams p;
      p.x = x + ci0; p.sxb = (long long)T * HB_D; p.sxc = 1; p.sxt = HB_D;
      p.w = h->pos_w[g][hf]; p.cout_pad = HB_PHALF; p.bias = h->pos_b + co0;
      p.y = y + co0; p.syb = (long long)T * HB_D; p.syc = 1; p.syt = HB_D;
      p.res = x + co0;
      p.B = B; p.Cin = HB_D / HB_PG; p.Cout = HB_PHALF; p.Tin = T; p.K = HB_PK; p.stride = 1; p.pad = HB_PK / 2; p.nq = T;
      p.act = ACT_GELU;
      SVCB_TRY(launch_conv1d(p, s));
    }
  SVCB_TRY(launch_ln_rows(y, h->norm_g, h->norm_b, a, M, HB_D, true, s, x));
  SVCB_TRY(tap(2, x, (size_t)M * HB_D));
  if (qkv_heads_tp(T) != T) SVCB_CUDA_CHECK(cudaMemsetAsync(qkv, 0, (size_t)B * qkv_heads_tp(T) * 3 * HB_D * 2, s));
  for (int i = 0; i < h->n_layer; ++i) {   // post-LN layers: x = LN1(x + SA(x)); x = LN2(x + W2 gelu(W1 x))
    const HLayer& l = h->layers[i];
    SVCB_TRY(launch_gemm_tc(a, l.wqkv, l.bqkv, qkv, nullptr, M, 3 * HB_D, HB_D, EPI_QKV_HEADS, s, T));
    SVCB_TRY(launch_whisper_attention_tc(qkv, att, B, T, HB_D, HB_H, 0, s, ragged.out_lens));
    SVCB_TRY(launch_gemm_tc(att, l.wo, l.bo, y, x, M, HB_D, HB_D, EPI_RESID_F32, s));
    SVCB_TRY(launch_ln_rows(y, l.ln1g, l.ln1b, a, M, HB_D, true, s, x));
    SVCB_TRY(launch_gemm_tc(a, l.w1, l.b1, mid, nullptr, M, HB_FF, HB_D, EPI_GELU_BF16_IMAGE, s));
    SVCB_TRY(launch_gemm_tc(mid, l.w2, l.b2, y, x, M, HB_D, HB_FF, EPI_RESID_F32, s));
    SVCB_TRY(launch_ln_rows(y, l.ln2g, l.ln2b, a, M, HB_D, true, s, x));
    if (i == 0) SVCB_TRY(tap(3, x, (size_t)M * HB_D));
  }
  SVCB_TRY(tap(4, x, (size_t)M * HB_D));
  SVCB_TRY(launch_gemm_tc(a, h->proj_w, h->proj_b, out, nullptr, M, HB_OUT, HB_D, EPI_RESID_F32, s));
  return ragged.zero_tail(out, T, HB_OUT, s);
}

extern "C" {

int svcb_hubert_units(const svcb_hubert* h, const float* wav, float* out, int32_t B, int32_t n_samples, void* ws,
                      size_t ws_bytes, float* const* taps, int32_t flags, svcb_stream stream) {
  return hubert_units(h, wav, out, B, n_samples, ws, ws_bytes, taps, flags, nullptr, static_cast<cudaStream_t>(stream));
}

int svcb_hubert_units_ragged(const svcb_hubert* h, const float* wav, const int32_t* n_samples_host, float* out, int32_t B,
                             int32_t n_samples, void* ws, size_t ws_bytes, svcb_stream stream) {
  if (!n_samples_host) { set_error("svcb_hubert_units_ragged: null lengths"); return SVCB_E_BAD_SHAPE; }
  return hubert_units(h, wav, out, B, n_samples, ws, ws_bytes, nullptr, 0, n_samples_host, static_cast<cudaStream_t>(stream));
}

}  // extern "C"

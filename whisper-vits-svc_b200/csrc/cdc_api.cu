// Cutting the two lowest STFT bins out of raw recordings (prepare/preprocess_cdc.py:16-27, cut_direct_content) on the
// device.
//
//   cdc   torch.istft(stft with bins 0 and 1 set to zero) of a 1024 / 256 periodic-Hann STFT (center, reflect padding
//         of 512), then x 32768, clamp to [-32768, 32767] and truncation to int16
//
// No transform is taken.  Zeroing bins 0 and 1 of frame f's onesided spectrum X_f subtracts
//   c_f(m) = (Re X0_f + 2 Re(X1_f e^{2 pi i m / 1024})) / 1024 = A0_f / 1024 + (A1_f cos + S_f sin)(2 pi m / 1024) / 512
// from its irfft, with A0 = sum w xp, A1 = sum w xp cos, S = sum w xp sin over the frame's 1024 reflect-padded samples xp.
// The rest of the round trip is the identity wherever the window envelope is non-zero, so padded sample p becomes
//   y(p) = xp(p) - sum_f w(m) c_f(m) / sum_f w(m)^2,   m = p - 256 f,
// over the <= 4 frames covering p; outputs are p = 512 .. 512 + 256 (n / 256) - 1.  Tables, sums and the division are
// fp64, and y is rounded once to fp32 before the int16 step, as the reference's float32 istft output is.
//
// Ragged batches: each pass of up to CDC_GROUP items rides in the kernel parameters (ItemPass, in samples and out in
// hops of 256 outputs).  A CTA takes CDC_TH consecutive hops of the pass, which may straddle items, computes the
// coefficients of every frame they need, then writes their samples.  A frame's coefficients and an output depend on
// their own item only and come from the same instructions in any tile, so a ragged batch is bitwise equal to each item
// run alone.
#include <cstdint>
#include <string>

#include "common.cuh"

namespace svcb {

constexpr int CDC_N = 1024, CDC_HOP = 256, CDC_PAD = CDC_N / 2;
constexpr int CDC_THREADS = CDC_HOP;    // thread r writes sample r of every hop of the tile
constexpr int CDC_WARPS = CDC_THREADS / 32;
constexpr int CDC_TH = 61;              // hops per CTA: inside one item they need 61 + 3 = 64 frames, 8 per warp
constexpr int CDC_SLOTS = 4 * CDC_TH;   // frames a tile can need: a run of k hops of one item needs at most k + 3
constexpr int CDC_GROUP = 128;          // items per pass

// grid ceil(hops / CDC_TH), CDC_THREADS threads.  Item b has n_b samples, H_b = n_b / 256 output hops and H_b + 1
// frames; its local hop q (samples 256 q .. 256 q + 255 of its output, padded samples 256 (q + 2) + r) is covered by
// frames q - 1 .. q + 2 that exist (0 .. H_b).  out: item b's hops start at hop it.out[b] of the batch.
__global__ void __launch_bounds__(CDC_THREADS)
cdc_kernel(const float* __restrict__ x, int16_t* __restrict__ out, ItemPass<CDC_GROUP> it) {
  __shared__ double gw[CDC_N], gc[CDC_N], gs[CDC_N];   // w(m), w(m) cos(2 pi m / 1024), w(m) sin(2 pi m / 1024)
  __shared__ double coef[CDC_SLOTS][3];                 // per frame slot: A0 / 1024, A1 / 512, S / 512
  // runs of the tile's hops that share an item: the item, its first frame and that frame's slot (seg_slot[n_seg] =
  // slots in all)
  __shared__ int seg_b[CDC_TH], seg_f0[CDC_TH], seg_slot[CDC_TH + 1];
  __shared__ int n_seg;
  // per hop of the tile: its item's input offset + 256 q, the slot of frame q - 1, and 1 | 2 for the item's first |
  // last hop (no frame q - 1 | q + 2)
  __shared__ long long hop_x[CDC_TH];
  __shared__ int hop_slot[CDC_TH], hop_edge[CDC_TH];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const long long h0 = it.out[0] + (long long)blockIdx.x * CDC_TH, h1 = min(h0 + CDC_TH, it.out[it.n]);
  for (int m = tid; m < CDC_N; m += CDC_THREADS) {
    double s, c;
    sincospi((double)m / (CDC_N / 2), &s, &c);
    const double w = 0.5 - 0.5 * c;   // periodic Hann
    gw[m] = w;
    gc[m] = w * c;
    gs[m] = w * s;
  }
  if (tid == 0) {
    int b = item_of(it.out, h0), s = 0, slot = 0;
    for (long long h = h0; h < h1; ++s, ++b) {
      const long long hb = it.out[b + 1] - it.out[b], q0 = h - it.out[b], q1 = min(h1, it.out[b + 1]) - it.out[b];
      const long long f0 = max(q0 - 1, 0ll), f1 = min(q1 + 1, hb);
      seg_b[s] = b;
      seg_f0[s] = (int)f0;
      seg_slot[s] = slot;
      slot += (int)(f1 - f0 + 1);
      h = it.out[b] + q1;
    }
    n_seg = s;
    seg_slot[s] = slot;
  }
  __syncthreads();
  if (tid < CDC_TH && h0 + tid < h1) {
    const long long gh = h0 + tid;
    int s = 0;
    while (gh >= it.out[seg_b[s] + 1]) ++s;
    const int b = seg_b[s];
    const long long q = gh - it.out[b];
    hop_x[tid] = it.in[b] + CDC_HOP * q;
    hop_slot[tid] = seg_slot[s] + (int)(q - 1 - seg_f0[s]);
    hop_edge[tid] = (q == 0 ? 1 : 0) | (q == it.out[b + 1] - it.out[b] - 1 ? 2 : 0);
  }
  // one warp per frame slot: three fp64 dot products over the frame's reflect-padded samples
  const int n_slot = seg_slot[n_seg];
  for (int slot = warp; slot < n_slot; slot += CDC_WARPS) {
    int s = 0;
    while (seg_slot[s + 1] <= slot) ++s;
    const int b = seg_b[s];
    const long long f = seg_f0[s] + (slot - seg_slot[s]), N = it.in[b + 1] - it.in[b];
    const float* xb = x + it.in[b];
    double a0 = 0.0, a1 = 0.0, a2 = 0.0;
#pragma unroll 4
    for (int m = lane; m < CDC_N; m += 32) {
      long long p = CDC_HOP * f - CDC_PAD + m;   // reflect padding; N > 512 keeps one reflection in range
      if (p < 0) p = -p;
      if (p >= N) p = 2 * (N - 1) - p;
      const double v = (double)__ldg(xb + p);
      a0 = fma(gw[m], v, a0);
      a1 = fma(gc[m], v, a1);
      a2 = fma(gs[m], v, a2);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a0 += __shfl_xor_sync(0xffffffffu, a0, o);
      a1 += __shfl_xor_sync(0xffffffffu, a1, o);
      a2 += __shfl_xor_sync(0xffffffffu, a2, o);
    }
    if (lane == 0) {
      coef[slot][0] = a0 * (1.0 / CDC_N);
      coef[slot][1] = a1 * (2.0 / CDC_N);
      coef[slot][2] = a2 * (2.0 / CDC_N);
    }
  }
  // frame q - 1 + j reaches sample r of hop q at m = 256 (3 - j) + r
  double tw[4], tc[4], ts[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int m = CDC_HOP * (3 - j) + tid;
    tw[j] = gw[m];
    tc[j] = gc[m];
    ts[j] = gs[m];
  }
  // 1 / the window envelope: all four frames, none before the first hop, none after the last (w(256 + r) > 0 and
  // w(512 + r) > 0, so no envelope is zero)
  const double e01 = tw[0] * tw[0] + tw[1] * tw[1], e2 = tw[2] * tw[2], e3 = tw[3] * tw[3];
  const double inv_mid = 1.0 / (e01 + e2 + e3), inv_first = 1.0 / (tw[1] * tw[1] + e2 + e3), inv_last = 1.0 / (e01 + e2);
  __syncthreads();
  for (int k = 0; k < CDC_TH && h0 + k < h1; ++k) {
    const int edge = hop_edge[k];
    const double(*c)[3] = coef + hop_slot[k];
    double num = 0.0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if ((j == 0 && (edge & 1)) || (j == 3 && (edge & 2))) continue;
      num = fma(c[j][0], tw[j], num);
      num = fma(c[j][1], tc[j], num);
      num = fma(c[j][2], ts[j], num);
    }
    const double inv = (edge & 1) ? inv_first : (edge & 2) ? inv_last : inv_mid;
    const double y = (double)__ldg(x + hop_x[k] + tid) - num * inv;
    const float v = fminf(fmaxf(__double2float_rn(y) * 32768.f, -32768.f), 32767.f);   // x 32768 is exact
    out[CDC_HOP * (h0 + k) + tid] = (int16_t)__float2int_rz(v);
  }
}

}  // namespace svcb

using namespace svcb;

extern "C" {

int svcb_cdc_ragged(const float* x, const int64_t* offsets_host, int32_t B, int16_t* out, svcb_stream stream) {
  static const char* who = "svcb_cdc_ragged";
  if (!x || !out || !offsets_host) { set_error(std::string(who) + ": null pointer"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_ragged(who, offsets_host, B, 1, CDC_PAD + 1, "samples",
                        "torch.stft's reflect padding of 512 needs more than 512 samples"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  return for_each_pass<CDC_GROUP>(offsets_host, B, [](long long n) { return n / CDC_HOP; },
                                  [&](const ItemPass<CDC_GROUP>& it, int) -> int {
    const long long hops = it.out[it.n] - it.out[0], frames = hops + it.n;
    KernelScope ks("cdc", s, 2.0 * 3 * CDC_N * (double)frames + 2.0 * 12 * CDC_HOP * (double)hops,
                   4.0 * (double)(it.in[it.n] - it.in[0]) + 2.0 * CDC_HOP * (double)hops);
    cdc_kernel<<<(unsigned)((hops + CDC_TH - 1) / CDC_TH), CDC_THREADS, 0, s>>>(x, out, it);
    SVCB_LAUNCH_CHECK("cdc");
    return SVCB_OK;
  });
}

}  // extern "C"

// Whole AMP block fused in shared memory — for the narrow generator stages (C = 20, 10).
//
// Replaces one AMPBlock.forward (vits_decoder/bigv.py:50-58): three units of
//   x = x + conv2(SnakeAlias(conv1_d(SnakeAlias(x))))                d = 1, 3, 5
// i.e. 6 Conv1d + 6 SnakeAlias (vits_decoder/alias/act.py:124-128) + 3 residual adds, plus the
// stage-mean bookkeeping of generator.py:188-194, in ONE kernel: x is read once, the result is
// written once (SURVEY.md §8a row a9 "per-block fused kernel", row a10).
//
// Why CUDA cores here: with C = 10 / 20 a tensor-core MMA has N = 16 / 32 and costs as much issue time
// as a full-width one (measured: these two stages took 75 of 107 ms of the tensor-core AMP path
// while holding 20 % of its FLOPs — profiles/r01_notes.md); their arithmetic intensity unfused is
// ~45-330 FLOP/B (fp32-FMA side of the ridge).  Fused, the stage is bound by fp32 FMA issue and
// exact fp32 — no operand splitting.
//
// One CTA = (item, TOUT output samples) with a halo H = sum over units of the receptive field
// (6 + d(K-1)/2 + 6 + (K-1)/2).  Three [C][W] buffers live in shared memory (X residual stream,
// Y, Z) with zeroed guard bands so the convolutions need no bounds checks; positions outside the
// sequence are kept at zero (= the convs' zero padding) and SnakeAlias clamps its taps to the
// sequence (= its replicate padding), so tile edges reproduce the reference exactly.
#include <cstdio>
#include <cstdlib>

#include "common.cuh"

namespace svcb {

constexpr int AB_GUARD = 32;   // zeroed floats on both sides of every row (>= max conv reach 25)

__host__ __device__ inline int ab_halo(int K, const int* dil) {
  int h = 0;
  for (int d = 0; d < 3; ++d) h += 6 + dil[d] * (K - 1) / 2 + 6 + (K - 1) / 2;
  return h;
}

template <int C, int V>
struct AbCfg {
  static constexpr int CP = (C + 3) / 4 * 4;
  // The buffer width W (tile + both halos) is fixed so that the convolution's NT*THREADS time slots
  // are exactly filled (a 1216-wide buffer on 2x512 slots wasted 40 % of the FMA issue, r01 profile);
  // the number of output samples per CTA follows from the block's receptive field: TOUT = W - 2H.
  // Variant 1 trades threads for a taller register tile (NT x C accumulators per thread: every
  // weight vector load then feeds NT*4 FMAs) — C=10: 3 x 512 slots (W=1536, also a smaller halo
  // share), C=20: 3 x 256 (same W; shared memory holds no more).
  static constexpr int THREADS = C <= 10 ? 512 : (V == 0 ? 384 : 256);
  static constexpr int NT = V == 0 ? 2 : 3;              // time steps per thread in the convolution
  static constexpr int W = NT * THREADS;                 // V0: 1024 (C=10) / 768 (C=20); V1: 1536 / 768
  static constexpr int ROWS8 = (C <= 10 && V == 0) ? 8 : C;   // Snake rows done in 8-sample runs (rest: 4)
};

// SnakeAlias of src rows -> dst rows over buffer positions [0, W); lo_i / hi_i = first / last buffer
// index inside the sequence.  Register-resident: a thread owns R consecutive outputs of one channel,
// loads the R+16 inputs around them with 16-byte shared loads, forms the 2(R+6) up-sampled Snake
// values in registers and decimates them — no scratch buffer, no barrier, and R+6 independent
// dependency chains per thread (the earlier warp-private version ran one 12-deep FMA chain per
// thread on 12 resident warps and was latency-bound: profiles/r01_notes.md §7).
//   position a = n0-3+p (p in [0,R+6)):  u[2a]   = 2*sum_{d=0..5} x[a-3+d] f[11-2d]
//                                        u[2a+1] = 2*sum_{d=1..6} x[a-3+d] f[12-2d]
//   v = u + sin^2(u e^alpha) / (e^beta + 1e-9);   out[n] = sum_{k<12} v[2n-5+k] f[k]
// (alias/resample.py:25-33, alias/act.py:79-92, alias/filter.py:86-94).  Runs that touch the
// sequence ends take a scalar path with the replicate-padding clamps.
template <int R>
__device__ __forceinline__ void ab_snake_run(const float* __restrict__ xr, float* __restrict__ dr, int n0,
                                             const float (&fu)[12], const float (&fdn)[12],
                                             const float* f_up, const float* f_dn, float a_, float b_,
                                             int lo_i, int hi_i, bool seq_lo, bool seq_hi) {
  // the clamped path is only needed where a tap crosses a real sequence end; at a mere tile edge the
  // guard band is read instead — those outputs lie in the halo and are never used
  if (!((seq_lo && n0 - 6 < lo_i) || (seq_hi && n0 + R + 5 > hi_i))) {
    float x[R + 16];  // xr[n0-8 .. n0+R+8)
#pragma unroll
    for (int q = 0; q < (R + 16) / 4; ++q) {
      const float4 t4 = *reinterpret_cast<const float4*>(xr + n0 - 8 + 4 * q);
      x[4 * q] = t4.x; x[4 * q + 1] = t4.y; x[4 * q + 2] = t4.z; x[4 * q + 3] = t4.w;
    }
    float vv[2 * R + 12];
#pragma unroll
    for (int p = 0; p < R + 6; ++p) {
      float ue = x[p + 2] * fu[11];
      ue = fmaf(x[p + 3], fu[9], ue); ue = fmaf(x[p + 4], fu[7], ue); ue = fmaf(x[p + 5], fu[5], ue);
      ue = fmaf(x[p + 6], fu[3], ue); ue = fmaf(x[p + 7], fu[1], ue);
      float uo = x[p + 3] * fu[10];
      uo = fmaf(x[p + 4], fu[8], uo); uo = fmaf(x[p + 5], fu[6], uo); uo = fmaf(x[p + 6], fu[4], uo);
      uo = fmaf(x[p + 7], fu[2], uo); uo = fmaf(x[p + 8], fu[0], uo);
      const float se = snake_sin(ue * a_), so = snake_sin(uo * a_);   // (the x2 gain is folded into fu: exact)
      vv[2 * p] = fmaf(b_, se * se, ue);
      vv[2 * p + 1] = fmaf(b_, so * so, uo);
    }
    float o[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      float acc = 0.f;
#pragma unroll
      for (int k = 0; k < 12; ++k) acc = fmaf(vv[2 * i + 1 + k], fdn[k], acc);
      o[i] = acc;
    }
#pragma unroll
    for (int q = 0; q < R / 4; ++q)
      *reinterpret_cast<float4*>(dr + n0 + 4 * q) = make_float4(o[4 * q], o[4 * q + 1], o[4 * q + 2], o[4 * q + 3]);
  } else {
    const int mlo = 2 * lo_i, mhi = 2 * hi_i + 1;
    for (int i = 0; i < R; ++i) {
      const int n = n0 + i;
      float acc = 0.f;
      if (n >= lo_i && n <= hi_i) {
        for (int k = 0; k < 12; ++k) {
          const int m = min(max(2 * n - 5 + k, mlo), mhi);
          const int a = m >> 1, q = m & 1;
          float u = 0.f;
          for (int d = q; d < q + 6; ++d) u = fmaf(xr[min(max(a - 3 + d, lo_i), hi_i)], f_up[11 + q - 2 * d], u);
          u *= 2.f;
          const float sn = snake_sin(u * a_);
          acc = fmaf(fmaf(b_, sn * sn, u), f_dn[k], acc);
        }
      }
      dr[n] = acc;  // zero outside the sequence = zero padding of the next conv
    }
  }
}

// Rows [0, ROWS8) are covered by 8-sample runs and the remaining rows by 4-sample runs, chosen so
// that both task counts are whole multiples of the CTA size (C=20: 20 rows x 96 runs = 5 x 384;
// C=10: 8 x 128 = 2 x 512 and 2 x 256 = 512) — no partially filled pass.
template <int C, int V>
__device__ __forceinline__ void ab_snake(const float* __restrict__ src, float* __restrict__ dst,
                                         const float* f_up, const float* f_dn, const float* ea,
                                         const float* ib, int lo_i, int hi_i, bool seq_lo, bool seq_hi, int tid) {
  constexpr int AB_THREADS = AbCfg<C, V>::THREADS;
  constexpr int W = AbCfg<C, V>::W, WS = W + 2 * AB_GUARD;
  constexpr int ROWS8 = AbCfg<C, V>::ROWS8;
  constexpr int T8 = ROWS8 * (W / 8), T4 = (C - ROWS8) * (W / 4);
  static_assert(V != 0 || (T8 % AB_THREADS == 0 && T4 % AB_THREADS == 0), "Snake passes must be exactly filled");
  float fu[12], fdn[12];
#pragma unroll
  for (int k = 0; k < 12; ++k) { fu[k] = 2.f * f_up[k]; fdn[k] = f_dn[k]; }  // UpSample1d's ratio gain (resample.py:31)
  for (int task = tid; task < T8; task += AB_THREADS) {
    const int c = task / (W / 8), n0 = (task - c * (W / 8)) * 8;
    ab_snake_run<8>(src + c * WS + AB_GUARD, dst + c * WS + AB_GUARD, n0, fu, fdn, f_up, f_dn, ea[c], ib[c], lo_i, hi_i, seq_lo, seq_hi);
  }
  for (int task = tid; task < T4; task += AB_THREADS) {
    const int c = ROWS8 + task / (W / 4), n0 = (task % (W / 4)) * 4;
    ab_snake_run<4>(src + c * WS + AB_GUARD, dst + c * WS + AB_GUARD, n0, fu, fdn, f_up, f_dn, ea[c], ib[c], lo_i, hi_i, seq_lo, seq_hi);
  }
}

// dst[co][t] = bias[co] + sum_ci sum_j w[ci][j][co] * src[ci][t + j*dil - P]  (+ dst[co][t] if RES);
// a thread owns NT time steps (t + i*AB_THREADS) so every weight vector load feeds NT*C FMAs.
template <int C, int K, bool RES, int V>
__device__ __forceinline__ void ab_conv(const float* __restrict__ src, float* __restrict__ dst,
                                        const float* __restrict__ wsm, const float* __restrict__ bsm,
                                        int dil, int W, int WS, int lo_i, int hi_i, int tid) {
  constexpr int CP = AbCfg<C, V>::CP;
  constexpr int NT = AbCfg<C, V>::NT;
  constexpr int AB_THREADS = AbCfg<C, V>::THREADS;
  const int P = dil * (K - 1) / 2;
  for (int tb = tid; tb < W; tb += NT * AB_THREADS) {
    float acc[NT][CP];
    int toff[NT];
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      const int t = tb + i * AB_THREADS;
      toff[i] = (t < W ? t : tb) - P + AB_GUARD;
#pragma unroll
      for (int co = 0; co < CP; ++co) acc[i][co] = co < C ? bsm[co] : 0.f;
    }
#pragma unroll 2
    for (int ci = 0; ci < C; ++ci) {
      const float* sr = src + ci * WS;
      const float* wr = wsm + ci * K * CP;
#pragma unroll
      for (int j = 0; j < K; ++j) {
        float xv[NT];
#pragma unroll
        for (int i = 0; i < NT; ++i) xv[i] = sr[toff[i] + j * dil];
        const float4* w4 = reinterpret_cast<const float4*>(wr + j * CP);
#pragma unroll
        for (int q = 0; q < CP / 4; ++q) {
          const float4 w = w4[q];
#pragma unroll
          for (int i = 0; i < NT; ++i) {
            acc[i][4 * q + 0] = fmaf(xv[i], w.x, acc[i][4 * q + 0]);
            acc[i][4 * q + 1] = fmaf(xv[i], w.y, acc[i][4 * q + 1]);
            acc[i][4 * q + 2] = fmaf(xv[i], w.z, acc[i][4 * q + 2]);
            acc[i][4 * q + 3] = fmaf(xv[i], w.w, acc[i][4 * q + 3]);
          }
        }
      }
    }
#pragma unroll
    for (int i = 0; i < NT; ++i) {
      const int t = tb + i * AB_THREADS;
      if (t < W) {
        const bool inside = t >= lo_i && t <= hi_i;
#pragma unroll
        for (int co = 0; co < C; ++co) {
          float* d = dst + co * WS + AB_GUARD + t;
          float o = acc[i][co];
          if (RES) o += *d;
          *d = inside ? o : 0.f;
        }
      }
    }
  }
}

template <int C, int K, int V>
__global__ void __launch_bounds__(AbCfg<C, V>::THREADS, 1)
amp_block_fused_kernel(const AmpBlockParams p) {
  constexpr int AB_THREADS = AbCfg<C, V>::THREADS;
  constexpr int CP = AbCfg<C, V>::CP;
  constexpr int W = AbCfg<C, V>::W;
  extern __shared__ __align__(16) float ab_smem[];
  __shared__ float f_up[12], f_dn[12], s_ea[C], s_ib[C], s_bias[CP];
  const int tid = threadIdx.x;
  const int b = blockIdx.y;
  const int H = ab_halo(K, p.dil);
  const int TOUT = W - 2 * H;
  const int t0 = blockIdx.x * TOUT;
  constexpr int WS = W + 2 * AB_GUARD;
  float* X = ab_smem;
  float* Y = X + C * WS;
  float* Z = Y + C * WS;
  float* wsm = Z + C * WS;                     // [C][K][CP]
  const int base = t0 - H;                     // sequence position of buffer index 0
  const int lo_i = max(0, -base), hi_i = min(W - 1, p.L - 1 - base);
  const bool seq_lo = base <= 0, seq_hi = base + W >= p.L;  // does the buffer contain a sequence end?

  // zero everything once (guard bands must stay zero), then load x
  for (int i = tid; i < 3 * C * WS; i += AB_THREADS) X[i] = 0.f;
  __syncthreads();
  const float* xb = p.x + (long long)b * C * p.L;
  for (int i = tid; i < C * W; i += AB_THREADS) {
    const int c = i / W, n = i - c * W;
    if (n >= lo_i && n <= hi_i) X[c * WS + AB_GUARD + n] = __ldg(xb + (long long)c * p.L + base + n);
  }
  __syncthreads();

  for (int d = 0; d < 3; ++d) {
    for (int half = 0; half < 2; ++half) {
      const int a = 2 * d + half;
      // stage this link's parameters: Snake a, conv (half == 0 ? c1[d] : c2[d])
      if (tid < 12) { f_up[tid] = __ldg(p.fu[a] + tid); f_dn[tid] = __ldg(p.fd[a] + tid); }
      if (tid >= 32 && tid < 32 + C) { s_ea[tid - 32] = __ldg(p.ea[a] + tid - 32); s_ib[tid - 32] = __ldg(p.ib[a] + tid - 32); }
      const float* wg = half == 0 ? p.w1[d] : p.w2[d];
      const float* bg = half == 0 ? p.b1[d] : p.b2[d];
      if (tid >= 64 && tid < 64 + CP) s_bias[tid - 64] = (tid - 64 < C) ? __ldg(bg + tid - 64) : 0.f;
      for (int i = tid; i < C * K * CP; i += AB_THREADS) {
        // packed global layout [ci][j][CoutPad8] -> [ci][j][CP]
        const int co = i % CP, cj = i / CP;
        wsm[i] = co < p.cout_pad ? __ldg(wg + (long long)cj * p.cout_pad + co) : 0.f;
      }
      __syncthreads();
      ab_snake<C, V>(half == 0 ? X : Z, Y, f_up, f_dn, s_ea, s_ib, lo_i, hi_i, seq_lo, seq_hi, tid);
      __syncthreads();
      if (half == 0) ab_conv<C, K, false, V>(Y, Z, wsm, s_bias, p.dil[d], W, WS, lo_i, hi_i, tid);
      else ab_conv<C, K, true, V>(Y, X, wsm, s_bias, 1, W, WS, lo_i, hi_i, tid);
      __syncthreads();
    }
  }
  // write the exact region, folding the stage mean (generator.py:188-194)
  float* yb = p.y + (long long)b * C * p.L;
  for (int i = tid; i < C * TOUT; i += AB_THREADS) {
    const int c = i / TOUT, n = i - c * TOUT;
    const int t = t0 + n;
    if (t < p.L) {
      float o = X[c * WS + AB_GUARD + H + n];
      const long long off = (long long)c * p.L + t;
      if (p.accum) o += yb[off];
      if (p.out_div != 0.f) { asm volatile(""); o = o / p.out_div; }  // keep a uniform branch (no if-converted x/0)
      yb[off] = o;
    }
  }
}

template <int C, int K, int V>
static int launch_ab(const AmpBlockParams& p, cudaStream_t s) {
  constexpr int AB_THREADS = AbCfg<C, V>::THREADS;
  const int H = ab_halo(p.K, p.dil);
  const int W = AbCfg<C, V>::W, WS = W + 2 * AB_GUARD, TOUT = W - 2 * H;
  if (TOUT < 64) { set_error("amp_block_fused: receptive field too large for the tile"); return SVCB_E_UNSUPPORTED; }
  const size_t smem = ((size_t)3 * C * WS + (size_t)C * p.K * AbCfg<C, V>::CP) * sizeof(float);
  if (smem > 227 * 1024 - 1024) { set_error("amp_block_fused: tile does not fit shared memory"); return SVCB_E_UNSUPPORTED; }
  static DevSmemCache attr_cache;
  SVCB_CUDA_CHECK(ensure_dyn_smem(amp_block_fused_kernel<C, K, V>, smem, attr_cache));
  dim3 grid((p.L + TOUT - 1) / TOUT, p.B);
  char kname[64];
  snprintf(kname, sizeof(kname), "amp_block_fused_c%dk%d", C, p.K);
  KernelScope ks(kname, s, 2.0 * 6 * C * C * p.K * (double)p.L * p.B, (p.accum ? 12.0 : 8.0) * C * (double)p.L * p.B,
                 6 * 70.0 * C * (double)p.L * p.B);
  amp_block_fused_kernel<C, K, V><<<grid, AB_THREADS, smem, s>>>(p);
  SVCB_LAUNCH_CHECK("amp_block_fused");
  return SVCB_OK;
}

bool amp_block_fused_supported(int C, int K, const int* dil) {
  if (C != 10 && C != 20) return false;
  if (K != 3 && K != 7 && K != 11) return false;
  for (int d = 0; d < 3; ++d) if (dil[d] * (K - 1) / 2 > AB_GUARD) return false;
  return true;
}

int launch_amp_block_fused(const AmpBlockParams& p, cudaStream_t s) {
  if (p.B <= 0 || p.L <= 0) return SVCB_OK;
  if (!amp_block_fused_supported(p.C, p.K, p.dil)) { set_error("amp_block_fused: unsupported channel count / reach"); return SVCB_E_UNSUPPORTED; }
  // variant 1 (the 3-step tile) for C = 10, measured 9 % faster there; for C = 20 it gained nothing
  if (p.C == 10) return p.K == 3 ? launch_ab<10, 3, 1>(p, s) : p.K == 7 ? launch_ab<10, 7, 1>(p, s) : launch_ab<10, 11, 1>(p, s);
  return p.K == 3 ? launch_ab<20, 3, 0>(p, s) : p.K == 7 ? launch_ab<20, 7, 0>(p, s) : launch_ab<20, 11, 0>(p, s);
}

}  // namespace svcb

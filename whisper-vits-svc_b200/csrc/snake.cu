// Stand-alone anti-aliased Snake (SnakeAlias) — fp32, one pass over [B,C,L].
//
// Replaces SnakeAlias.forward (vits_decoder/alias/act.py:124-128):
//   UpSample1d   (alias/resample.py:25-33): replicate-pad 5/5, depthwise ConvTranspose1d with the
//                12-tap Kaiser-sinc, stride 2, times 2, crop 15/15
//   SnakeBeta    (alias/act.py:79-92, log-scale): v = u + sin^2(u*e^alpha) / (e^beta + 1e-9)
//   DownSample1d (alias/filter.py:86-94): replicate-pad 5/6, depthwise 12-tap conv, stride 2
// in closed form (SURVEY.md §8a row a10):
//   u[2a]   = 2 * sum_{d=-3..2} x[clamp(a+d)] * fu[5-2d]
//   u[2a+1] = 2 * sum_{d=-2..3} x[clamp(a+d)] * fu[6-2d]
//   out[n]  = sum_{k=0..11} v[clamp(2n+k-5, 0, 2L-1)] * fd[k]
// The 2L-long intermediate lives only in shared memory.
#include "common.cuh"

namespace svcb {

constexpr int SA_TL = 1024;  // outputs per CTA

__global__ void __launch_bounds__(256)
snake_alias_kernel(const float* __restrict__ x, float* __restrict__ y,
                   const float* __restrict__ ea, const float* __restrict__ inv_b,
                   const float* __restrict__ fu, const float* __restrict__ fd, int C, int L) {
  __shared__ float xs[SA_TL + 12];
  __shared__ float vs[2 * SA_TL + 12];
  __shared__ float f_up[12], f_dn[12];
  const int c = blockIdx.y, b = blockIdx.z;
  const int n0 = blockIdx.x * SA_TL;
  const float* row = x + ((long long)b * C + c) * L;
  float* orow = y + ((long long)b * C + c) * L;
  const int tid = threadIdx.x;
  if (tid < 12) { f_up[tid] = __ldg(fu + tid); f_dn[tid] = __ldg(fd + tid); }
  for (int i = tid; i < SA_TL + 12; i += blockDim.x) {
    int g = n0 - 6 + i;
    g = min(max(g, 0), L - 1);
    xs[i] = __ldg(row + g);
  }
  __syncthreads();
  const float a_ = __ldg(ea + c), ib = __ldg(inv_b + c);
  const int nv = 2 * SA_TL + 10;
  for (int idx = tid; idx < nv; idx += blockDim.x) {
    int m = 2 * n0 - 5 + idx;
    m = min(max(m, 0), 2 * L - 1);
    const int a = m >> 1;
    const float* xp = xs + (a - (n0 - 6));
    float acc = 0.f;
    if ((m & 1) == 0) {
#pragma unroll
      for (int d = -3; d <= 2; ++d) acc = fmaf(xp[d], f_up[5 - 2 * d], acc);
    } else {
#pragma unroll
      for (int d = -2; d <= 3; ++d) acc = fmaf(xp[d], f_up[6 - 2 * d], acc);
    }
    const float u = 2.f * acc;
    const float sn = sinf(u * a_);
    vs[idx] = u + ib * (sn * sn);
  }
  __syncthreads();
  for (int i = tid; i < SA_TL; i += blockDim.x) {
    const int n = n0 + i;
    if (n >= L) break;
    const float* vp = vs + 2 * i;
    float acc = 0.f;
#pragma unroll
    for (int k = 0; k < 12; ++k) acc = fmaf(vp[k], f_dn[k], acc);
    orow[n] = acc;
  }
}

int launch_snake_alias(const float* x, float* y, const float* ea, const float* inv_b,
                       const float* fu, const float* fd, int B, int C, int L, cudaStream_t s) {
  if (B <= 0 || C <= 0 || L <= 0) return SVCB_OK;
  if (C > 65535 || B > 65535) { set_error("snake_alias: C or B exceeds grid limits"); return SVCB_E_BAD_SHAPE; }
  dim3 grid((L + SA_TL - 1) / SA_TL, C, B);
  KernelScope ks("snake_alias", s, 70.0 * B * C * (double)L, 8.0 * B * C * (double)L);
  snake_alias_kernel<<<grid, 256, 0, s>>>(x, y, ea, inv_b, fu, fd, C, L);
  SVCB_LAUNCH_CHECK("snake_alias");
  return SVCB_OK;
}

// ------------------------------------------------------------------------------------ generator tail
// activation_post + conv_post + tanh (vits_decoder/generator.py:196-199) in one pass: wave[b, t] =
// tanh(sum_c sum_k w[c][k] * SnakeAlias_c(x[b, c, :])[t + k - PAD]) with the conv's zero padding.  The two
// separate kernels moved the 10-channel full-rate signal through HBM three times and the 10 -> 1 conv ran at
// 1/24 of its bandwidth roof (1.44 ms); here a thread computes one run of 8 Snake values per channel
// (snake8_packed), the three values its conv taps need from either neighbouring run come through a
// double-buffered shared row, and only the waveform is written.
constexpr int PF_RUNS = 256, PF_OUT_RUNS = PF_RUNS - 2, PF_MAXC = 16, PF_K = 7;

struct PostTaps { float w[PF_MAXC][PF_K]; };

__global__ void __launch_bounds__(PF_RUNS, 2)
post_fused_kernel(const float* __restrict__ x, float* __restrict__ wave, const float* __restrict__ ea,
                  const float* __restrict__ inv_b, const SnakeTapsV tp, const PostTaps pw, int C, int L,
                  const int* __restrict__ lens, int lscale) {
  __shared__ __align__(16) float srow[2][PF_RUNS * 8];
  const int tid = threadIdx.x, b = blockIdx.y;
  const int n0 = blockIdx.x * (PF_OUT_RUNS * 8) - 8 + tid * 8;   // this thread's run of Snake values
  const int Lb = lens ? __ldg(lens + b) * lscale : L;             // a ragged item's end (a multiple of 8)
  const bool inside = n0 >= 0 && n0 < Lb;                         // outside the sequence: the conv's zero padding
  const bool stores = tid >= 1 && tid <= PF_OUT_RUNS && n0 >= 0 && n0 < L;
  const bool produces = stores && inside;
  float acc[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) acc[i] = 0.f;
  for (int c = 0; c < C; ++c) {
    float v[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) v[i] = 0.f;
    if (inside) {
      const float* xr = x + ((long long)b * C + c) * L;
      float xw[24];
      if (n0 - 8 >= 0 && n0 + 16 <= Lb) {
#pragma unroll
        for (int q = 0; q < 6; ++q) {
          const float4 t4 = __ldg(reinterpret_cast<const float4*>(xr + n0 - 8) + q);
          xw[4 * q] = t4.x; xw[4 * q + 1] = t4.y; xw[4 * q + 2] = t4.z; xw[4 * q + 3] = t4.w;
        }
      } else {   // replicate padding of x (alias/resample.py:28) = clamped loads
#pragma unroll
        for (int j = 0; j < 24; ++j) xw[j] = __ldg(xr + min(max(n0 - 8 + j, 0), Lb - 1));
      }
      snake8_packed(xw, tp, __ldg(ea + c), 0.5f * __ldg(inv_b + c), v, n0 == 0, n0 + 8 == Lb);
    }
    float* sr = srow[c & 1];
    *reinterpret_cast<float4*>(sr + tid * 8) = make_float4(v[0], v[1], v[2], v[3]);
    *reinterpret_cast<float4*>(sr + tid * 8 + 4) = make_float4(v[4], v[5], v[6], v[7]);
    __syncthreads();
    if (produces) {
      const float4 lf = *reinterpret_cast<const float4*>(sr + tid * 8 - 4);   // values 4..7 of the run before
      const float4 rt = *reinterpret_cast<const float4*>(sr + tid * 8 + 8);   // values 0..3 of the run behind
      const float e[14] = {lf.y, lf.z, lf.w, v[0], v[1], v[2], v[3], v[4], v[5], v[6], v[7], rt.x, rt.y, rt.z};
#pragma unroll
      for (int k = 0; k < PF_K; ++k) {
        const float wk = pw.w[c][k];
#pragma unroll
        for (int i = 0; i < 8; ++i) acc[i] = fmaf(e[i + k], wk, acc[i]);
      }
    }
  }
  if (produces) {
    float* o = wave + (long long)b * L + n0;
    *reinterpret_cast<float4*>(o) = make_float4(tanhf(acc[0]), tanhf(acc[1]), tanhf(acc[2]), tanhf(acc[3]));
    *reinterpret_cast<float4*>(o + 4) = make_float4(tanhf(acc[4]), tanhf(acc[5]), tanhf(acc[6]), tanhf(acc[7]));
  } else if (stores) {   // past a ragged item's end
    float4* o = reinterpret_cast<float4*>(wave + (long long)b * L + n0);
    o[0] = make_float4(0.f, 0.f, 0.f, 0.f);
    o[1] = o[0];
  }
}

bool post_fused_supported(int C, int L, int K, const float* x, const float* wave) {
  return C >= 1 && C <= PF_MAXC && K == PF_K && L % 8 == 0 && ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(wave)) & 15) == 0;
}

// w_host: the conv_post taps [C][7] on the host (out channel 0)
int launch_post_fused(const float* x, float* wave, const float* ea, const float* inv_b, const SnakeTapsV& tp,
                      const float* w_host, int B, int C, int L, cudaStream_t s, const int* lens, int lscale) {
  if (B <= 0 || L <= 0) return SVCB_OK;
  if (!post_fused_supported(C, L, PF_K, x, wave)) { set_error("post_fused: unsupported shape"); return SVCB_E_BAD_SHAPE; }
  PostTaps pw;
  for (int c = 0; c < PF_MAXC; ++c)
    for (int k = 0; k < PF_K; ++k) pw.w[c][k] = c < C ? w_host[c * PF_K + k] : 0.f;
  dim3 grid((L / 8 + PF_OUT_RUNS - 1) / PF_OUT_RUNS, B);
  KernelScope ks("post_fused", s, 2.0 * PF_K * B * C * (double)L, 4.0 * B * (C + 1) * (double)L, 70.0 * B * C * (double)L);
  post_fused_kernel<<<grid, PF_RUNS, 0, s>>>(x, wave, ea, inv_b, tp, pw, C, L, lens, lscale);
  SVCB_LAUNCH_CHECK("post_fused");
  return SVCB_OK;
}

}  // namespace svcb

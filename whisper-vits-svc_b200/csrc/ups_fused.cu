// Narrow up-sampling stages in one pass: polyphase ConvTranspose1d + noise convolution + both biases.
//
// Replaces, for the last generator stages (Cin <= 40), the line
//   x = self.ups[i](x) + self.noise_convs[i](har_source)              vits_decoder/generator.py:183-186
// which the general path runs as `rate` sub-convolutions into per-phase slabs followed by
// ups_finalize (interleave + bias + noise conv).  With 20 -> 10 or 40 -> 20 channels those
// sub-convolutions have nothing for a 128 x N tensor-core tile to chew on and were gather-bound
// (0.44 TB/s, profiles/r01_notes.md §8); here one thread owns one input position q and produces
// all `RATE` output phases x all COUT channels from x[:, q-M+1 .. q], exact fp32:
//   y[co][n] = b[co] + sum_ci sum_j w_r[ci][j][co] x[ci][q + j - (M-1)]  + bn[co] + sum_j wn[j][co] src[n*sf + j - padn]
//   with n = q*RATE - pad + r,   w_r = phase-r sub-filter (pack.py: w_r[co][ci][j] = w[ci][co][r + RATE*(M-1-j)])
// x is read once and y written once: 4*(Cin/RATE + COUT) bytes per output sample.
#include <cstdio>

#include "common.cuh"

namespace svcb {

template <int COUT, int RATE, int M>
__global__ void __launch_bounds__(256)
ups_fused_kernel(const UpsFusedParams p) {
  constexpr int CP = (COUT + 3) / 4 * 4;
  extern __shared__ __align__(16) float uf_smem[];
  float* wsm = uf_smem;                       // [RATE][Cin][M][CP]
  float* wns = wsm + RATE * p.Cin * M * CP;   // [Kn][CP]
  float* bsm = wns + p.Kn * CP;               // [CP]: conv bias + noise bias
  const int tid = threadIdx.x, b = blockIdx.y;
  for (int i = tid; i < RATE * p.Cin * M * CP; i += 256) {
    const int co = i % CP, cj = (i / CP) % (p.Cin * M), r = i / (CP * p.Cin * M);
    wsm[i] = co < COUT ? __ldg((r == 0 ? p.wph[0] : p.wph[1]) + (long long)cj * p.cout_pad + co) : 0.f;
  }
  for (int i = tid; i < p.Kn * CP; i += 256) {
    const int co = i % CP, j = i / CP;
    wns[i] = co < COUT ? __ldg(p.wn + (long long)j * p.cout_pad_n + co) : 0.f;
  }
  if (tid < CP) bsm[tid] = tid < COUT ? __ldg(p.bias + tid) + __ldg(p.bn + tid) : 0.f;
  __syncthreads();

  const int q = blockIdx.x * 256 + tid;
  if (q > (p.Ln - 1 + p.pad) / RATE) return;
  float acc[RATE][CP];
#pragma unroll
  for (int r = 0; r < RATE; ++r)
#pragma unroll
    for (int co = 0; co < CP; ++co) acc[r][co] = bsm[co];

  const float* xb = p.x + (long long)b * p.Cin * p.L;
  bool ok[M];
#pragma unroll
  for (int j = 0; j < M; ++j) ok[j] = (q + j - (M - 1)) >= 0 && (q + j - (M - 1)) < p.L;
#pragma unroll 4
  for (int ci = 0; ci < p.Cin; ++ci) {
    float xv[M];
#pragma unroll
    for (int j = 0; j < M; ++j) xv[j] = ok[j] ? __ldg(xb + (long long)ci * p.L + q + j - (M - 1)) : 0.f;
#pragma unroll
    for (int r = 0; r < RATE; ++r)
#pragma unroll
      for (int j = 0; j < M; ++j) {
        const float4* w4 = reinterpret_cast<const float4*>(wsm + ((r * p.Cin + ci) * M + j) * CP);
#pragma unroll
        for (int g = 0; g < CP / 4; ++g) {
          const float4 w = w4[g];
          acc[r][4 * g + 0] = fmaf(xv[j], w.x, acc[r][4 * g + 0]);
          acc[r][4 * g + 1] = fmaf(xv[j], w.y, acc[r][4 * g + 1]);
          acc[r][4 * g + 2] = fmaf(xv[j], w.z, acc[r][4 * g + 2]);
          acc[r][4 * g + 3] = fmaf(xv[j], w.w, acc[r][4 * g + 3]);
        }
      }
  }
  const float* sb = p.src + (long long)b * p.Ltot;
  const long long nsrc = p.lens ? (long long)__ldg(p.lens + b) * p.src_scale : p.Ltot;   // a ragged item's source end
  float* yb = p.y + (long long)b * COUT * p.Ln;
#pragma unroll
  for (int r = 0; r < RATE; ++r) {
    const int n = q * RATE - p.pad + r;
    if (n >= 0 && n < p.Ln) {
      for (int j = 0; j < p.Kn; ++j) {
        const long long si = (long long)n * p.sf + j - p.padn;
        const float sv = (si >= 0 && si < nsrc) ? __ldg(sb + si) : 0.f;
#pragma unroll
        for (int co = 0; co < COUT; ++co) acc[r][co] = fmaf(sv, wns[j * CP + co], acc[r][co]);
      }
#pragma unroll
      for (int co = 0; co < COUT; ++co) yb[(long long)co * p.Ln + n] = acc[r][co];
    }
  }
}

bool ups_fused_supported(int Cin, int Cout, int rate, int taps, int Kn) {
  return rate == 2 && taps == 2 && Kn >= 1 && Kn <= 8 && Cin <= 40 && (Cout == 10 || Cout == 20);
}

template <int COUT>
static int launch_uf(const UpsFusedParams& p, cudaStream_t s) {
  constexpr int CP = (COUT + 3) / 4 * 4;
  const size_t smem = ((size_t)2 * p.Cin * 2 * CP + (size_t)p.Kn * CP + CP) * sizeof(float);
  const int nq = (p.Ln - 1 + p.pad) / 2 + 1;
  dim3 grid((nq + 255) / 256, p.B);
  char kname[64];
  snprintf(kname, sizeof(kname), "ups_fused_%dto%d", p.Cin, COUT);
  KernelScope ks(kname, s, 2.0 * p.B * (double)p.Ln * COUT * (p.Cin * 2 + p.Kn),
                 4.0 * p.B * ((double)p.Cin * p.L + (double)COUT * p.Ln + (double)p.Ln * p.sf));
  ups_fused_kernel<COUT, 2, 2><<<grid, 256, smem, s>>>(p);
  SVCB_LAUNCH_CHECK("ups_fused");
  return SVCB_OK;
}

int launch_ups_fused(const UpsFusedParams& p, cudaStream_t s) {
  if (p.B <= 0 || p.Ln <= 0) return SVCB_OK;
  if (!ups_fused_supported(p.Cin, p.Cout, p.rate, p.M, p.Kn)) {
    set_error("ups_fused: unsupported stage shape");
    return SVCB_E_UNSUPPORTED;
  }
  return p.Cout == 10 ? launch_uf<10>(p, s) : launch_uf<20>(p, s);
}

}  // namespace svcb

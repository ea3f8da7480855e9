// Generic fp32 Conv1d on the CUDA cores (register-tiled direct convolution).
//
// Replaces every torch.nn.functional.conv1d / conv_transpose1d call site of the reference's
// inference path that is not served by the tensor-core kernels: enc_p.pre/hub, the 1x1
// attention/FFN/flow convs (vits/models.py:44-49, vits/attentions.py:215-223,390-398,
// vits/modules.py:184-198,296-299), conv_pre / noise_convs / conv_post and, as per-phase
// sub-convolutions, the ConvTranspose1d upsamplers (vits_decoder/generator.py:177-199).
//
// Tiling: one CTA = 32 time lanes x COG channel groups; a thread owns 8 output channels x TPT
// time steps (t = lane + 32*i, so shared-memory reads of x are conflict-free and global stores
// are coalesced along T).  Input channels are streamed through shared memory CI_T at a time:
// x tile [CI_T][span] and weight tile [CI_T][K][8*COG] (co innermost -> two LDS.128 per tap).
#include <algorithm>
#include <climits>
#include <cstdio>

#include "common.cuh"

namespace svcb {

__device__ __forceinline__ float act_apply(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_MISH: {
      // x * tanh(softplus(x)); torch softplus switches to identity above threshold 20
      float sp = v > 20.f ? v : log1pf(expf(v));
      return v * tanhf(sp);
    }
    case ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    case ACT_TANH: return tanhf(v);
    default: return v;
  }
}

template <int TPT>
__global__ void __launch_bounds__(256)
conv1d_kernel(const ConvParams p, const int ci_tile, const int xspan) {
  extern __shared__ __align__(16) float smem[];
  const int COT = blockDim.y * 8;
  float* xs = smem;
  float* ws = smem + ci_tile * xspan;  // xspan is a multiple of 4 -> 16 B aligned
  const int lane = threadIdx.x, cg = threadIdx.y;
  const int tid = cg * 32 + lane, nthreads = blockDim.y * 32;
  const int b = blockIdx.z;
  const int co0 = blockIdx.y * COT;
  const int tq0 = blockIdx.x * 32 * TPT;
  const int x_start = (p.q0 + tq0) * p.stride - p.pad;
  const long long len = p.lengths ? p.lengths[b] : LLONG_MAX;
  const float* xb = p.x + (long long)b * p.sxb;
  const int K = p.K;

  float acc[TPT][8];
#pragma unroll
  for (int i = 0; i < TPT; ++i)
#pragma unroll
    for (int h = 0; h < 8; ++h) acc[i][h] = 0.f;

  for (int ci0 = 0; ci0 < p.Cin; ci0 += ci_tile) {
    __syncthreads();
    // ---- x tile
    const int nx = ci_tile * xspan;
    if (p.sxc == 1) {  // channel-contiguous (time-major) input: let ci run fastest
      for (int idx = tid; idx < nx; idx += nthreads) {
        const int c = idx % ci_tile, s = idx / ci_tile;
        const int ci = ci0 + c, ti = x_start + s;
        float v = 0.f;
        if (ci < p.Cin && ti >= 0 && ti < p.Tin && (!(p.flags & CONV_IN_MASK) || ti < len))
          v = __ldg(xb + (long long)ci + (long long)ti * p.sxt);
        xs[c * xspan + s] = v;
      }
    } else {
      for (int idx = tid; idx < nx; idx += nthreads) {
        const int c = idx / xspan, s = idx - c * xspan;
        const int ci = ci0 + c, ti = x_start + s;
        float v = 0.f;
        if (ci < p.Cin && ti >= 0 && ti < p.Tin && (!(p.flags & CONV_IN_MASK) || ti < len))
          v = __ldg(xb + (long long)ci * p.sxc + (long long)ti * p.sxt);
        xs[c * xspan + s] = v;
      }
    }
    // ---- weight tile: rows (ci,j) are contiguous in the packed layout
    const int nw = ci_tile * K * COT;
    for (int idx = tid; idx < nw; idx += nthreads) {
      const int col = idx % COT, cj = idx / COT;
      const int ci = ci0 + cj / K, co = co0 + col;
      float v = 0.f;
      if (ci < p.Cin && co < p.cout_pad)
        v = __ldg(p.w + ((long long)ci0 * K + cj) * p.cout_pad + co);
      ws[idx] = v;
    }
    __syncthreads();
    const int cmax = min(ci_tile, p.Cin - ci0);
    for (int c = 0; c < cmax; ++c) {
      const float* xr = xs + c * xspan + lane * p.stride;
      const float* wr = ws + c * K * COT + cg * 8;
      for (int j = 0; j < K; ++j) {
        const float4 wa = *reinterpret_cast<const float4*>(wr + j * COT);
        const float4 wb = *reinterpret_cast<const float4*>(wr + j * COT + 4);
        const float* xj = xr + j * p.dil;
#pragma unroll
        for (int i = 0; i < TPT; ++i) {
          const float xv = xj[i * 32 * p.stride];
          acc[i][0] = fmaf(xv, wa.x, acc[i][0]);
          acc[i][1] = fmaf(xv, wa.y, acc[i][1]);
          acc[i][2] = fmaf(xv, wa.z, acc[i][2]);
          acc[i][3] = fmaf(xv, wa.w, acc[i][3]);
          acc[i][4] = fmaf(xv, wb.x, acc[i][4]);
          acc[i][5] = fmaf(xv, wb.y, acc[i][5]);
          acc[i][6] = fmaf(xv, wb.z, acc[i][6]);
          acc[i][7] = fmaf(xv, wb.w, acc[i][7]);
        }
      }
    }
  }

  // ---- epilogue
  const int cbase = co0 + cg * 8;
  float* yb = p.y + (long long)b * p.syb;
  const float* rb = p.res ? p.res + (long long)b * p.syb : nullptr;
#pragma unroll
  for (int i = 0; i < TPT; ++i) {
    const int tq = tq0 + lane + 32 * i;
    if (tq >= p.nq) continue;
    const bool keep = !(p.flags & CONV_OUT_MASK) || tq < len;
    auto finish = [&](float v, int co) {
      if (!keep) v = 0.f;
      const long long off = (long long)co * p.syc + (long long)tq * p.syt;
      if (rb) v += rb[off];
      if (p.flags & CONV_ACCUM) v += yb[off];
      if (p.out_div != 0.f) { asm volatile(""); v = v / p.out_div; }
      yb[off] = v;
    };
    if (p.flags & CONV_GATE) {
#pragma unroll
      for (int h = 0; h < 4; ++h) {
        const int cp = cbase + 2 * h;
        if (cp + 1 < p.Cout) {
          float a = acc[i][2 * h], g = acc[i][2 * h + 1];
          if (p.bias) { a += __ldg(p.bias + cp); g += __ldg(p.bias + cp + 1); }
          const float v = tanhf(a) * (1.f / (1.f + expf(-g)));
          finish(v, cp >> 1);
        }
      }
    } else {
#pragma unroll
      for (int h = 0; h < 8; ++h) {
        const int co = cbase + h;
        if (co < p.Cout) {
          float v = acc[i][h];
          if (p.bias) v += __ldg(p.bias + co);
          v = act_apply(v, p.act);
          finish(v, co);
        }
      }
    }
  }
}

static int pick_cog(int cout_pad) {
  const int ng = cout_pad / 8;
  int best = 1, best_cost = INT_MAX;
  for (int c = 1; c <= 8; ++c) {
    const int cost = ((ng + c - 1) / c) * c;
    if (cost <= best_cost) { best_cost = cost; best = c; }
  }
  return best;
}

template <int TPT>
static int launch_t(const ConvParams& p, int cog, int ci_tile, int xspan, size_t smem,
                    cudaStream_t s) {
  static DevSmemCache attr_cache;
  SVCB_CUDA_CHECK(ensure_dyn_smem(conv1d_kernel<TPT>, 200 * 1024, attr_cache));
  dim3 block(32, cog);
  dim3 grid((p.nq + 32 * TPT - 1) / (32 * TPT), (p.cout_pad / 8 + cog - 1) / cog, p.B);
  const int cout_real = (p.flags & CONV_GATE) ? p.Cout / 2 : p.Cout;
  char kname[64];
  snprintf(kname, sizeof(kname), "conv1d_fp32_%dto%d_k%d_o1", p.Cin, p.Cout, p.K);
  KernelScope ks(kname, s, 2.0 * p.Cin * p.K * p.Cout * (double)p.nq * p.B,
                 4.0 * ((double)p.B * p.Cin * p.nq * p.stride + (double)p.B * cout_real * p.nq * (p.res ? 2 : 1) +
                        (double)p.Cin * p.K * p.Cout));
  conv1d_kernel<TPT><<<grid, block, smem, s>>>(p, ci_tile, xspan);
  SVCB_LAUNCH_CHECK("conv1d");
  return SVCB_OK;
}

int launch_conv1d(const ConvParams& p, cudaStream_t s) {
  if (p.nq <= 0 || p.B <= 0) return SVCB_OK;
  if (p.cout_pad % 8 != 0 || p.cout_pad < p.Cout) {
    set_error("conv1d: cout_pad must be a multiple of 8 and >= Cout");
    return SVCB_E_BAD_SHAPE;
  }
  const int cog = pick_cog(p.cout_pad);
  const int ci_tile = std::min(8, p.Cin);
  auto span = [&](int tpt) { return (((32 * tpt - 1) * p.stride + (p.K - 1) * p.dil + 1) + 3) & ~3; };
  auto bytes = [&](int tpt) {
    return (size_t)(ci_tile * span(tpt) + ci_tile * p.K * cog * 8) * sizeof(float);
  };
  if (p.nq > 64 && bytes(8) <= 96 * 1024) return launch_t<8>(p, cog, ci_tile, span(8), bytes(8), s);
  if (bytes(2) <= 200 * 1024) return launch_t<2>(p, cog, ci_tile, span(2), bytes(2), s);
  set_error("conv1d: tile does not fit shared memory");
  return SVCB_E_UNSUPPORTED;
}

}  // namespace svcb

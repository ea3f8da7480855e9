// General Conv1d as an implicit GEMM on wgmma (bf16 or bf16x3 operands, fp32 accumulate).
//
// Serves every dense convolution of the prior encoder, the flow and the generator head
// (vits/models.py:44-49, vits/attentions.py:215-223,390-398, vits/modules.py:184-198,296-299,
// vits_decoder/generator.py:177-178) — the F.conv1d call sites whose contraction is wide enough for
// the tensor cores (SURVEY.md §8a rows a2-a7).
//
//   D[t, co] = sum_cc sum_tap  A_cc[t + tap*dil, :] . W[tap, cc][co, :]      M = 128, N = BN, K = 32
// * Input channels are processed in chunks of 32 (kConvTcKch).  Two warpgroups gather one chunk of x
//   (fp32, any strides — the time-major PPG input included), apply the optional input mask and the
//   conv's zero padding, split to bf16 hi/lo and write the K-major panel layout of tc.cuh into a
//   2-deep A ring; the gather of chunk cc+1 overlaps the MMAs of chunk cc still in flight.
// * For every (chunk, tap) the pre-packed weight tiles (hi, lo) arrive by 1-D bulk copy into a
//   3-deep W ring (producer thread).  Each warpgroup issues wgmma m64nBNk16 for its 64 rows: taps
//   reuse the same A chunk through a row-shifted descriptor.
// * Epilogue (the same warpgroups, through a shared-memory strip): bias -> {none, ReLU, Mish, tanh,
//   WaveNet gate on interleaved channel pairs} -> output mask -> residual -> accumulate -> store [B,C,T].
#include <cstdio>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

constexpr int CT_M = 128;
constexpr int CT_WST = 3;  // W ring depth (max)
constexpr int CT_EPI_LD = 72;   // floats per row of an epilogue strip
constexpr int CT_THREADS = 288;
constexpr size_t CT_STRIP_BYTES = 2 * 64 * CT_EPI_LD * 4;

__device__ __forceinline__ float ct_act(float v, int act) {
  switch (act) {
    case ACT_RELU: return fmaxf(v, 0.f);
    case ACT_MISH: { const float sp = v > 20.f ? v : log1pf(expf(v)); return v * tanhf(sp); }
    case ACT_GELU: return 0.5f * v * (1.f + erff(v * 0.70710678118654752440f));
    case ACT_TANH: return tanhf(v);
    default: return v;
  }
}

template <int BN>
__global__ void __launch_bounds__(CT_THREADS, 1)
conv_tc_kernel(const ConvTcParams p, const int wst) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t w_full[CT_WST], w_empty[CT_WST];
  const int tid = threadIdx.x, warp = tid >> 5;
  const int b = blockIdx.z, nt = blockIdx.y;
  const int t0 = blockIdx.x * CT_M;
  const int P = p.pad;
  const int R = CT_M + (p.K - 1) * p.dil;
  constexpr int KC = kConvTcKch / 8;
  const int n0row = t0 - P;                       // sequence position of A row 0
  const uint32_t a_part = (uint32_t)KC * R * 16u; // one of hi / lo
  const int nparts = p.nsplit == 3 ? 2 : 1;
  const uint32_t a_buf = a_part * nparts;
  constexpr uint32_t w_tile = (uint32_t)kConvTcKch * BN * 2u;
  uint8_t* A0 = smem;
  uint8_t* W0 = smem + 2 * a_buf;
  float* Strips = reinterpret_cast<float*>(W0 + (size_t)wst * w_tile);
  const int ncc = p.cin_pad / kConvTcKch;
  const long long len = p.lengths ? p.lengths[b] : (long long)1 << 60;

  if (tid == 0) {
    for (int i = 0; i < wst; ++i) { tc::mbar_init(&w_full[i], 1); tc::mbar_init(&w_empty[i], 2); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (tid == 256) {
    // ---------------------------------------------------------------- W producer
    const int total = ncc * p.K * nparts;
    for (int i = 0; i < total; ++i) {
      const int st = i % wst;
      if (i >= wst) tc::mbar_wait(&w_empty[st], (uint32_t)(((i / wst) - 1) & 1));
      const int part = i % nparts, tap = (i / nparts) % p.K, cc = i / (nparts * p.K);
      const size_t tile = (((size_t)tap * ncc + cc) * 2 + part) * p.ntiles + nt;
      tc::mbar_arrive_expect_tx(&w_full[st], w_tile);
      tc::bulk_g2s(W0 + (size_t)st * w_tile, p.wpk + tile * w_tile, w_tile, &w_full[st]);
    }
  }
  if (warp == 8) return;
  // -------------------------------------------------------------------- gather + MMA + epilogue (warps 0-7)
  // A thread fetches TWO items (16 scalar or 4 vector loads in flight) before it converts either.
  const int pid = tid;   // 0 .. 255
  const int wg = warp >> 2, t = tid & 127;
    const float* xb = p.x + (long long)b * p.sxb;
    const float* x2b = p.x2 ? p.x2 + (long long)b * p.sx2b : nullptr;
    const int n_items = R * KC;
    auto fetch = [&](int item, int cc, float (&v)[8]) {
      const int r = item % R, kc = item / R;
      const int tau = n0row + r;
      const int c0 = cc * kConvTcKch + kc * 8;
      const bool row_ok = tau >= 0 && tau < p.Tin && (!(p.flags & CONV_IN_MASK) || tau < len);
      if (row_ok && x2b && c0 >= p.cin1) {   // second input: channel-contiguous windows (unaligned)
        const float* s2 = x2b + (long long)tau * p.sx2t + (c0 - p.cin1);
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = (c0 - p.cin1 + e < p.cin2) ? __ldg(s2 + e) : 0.f;
      } else if (row_ok) {
        if (p.sxc == 1 && c0 + 8 <= p.Cin) {  // channel-contiguous input: two 16-byte loads
          const float4* s4 = reinterpret_cast<const float4*>(xb + (long long)tau * p.sxt + c0);
          const float4 u0 = __ldg(s4), u1 = __ldg(s4 + 1);
          v[0] = u0.x; v[1] = u0.y; v[2] = u0.z; v[3] = u0.w; v[4] = u1.x; v[5] = u1.y; v[6] = u1.z; v[7] = u1.w;
        } else {
#pragma unroll
          for (int e = 0; e < 8; ++e)
            v[e] = (c0 + e < p.Cin) ? __ldg(xb + (long long)(c0 + e) * p.sxc + (long long)tau * p.sxt) : 0.f;
        }
      } else {
#pragma unroll
        for (int e = 0; e < 8; ++e) v[e] = 0.f;
      }
    };
    auto put = [&](int item, uint8_t* Ah, uint8_t* Al, const float (&v)[8]) {
      const int r = item % R, kc = item / R;
      __align__(16) __nv_bfloat16 hi[8], lo[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        hi[e] = __float2bfloat16_rn(v[e]);
        lo[e] = __float2bfloat16_rn(v[e] - __bfloat162float(hi[e]));
      }
      *reinterpret_cast<uint4*>(Ah + ((size_t)kc * R + r) * 16) = *reinterpret_cast<const uint4*>(hi);
      if (nparts == 2)
        *reinterpret_cast<uint4*>(Al + ((size_t)kc * R + r) * 16) = *reinterpret_cast<const uint4*>(lo);
    };
  auto gather = [&](int cc) {
    uint8_t* Ah = A0 + (size_t)(cc & 1) * a_buf;
    uint8_t* Al = Ah + a_part;
    for (int it0 = pid; it0 < n_items; it0 += 512) {
      const int it1 = it0 + 256;
      float va[8], vb[8];
      fetch(it0, cc, va);
      if (it1 < n_items) fetch(it1, cc, vb);
      put(it0, Ah, Al, va);
      if (it1 < n_items) put(it1, Ah, Al, vb);
    }
    tc::fence_proxy_async_smem();
  };
  const uint32_t a_base = tc::smem_u32(A0) + (uint32_t)wg * 64u * 16u, w_base = tc::smem_u32(W0);
  const uint32_t lbo_a = (uint32_t)R * 16u, lbo_b = (uint32_t)BN * 16u;
  const uint64_t ks_a = (2u * lbo_a) >> 4, ks_b = (2u * lbo_b) >> 4;
  constexpr int nk = kConvTcKch / 16;
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  gather(0);
  int wi = 0;
  for (int cc = 0; cc < ncc; ++cc) {
    tc::named_sync(1, 256);                    // chunk cc gathered by both warpgroups; no MMA reads the other buffer
    const uint32_t ah = a_base + (uint32_t)(cc & 1) * a_buf, al = ah + a_part;
    for (int tap = 0; tap < p.K; ++tap) {
      const uint32_t row_off = (uint32_t)(tap * p.dil) * 16u;
      for (int part = 0; part < nparts; ++part, ++wi) {
        const int st = wi % wst;
        tc::mbar_wait(&w_full[st], (uint32_t)((wi / wst) & 1));
        const uint64_t bd = tc::smem_desc(w_base + (uint32_t)st * w_tile, lbo_b);
        const int n_a = (part == 0 && nparts == 2) ? 2 : 1;
        tc::wg_fence();
        for (int ap = 0; ap < n_a; ++ap) {
          const uint64_t ad = tc::smem_desc((ap == 0 ? ah : al) + row_off, lbo_a);
          for (int kk = 0; kk < nk; ++kk) tc::Wg<BN, 0>::ss(acc, ad + kk * ks_a, bd + kk * ks_b, 1u);
        }
        tc::wg_commit();
        tc::wg_wait<1>();                      // the previous weight slot's MMAs are done: release it
        if (wi > 0 && t == 0) tc::mbar_arrive(&w_empty[(wi - 1) % wst]);
      }
    }
    if (cc + 1 < ncc) gather(cc + 1);          // overlaps the last MMAs of this chunk
    tc::wg_wait<0>();
  }
  tc::wg_hold(acc);
  if (t == 0) tc::mbar_arrive(&w_empty[(wi - 1) % wst]);

  // ---------------------------------------------------------------- epilogue: thread = (row t % 64, 32-column half)
  float* strip = Strips + wg * 64 * CT_EPI_LD;
  const int tq = t0 + wg * 64 + (t & 63);
  const bool gate = (p.flags & CONV_GATE) != 0;
  const int cout_real = gate ? p.Cout / 2 : p.Cout;
  const bool keep = !(p.flags & CONV_OUT_MASK) || tq < len;
  float* yb = p.y + (long long)b * cout_real * p.Tout;
  const float* rb = p.res ? p.res + (long long)b * cout_real * p.Tout : nullptr;
#pragma unroll 1
  for (int ch = 0; ch < (BN + 63) / 64; ++ch) {
    tc::named_sync(2 + wg, 128);
    tc::acc_to_smem<BN>(acc, strip, CT_EPI_LD, 8 * ch, 8 * ch + 8);
    tc::named_sync(2 + wg, 128);
#pragma unroll 1
    for (int sub = 0; sub < 2; ++sub) {
      const int cl = (t >> 6) * 32 + sub * 16, c0 = ch * 64 + cl;
      if (c0 >= BN) continue;
      float vf[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) vf[j] = strip[(t & 63) * CT_EPI_LD + cl + j];
      const int t = tq;
    if (p.ilv) {   // interleaved store: ilv consecutive samples of one channel per thread (one 8 / 16-byte store)
      float* yi = p.y + (long long)b * p.Cout * p.Tout;   // = [Cout / ilv][Tout * ilv]
      {
        if (t < p.Tout) {
#pragma unroll
          for (int j = 0; j < 16; j += 4) {
            const int cp = nt * BN + c0 + j;
            if (cp < p.Cout) {
              float o[4];
#pragma unroll
              for (int e = 0; e < 4; ++e) o[e] = ct_act(vf[j + e] + (p.bias ? __ldg(p.bias + cp + e) : 0.f), p.act);
              if (p.ilv == 4) {
                *reinterpret_cast<float4*>(yi + ((long long)(cp >> 2) * p.Tout + t) * 4) = make_float4(o[0], o[1], o[2], o[3]);
              } else {
                *reinterpret_cast<float2*>(yi + ((long long)(cp >> 1) * p.Tout + t) * 2) = make_float2(o[0], o[1]);
                *reinterpret_cast<float2*>(yi + ((long long)((cp >> 1) + 1) * p.Tout + t) * 2) = make_float2(o[2], o[3]);
              }
            }
          }
        }
      }
    } else
    {
      const bool live = t < p.Tout;
      const int step = gate ? 2 : 1;
      // residual / accumulator loads of the strip first (all in flight), stores afterwards
      float add[16];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float a = 0.f;
        const int cp = nt * BN + c0 + j;
        if (live && (j % step) == 0 && cp + (step - 1) < p.Cout) {
          const long long off = (long long)(gate ? (cp >> 1) : cp) * p.Tout + t;
          if (rb) a = rb[off];
          if (p.flags & CONV_ACCUM) a += yb[off];
        }
        add[j] = a;
      }
      if (live) {
        if (gate) {
#pragma unroll
          for (int j = 0; j < 16; j += 2) {
            const int cp = nt * BN + c0 + j;
            if (cp + 1 < p.Cout) {
              const float a = vf[j] + __ldg(p.bias + cp);
              const float g = vf[j + 1] + __ldg(p.bias + cp + 1);
              float o = tanhf(a) * (1.f / (1.f + expf(-g)));
              if (!keep) o = 0.f;
              yb[(long long)(cp >> 1) * p.Tout + t] = o + add[j];
            }
          }
        } else {
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int co = nt * BN + c0 + j;
            if (co < p.Cout) {
              float o = ct_act(vf[j] + (p.bias ? __ldg(p.bias + co) : 0.f), p.act);
              if (!keep) o = 0.f;
              yb[(long long)co * p.Tout + t] = o + add[j];
            }
          }
        }
      }
    }
    }
  }
}

static size_t conv_tc_smem_bytes(const ConvTcParams& p, int wst) {
  const int R = CT_M + (p.K - 1) * p.dil;
  const size_t a_buf = (size_t)(kConvTcKch / 8) * R * 16 * (p.nsplit == 3 ? 2 : 1);
  return 2 * a_buf + (size_t)wst * kConvTcKch * p.bn * 2 + CT_STRIP_BYTES + 128;
}

int launch_conv_tc(const ConvTcParams& p, cudaStream_t s) {
  if (p.B <= 0 || p.Tout <= 0) return SVCB_OK;
  if (p.cin_pad % kConvTcKch || p.bn % 16 || p.bn < 16 || p.bn > 256 ||
      p.ntiles * p.bn < p.Cout || (p.nsplit != 1 && p.nsplit != 3) || p.Tout > p.Tin) {
    set_error("conv_tc: unsupported tiling (stride-1 'same' convolutions only)");
    return SVCB_E_BAD_SHAPE;
  }
  if (p.x2 && (p.cin1 % 8 || p.cin1 < p.Cin || p.cin1 + p.cin2 > p.cin_pad)) {
    set_error("conv_tc: second input must start at a multiple of 8 channels behind the first");
    return SVCB_E_BAD_SHAPE;
  }
  if (p.ilv && ((p.ilv != 2 && p.ilv != 4) || p.Cout % 4 || p.res || (p.flags & (CONV_ACCUM | CONV_GATE | CONV_OUT_MASK)) ||
                (reinterpret_cast<uintptr_t>(p.y) & 15))) {
    set_error("conv_tc: interleaved output needs ilv in {2, 4}, Cout % 4 == 0, a 16-byte aligned y and a plain epilogue");
    return SVCB_E_BAD_SHAPE;
  }
  // a 2-deep weight ring when that lets two CTAs share an SM (one CTA's epilogue then overlaps the
  // other's gather + MMA; the 1x1 convolutions are epilogue-bound), else the 3-deep ring
  int wst = CT_WST;
  if (conv_tc_smem_bytes(p, 2) <= 113 * 1024) wst = 2;
  const size_t smem = conv_tc_smem_bytes(p, wst);
  if (smem > 227 * 1024 - 512) { set_error("conv_tc: tile does not fit shared memory"); return SVCB_E_UNSUPPORTED; }
  dim3 grid((p.Tout + CT_M - 1) / CT_M, p.ntiles, p.B);
  const int cout_real = (p.flags & CONV_GATE) ? p.Cout / 2 : p.Cout;
  char kname[64];
  snprintf(kname, sizeof(kname), "conv_tc_%s_%dto%d_k%d_o1", p.nsplit == 3 ? "bf16x3" : "bf16", p.Cin, p.Cout, p.K);
  KernelScope ks(kname, s,
                 2.0 * p.Cin * p.K * p.Cout * (double)p.Tout * p.B,
                 4.0 * ((double)p.B * p.Cin * p.Tin + (double)p.B * cout_real * p.Tout * (p.res ? 2 : 1)) +
                     2.0 * (double)p.Cin * p.K * p.Cout);
  switch (p.bn / 16) {
#define SVCB_CONV_BN(nb)                                                           \
  case nb: {                                                                       \
    static DevSmemCache attr_cache;                                                \
    SVCB_CUDA_CHECK(ensure_dyn_smem(conv_tc_kernel<16 * nb>, smem, attr_cache));   \
    conv_tc_kernel<16 * nb><<<grid, CT_THREADS, smem, s>>>(p, wst);                \
    break;                                                                         \
  }
    SVCB_CONV_BN(1) SVCB_CONV_BN(2) SVCB_CONV_BN(3) SVCB_CONV_BN(4) SVCB_CONV_BN(5) SVCB_CONV_BN(6) SVCB_CONV_BN(7) SVCB_CONV_BN(8)
    SVCB_CONV_BN(9) SVCB_CONV_BN(10) SVCB_CONV_BN(11) SVCB_CONV_BN(12) SVCB_CONV_BN(13) SVCB_CONV_BN(14) SVCB_CONV_BN(15) SVCB_CONV_BN(16)
#undef SVCB_CONV_BN
  }
  SVCB_LAUNCH_CHECK("conv_tc");
  return SVCB_OK;
}

}  // namespace svcb

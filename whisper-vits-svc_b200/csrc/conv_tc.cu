// General Conv1d as an implicit GEMM on wgmma (bf16 or bf16x3 operands, fp32 accumulate).
//
// Serves every dense convolution of the prior encoder, the flow and the generator head
// (vits/models.py:44-49, vits/attentions.py:215-223,390-398, vits/modules.py:184-198,296-299,
// vits_decoder/generator.py:177-178) — the F.conv1d call sites whose contraction is wide enough for
// the tensor cores (SURVEY.md §8a rows a2-a7).
//
//   D[t, co] = sum_cc sum_tap  A_cc[t + tap*dil, :] . W[tap, cc][co, :]      M = 128 * MB, N = BN, K = 32
// A persistent, warp-specialised kernel: one CTA per SM walks the (item, t-tile, n-tile) tiles, n fastest so
// the N tiles of one t-tile run side by side and their repeated reads of x hit L2.
// * Producer warpgroup (warps 0-3, registers given away with setmaxnreg):
//   - warps 0-2 gather one 32-channel chunk of x at a time (fp32, any strides — the time-major PPG input
//     included), apply the optional input mask and the conv's zero padding, split to bf16 hi/lo and write
//     the K-major panel layout of tc.cuh into an A ring of up to 4 stages (mbarrier full / empty pairs);
//   - one thread of warp 3 streams the pre-packed weight tiles (hi, lo) of every (chunk, tap) by 1-D bulk
//     copy into a W ring of 4-8 slots.
//   Both run ahead of the MMAs across chunk and tile boundaries, so tile i+1's loads overlap tile i's epilogue.
// * Two consumer warpgroups only issue wgmma and run the epilogue.  Each owns 64 * MB rows of the tile: with
//   MB = 2 (BN <= 192) every weight tile fetched feeds 256 output rows.  Taps reuse the same A chunk through
//   a row-shifted descriptor; one wgmma group stays in flight across slot, tap and chunk boundaries.
//   The accumulation order per output (chunk, tap, hi/lo part) does not depend on the tiling.
// * Epilogue (through a shared-memory strip per warpgroup): bias -> {none, ReLU, Mish, tanh, WaveNet gate on
//   interleaved channel pairs} -> output mask -> residual -> accumulate -> store [B,C,T] (or the interleaved
//   store of the combined upsampler).
#include <cstdio>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

constexpr int CT_AST = 4;       // A ring depth (max)
constexpr int CT_WST = 8;       // W ring depth (max)
constexpr int CT_WST_MIN = 4;
constexpr int CT_EPI_LD = 72;   // floats per row of an epilogue strip
constexpr int CT_THREADS = 384;
constexpr int CT_GATHER = 96;   // producer threads that gather A (warps 0-2)
constexpr int CT_PRODUCER_REGS = 56, CT_CONSUMER_REGS = 224;   // 128 * 56 + 256 * 224 <= 64 K registers
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

struct CtTile { int b, t0, nt; };
template <int M>
__device__ __forceinline__ CtTile ct_tile(const ConvTcParams& p, int tile) {
  const int n_t = (p.Tout + M - 1) / M;
  const int rest = tile / p.ntiles;
  return {rest / n_t, (rest % n_t) * M, tile % p.ntiles};
}

template <int BN, int MB>
__global__ void __launch_bounds__(CT_THREADS, 1)
conv_tc_kernel(const ConvTcParams p, const int ast, const int wst) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t a_full[CT_AST], a_empty[CT_AST], w_full[CT_WST], w_empty[CT_WST];
  constexpr int M = 128 * MB;
  constexpr int KC = kConvTcKch / 8;
  constexpr uint32_t w_tile = (uint32_t)kConvTcKch * BN * 2u;
  const int tid = threadIdx.x, warp = tid >> 5;
  const int R = M + (p.K - 1) * p.dil;
  const uint32_t a_part = (uint32_t)KC * R * 16u; // one of hi / lo
  const int nparts = p.nsplit == 3 ? 2 : 1;
  const uint32_t a_buf = a_part * nparts;
  uint8_t* A0 = smem;
  uint8_t* W0 = smem + (size_t)ast * a_buf;
  float* Strips = reinterpret_cast<float*>(W0 + (size_t)wst * w_tile);
  const int ncc = p.cin_pad / kConvTcKch;
  const int n_tiles = p.B * ((p.Tout + M - 1) / M) * p.ntiles;

  if (tid == 0) {
    for (int i = 0; i < ast; ++i) { tc::mbar_init(&a_full[i], CT_GATHER); tc::mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < wst; ++i) { tc::mbar_init(&w_full[i], 1); tc::mbar_init(&w_empty[i], 2); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    tc::setmaxnreg_dec<CT_PRODUCER_REGS>();
    if (warp == 3) {
      // ---------------------------------------------------------------- W producer
      if ((tid & 31) != 0) return;
      const int total = ncc * p.K * nparts;
      int wi = 0;
      for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
        const int nt = ct_tile<M>(p, tile).nt;
        for (int i = 0; i < total; ++i, ++wi) {
          const int st = wi % wst;
          if (wi >= wst) tc::mbar_wait(&w_empty[st], (uint32_t)(((wi / wst) - 1) & 1));
          const int part = i % nparts, tap = (i / nparts) % p.K, cc = i / (nparts * p.K);
          const size_t wt = (((size_t)tap * ncc + cc) * 2 + part) * p.ntiles + nt;
          tc::mbar_arrive_expect_tx(&w_full[st], w_tile);
          tc::bulk_g2s(W0 + (size_t)st * w_tile, p.wpk + wt * w_tile, w_tile, &w_full[st]);
        }
      }
      return;
    }
    // ------------------------------------------------------------------ A producer (warps 0-2)
    // A thread fetches TWO items (16 scalar or 4 vector loads in flight) before it converts either.
    const int n_items = R * KC;
    int ai = 0;
    for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
      const CtTile tl = ct_tile<M>(p, tile);
      const int n0row = tl.t0 - p.pad;            // sequence position of A row 0
      const long long len = p.lengths ? p.lengths[tl.b] : (long long)1 << 60;
      const float* xb = p.x + (long long)tl.b * p.sxb;
      const float* x2b = p.x2 ? p.x2 + (long long)tl.b * p.sx2b : nullptr;
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
            const float* s = xb + (long long)c0 * p.sxc + (long long)tau * p.sxt;
#pragma unroll
            for (int e = 0; e < 8; ++e) v[e] = (c0 + e < p.Cin) ? __ldg(s + e * p.sxc) : 0.f;
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
      for (int cc = 0; cc < ncc; ++cc, ++ai) {
        const int st = ai % ast;
        if (ai >= ast) tc::mbar_wait(&a_empty[st], (uint32_t)(((ai / ast) - 1) & 1));
        uint8_t* Ah = A0 + (size_t)st * a_buf;
        uint8_t* Al = Ah + a_part;
        for (int it0 = tid; it0 < n_items; it0 += 2 * CT_GATHER) {
          const int it1 = it0 + CT_GATHER;
          float va[8], vb[8];
          fetch(it0, cc, va);
          if (it1 < n_items) fetch(it1, cc, vb);
          put(it0, Ah, Al, va);
          if (it1 < n_items) put(it1, Ah, Al, vb);
        }
        tc::fence_proxy_async_smem();
        tc::mbar_arrive(&a_full[st]);
      }
    }
    return;
  }

  // -------------------------------------------------------------------- MMA + epilogue (warps 4-11)
  tc::setmaxnreg_inc<CT_CONSUMER_REGS>();
  const int wg = (warp - 4) >> 2, t = tid & 127;
  const uint32_t a_row0 = (uint32_t)wg * (64u * MB) * 16u, w_base = tc::smem_u32(W0);
  const uint32_t lbo_a = (uint32_t)R * 16u, lbo_b = (uint32_t)BN * 16u;
  const uint64_t ks_a = (2u * lbo_a) >> 4, ks_b = (2u * lbo_b) >> 4;
  constexpr int nk = kConvTcKch / 16;
  float* strip = Strips + wg * 64 * CT_EPI_LD;
  const bool gate = (p.flags & CONV_GATE) != 0;
  const int cout_real = gate ? p.Cout / 2 : p.Cout;
  int ai = 0, wi = 0;
  for (int tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const CtTile tl = ct_tile<M>(p, tile);
    float acc[MB][BN / 2];
#pragma unroll
    for (int j = 0; j < MB; ++j)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[j][i] = 0.f;
    const int wi0 = wi;
    for (int cc = 0; cc < ncc; ++cc, ++ai) {
      const int ast_i = ai % ast;
      tc::mbar_wait(&a_full[ast_i], (uint32_t)((ai / ast) & 1));
      const uint32_t ah = tc::smem_u32(A0) + (uint32_t)ast_i * a_buf + a_row0, al = ah + a_part;
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
#pragma unroll
            for (int j = 0; j < MB; ++j)
              for (int kk = 0; kk < nk; ++kk)
                tc::Wg<BN, 0>::ss(acc[j], ad + 64u * j + kk * ks_a, bd + kk * ks_b, 1u);   // + 64 rows (address >> 4)
          }
          tc::wg_commit();
          tc::wg_wait<1>();                    // everything but this slot's MMAs is done: release what they read
          if (t == 0 && wi > wi0) {
            tc::mbar_arrive(&w_empty[(wi - 1) % wst]);
            if (cc > 0 && tap == 0 && part == 0) tc::mbar_arrive(&a_empty[(ai - 1) % ast]);
          }
        }
      }
    }
    tc::wg_wait<0>();
#pragma unroll
    for (int j = 0; j < MB; ++j) tc::wg_hold(acc[j]);
    if (t == 0) {
      tc::mbar_arrive(&w_empty[(wi - 1) % wst]);
      tc::mbar_arrive(&a_empty[(ai - 1) % ast]);
    }

    // -------------------------------------------------------------- epilogue: thread = (row t % 64, 32-column half)
    const long long len = p.lengths ? p.lengths[tl.b] : (long long)1 << 60;
    float* yb = p.y + (long long)tl.b * cout_real * p.Tout;
    const float* rb = p.res ? p.res + (long long)tl.b * cout_real * p.Tout : nullptr;
    const int nt = tl.nt;
#pragma unroll
    for (int j = 0; j < MB; ++j) {
      const int tq = tl.t0 + (wg * MB + j) * 64 + (t & 63);
      const bool keep = !(p.flags & CONV_OUT_MASK) || tq < len;
#pragma unroll
      for (int ch = 0; ch < (BN + 63) / 64; ++ch) {
        tc::named_sync(2 + wg, 128);
        tc::acc_to_smem<BN>(acc[j], strip, CT_EPI_LD, 8 * ch, 8 * ch + 8);
        tc::named_sync(2 + wg, 128);
#pragma unroll 1
        for (int sub = 0; sub < 4; ++sub) {   // 8 columns at a time: the accumulators of the other rows stay live
          const int cl = (t >> 6) * 32 + sub * 8, c0 = ch * 64 + cl;
          if (c0 >= BN) continue;
          float vf[8];
#pragma unroll
          for (int i = 0; i < 8; ++i) vf[i] = strip[(t & 63) * CT_EPI_LD + cl + i];
          if (p.ilv) {   // interleaved store: ilv consecutive samples of one channel per thread (one 8 / 16-byte store)
            float* yi = p.y + (long long)tl.b * p.Cout * p.Tout;   // = [Cout / ilv][Tout * ilv]
            if (tq < p.Tout) {
#pragma unroll
              for (int i = 0; i < 8; i += 4) {
                const int cp = nt * BN + c0 + i;
                if (cp < p.Cout) {
                  float o[4];
#pragma unroll
                  for (int e = 0; e < 4; ++e) o[e] = ct_act(vf[i + e] + (p.bias ? __ldg(p.bias + cp + e) : 0.f), p.act);
                  if (p.ilv == 4) {
                    *reinterpret_cast<float4*>(yi + ((long long)(cp >> 2) * p.Tout + tq) * 4) = make_float4(o[0], o[1], o[2], o[3]);
                  } else {
                    *reinterpret_cast<float2*>(yi + ((long long)(cp >> 1) * p.Tout + tq) * 2) = make_float2(o[0], o[1]);
                    *reinterpret_cast<float2*>(yi + ((long long)((cp >> 1) + 1) * p.Tout + tq) * 2) = make_float2(o[2], o[3]);
                  }
                }
              }
            }
          } else {
            const bool live = tq < p.Tout;
            const int step = gate ? 2 : 1;
            // residual / accumulator loads of the strip first (all in flight), stores afterwards
            float add[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              float a = 0.f;
              const int cp = nt * BN + c0 + i;
              if (live && (i % step) == 0 && cp + (step - 1) < p.Cout) {
                const long long off = (long long)(gate ? (cp >> 1) : cp) * p.Tout + tq;
                if (rb) a = rb[off];
                if (p.flags & CONV_ACCUM) a += yb[off];
              }
              add[i] = a;
            }
            if (live) {
              if (gate) {
#pragma unroll
                for (int i = 0; i < 8; i += 2) {
                  const int cp = nt * BN + c0 + i;
                  if (cp + 1 < p.Cout) {
                    const float a = vf[i] + __ldg(p.bias + cp);
                    const float g = vf[i + 1] + __ldg(p.bias + cp + 1);
                    float o = tanhf(a) * (1.f / (1.f + expf(-g)));
                    if (!keep) o = 0.f;
                    yb[(long long)(cp >> 1) * p.Tout + tq] = o + add[i];
                  }
                }
              } else {
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  const int co = nt * BN + c0 + i;
                  if (co < p.Cout) {
                    float o = ct_act(vf[i] + (p.bias ? __ldg(p.bias + co) : 0.f), p.act);
                    if (!keep) o = 0.f;
                    yb[(long long)co * p.Tout + tq] = o + add[i];
                  }
                }
              }
            }
          }
        }
      }
    }
  }
}

// 64-row blocks per consumer warpgroup: two (256-row tiles, each weight tile feeds 256 rows) while the two
// accumulator sets fit the consumer's registers
static int conv_tc_mb(int bn) { return bn <= 192 ? 2 : 1; }

static size_t conv_tc_smem_bytes(const ConvTcParams& p, int mb, int ast, int wst) {
  const int R = 128 * mb + (p.K - 1) * p.dil;
  const size_t a_buf = (size_t)(kConvTcKch / 8) * R * 16 * (p.nsplit == 3 ? 2 : 1);
  return (size_t)ast * a_buf + (size_t)wst * kConvTcKch * p.bn * 2 + CT_STRIP_BYTES + 128;
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
  // the deepest A ring (up to 4 stages) that fits beside 4 weight slots, then weight slots with what is left;
  // a 256-row tile that does not leave room for 2 A stages falls back to 128 rows
  constexpr size_t kSmemMax = 227 * 1024 - 512;
  int mb = conv_tc_mb(p.bn);
  if (mb == 2 && conv_tc_smem_bytes(p, 2, 2, CT_WST_MIN) > kSmemMax) mb = 1;
  int ast = CT_AST, wst = CT_WST_MIN;
  while (ast > 2 && conv_tc_smem_bytes(p, mb, ast, wst) > kSmemMax) --ast;
  while (wst < CT_WST && conv_tc_smem_bytes(p, mb, ast, wst + 1) <= kSmemMax) ++wst;
  const size_t smem = conv_tc_smem_bytes(p, mb, ast, wst);
  if (smem > kSmemMax) { set_error("conv_tc: tile does not fit shared memory"); return SVCB_E_UNSUPPORTED; }
  const int n_sm = device_sm_count();
  if (n_sm <= 0) { set_error("conv_tc: cannot query the SM count"); return SVCB_E_CUDA; }
  const long long n_tiles = (long long)p.B * ((p.Tout + 128 * mb - 1) / (128 * mb)) * p.ntiles;
  const int grid = (int)(n_tiles < n_sm ? n_tiles : n_sm);
  const int cout_real = (p.flags & CONV_GATE) ? p.Cout / 2 : p.Cout;
  char kname[64];
  snprintf(kname, sizeof(kname), "conv_tc_%s_%dto%d_k%d_o1", p.nsplit == 3 ? "bf16x3" : "bf16", p.Cin, p.Cout, p.K);
  KernelScope ks(kname, s,
                 2.0 * p.Cin * p.K * p.Cout * (double)p.Tout * p.B,
                 4.0 * ((double)p.B * p.Cin * p.Tin + (double)p.B * cout_real * p.Tout * (p.res ? 2 : 1)) +
                     2.0 * (double)p.Cin * p.K * p.Cout);
  switch (p.bn / 16 * 2 + mb - 1) {
#define SVCB_CONV_BN(nb, mb)                                                             \
  case nb * 2 + mb - 1: {                                                                \
    static DevSmemCache attr_cache;                                                      \
    SVCB_CUDA_CHECK(ensure_dyn_smem(conv_tc_kernel<16 * nb, mb>, smem, attr_cache));     \
    conv_tc_kernel<16 * nb, mb><<<grid, CT_THREADS, smem, s>>>(p, ast, wst);             \
    break;                                                                               \
  }
    SVCB_CONV_BN(1, 1) SVCB_CONV_BN(2, 1) SVCB_CONV_BN(3, 1) SVCB_CONV_BN(4, 1) SVCB_CONV_BN(5, 1) SVCB_CONV_BN(6, 1)
    SVCB_CONV_BN(7, 1) SVCB_CONV_BN(8, 1) SVCB_CONV_BN(9, 1) SVCB_CONV_BN(10, 1) SVCB_CONV_BN(11, 1) SVCB_CONV_BN(12, 1)
    SVCB_CONV_BN(13, 1) SVCB_CONV_BN(14, 1) SVCB_CONV_BN(15, 1) SVCB_CONV_BN(16, 1)
    SVCB_CONV_BN(1, 2) SVCB_CONV_BN(2, 2) SVCB_CONV_BN(3, 2) SVCB_CONV_BN(4, 2) SVCB_CONV_BN(5, 2) SVCB_CONV_BN(6, 2)
    SVCB_CONV_BN(7, 2) SVCB_CONV_BN(8, 2) SVCB_CONV_BN(9, 2) SVCB_CONV_BN(10, 2) SVCB_CONV_BN(11, 2) SVCB_CONV_BN(12, 2)
#undef SVCB_CONV_BN
  }
  SVCB_LAUNCH_CHECK("conv_tc");
  return SVCB_OK;
}

}  // namespace svcb

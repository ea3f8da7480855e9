// Windowed relative-position self-attention of the prior encoder on the Hopper tensor cores.
//
// Replaces MultiHeadAttention.attention (vits/attentions.py:225-274, rel-pos helpers :294-347) in its banded
// form, SURVEY.md §8a row a3:
//   s_ij = (q_i/sqrt(d)) . k_j + [|j-i|<=w] (q_i/sqrt(d)) . Ek[j-i+w];  masked_fill(-1e4) where i or j >= len;
//   p = softmax_j(s);  o_i = sum_j p_ij v_j + sum_{|r|<=w} p_{i,i+r} Ev[r+w]
// (2 heads, d = 96, w = 4, T <= 2520).  Round 1 ran this on the fp32 FMA pipe at 18 TFLOP/s (8.1 ms per
// 32 x 10 s step); the two contractions are dense and belong on wgmma with split bf16 operands
// (a = a_hi + a_lo: a.b ~ a_hi.b_hi + a_lo.b_hi + a_hi.b_lo, fp32 accumulate, error ~2^-16 relative).
//
// Two kernels:
//   rel_attn_pack   q (pre-scaled by 1/sqrt(d)), k, v of [B, 3H, T] -> bf16 hi/lo operand images in tile
//                   order (one contiguous bulk copy per tile), K-major SWIZZLE_NONE panels of tc.cuh
//   rel_attn_tc     one CTA = (item, head, 128 queries) = two warpgroups of 64 query rows and a producer warp.
//                   Two passes over the 64-key tiles:
//                   pass 1  S = Q K^T (18 MMAs, N = 64, accumulators in registers) -> row max and row sum;
//                   pass 2  S again, P = exp(S - m) / l split to bf16 hi/lo in registers as the A operand of
//                           O += P V (12 MMAs, N = 96); no rescaling of O is ever needed.
//                   The relative-key logits q.Ek are ONE extra MMA group (N = 16) whose 9 values per row the
//                   softmax adds on the band; the relative-value term is added to O in the epilogue from the
//                   9 band probabilities.  Scores never leave the SM.
#include <cstdint>
#include <cstdio>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

namespace ra {
constexpr int D = 96, KCD = D / 8, TQ = 128, TK = 64, NREL = 9, W = 4;
constexpr uint32_t Q_PART = KCD * TQ * 16, Q_TILE = 2 * Q_PART;          // 49,152
constexpr uint32_t K_PART = KCD * TK * 16, K_TILE = 2 * K_PART;          // 24,576
constexpr uint32_t V_PART = (TK / 8) * D * 16, V_TILE = 2 * V_PART;      // 24,576
constexpr uint32_t E_PART = KCD * 16 * 16, E_BYTES = 2 * E_PART;         // 6,144 (Ek padded to 16 rows)
constexpr uint32_t OFF_Q = 0, OFF_K = OFF_Q + Q_TILE, OFF_V = OFF_K + 2 * K_TILE,
                   OFF_E = OFF_V + 2 * V_TILE, OFF_QE = OFF_E + E_BYTES, OFF_PB = OFF_QE + TQ * 12 * 4,
                   OFF_EV = OFF_PB + TQ * 12 * 4, SMEM = OFF_EV + NREL * D * 4;
constexpr int SM_WARPS = 8;          // two warpgroups of 64 query rows
constexpr int THREADS = (SM_WARPS + 1) * 32;
}  // namespace ra

size_t rel_attention_ws_bytes(int B, int heads, int T) {
  const size_t nq = (T + ra::TQ - 1) / ra::TQ, nk = (T + ra::TK - 1) / ra::TK;
  return (size_t)B * heads * (nq * ra::Q_TILE + nk * (ra::K_TILE + ra::V_TILE)) + 256;
}

__device__ __forceinline__ void ra_split8(const float (&v)[8], uint4& hi, uint4& lo) {
  __align__(16) __nv_bfloat162 h2[4], l2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    h2[k] = __floats2bfloat162_rn(v[2 * k], v[2 * k + 1]);
    const float2 f = __bfloat1622float2(h2[k]);
    l2[k] = __floats2bfloat162_rn(v[2 * k] - f.x, v[2 * k + 1] - f.y);
  }
  hi = *reinterpret_cast<const uint4*>(h2);
  lo = *reinterpret_cast<const uint4*>(l2);
}

// ------------------------------------------------------------------------------------------------ pack
// grid (key tiles of 64, B * heads); 256 threads
__global__ void __launch_bounds__(256)
rel_attn_pack_kernel(const float* __restrict__ qkv, uint8_t* __restrict__ qimg, uint8_t* __restrict__ kimg,
                     uint8_t* __restrict__ vimg, int H, int heads, int T, int nq, int nk) {
  using namespace ra;
  const int kt = blockIdx.x, bh = blockIdx.y;
  const int b = bh / heads, h = bh - b * heads;
  const float* qb = qkv + ((long long)b * 3 * H + (long long)h * D) * T;
  const float* kb = qb + (long long)H * T;
  const float* vb = kb + (long long)H * T;
  const float qscale = rsqrtf((float)D);
  const int qt = kt >> 1, rq0 = (kt & 1) * TK;
  uint8_t* qdst = qimg + ((size_t)bh * nq + qt) * Q_TILE;
  uint8_t* kdst = kimg + ((size_t)bh * nk + kt) * K_TILE;
  uint8_t* vdst = vimg + ((size_t)bh * nk + kt) * V_TILE;
  for (int item = threadIdx.x; item < KCD * TK; item += 256) {   // Q and K: (octet of head dims, time row)
    const int r = item % TK, kc = item / TK;
    const int t = kt * TK + r;
    float q8[8], k8[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const long long off = (long long)(kc * 8 + e) * T + t;
      q8[e] = t < T ? __ldg(qb + off) * qscale : 0.f;
      k8[e] = t < T ? __ldg(kb + off) : 0.f;
    }
    uint4 hi, lo;
    ra_split8(q8, hi, lo);
    *reinterpret_cast<uint4*>(qdst + (size_t)(kc * TQ + rq0 + r) * 16) = hi;
    *reinterpret_cast<uint4*>(qdst + Q_PART + (size_t)(kc * TQ + rq0 + r) * 16) = lo;
    ra_split8(k8, hi, lo);
    *reinterpret_cast<uint4*>(kdst + (size_t)(kc * TK + r) * 16) = hi;
    *reinterpret_cast<uint4*>(kdst + K_PART + (size_t)(kc * TK + r) * 16) = lo;
  }
  for (int item = threadIdx.x; item < (TK / 8) * D; item += 256) {  // V: (octet of keys, head dim)
    const int n = item % D, kc = item / D;
    const int t0 = kt * TK + kc * 8;
    float v8[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) v8[e] = (t0 + e < T) ? __ldg(vb + (long long)n * T + t0 + e) : 0.f;
    uint4 hi, lo;
    ra_split8(v8, hi, lo);
    *reinterpret_cast<uint4*>(vdst + (size_t)(kc * D + n) * 16) = hi;
    *reinterpret_cast<uint4*>(vdst + V_PART + (size_t)(kc * D + n) * 16) = lo;
  }
  if ((kt & 1) == 0 && kt + 1 >= nk) {   // the second half of the last (ragged) query tile has no key tile: zero it
    for (int item = threadIdx.x; item < KCD * TK; item += 256) {
      const int r = item % TK, kc = item / TK;
      *reinterpret_cast<uint4*>(qdst + (size_t)(kc * TQ + TK + r) * 16) = make_uint4(0, 0, 0, 0);
      *reinterpret_cast<uint4*>(qdst + Q_PART + (size_t)(kc * TQ + TK + r) * 16) = make_uint4(0, 0, 0, 0);
    }
  }
}

// ------------------------------------------------------------------------------------------------ attention
// D (+)= A_hi B_hi + A_lo B_hi + A_hi B_lo over nk K-chunks of 16 (A and B K-major panels)
template <int N>
__device__ __forceinline__ void ra_mma3(float (&d)[N / 2], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, int nk,
                                        uint64_t ksa, uint64_t ksb) {
#pragma unroll 1
  for (int kk = 0; kk < nk; ++kk) {
    tc::Wg<N, 0>::ss(d, a_hi + kk * ksa, b_hi + kk * ksb, 1u);
    tc::Wg<N, 0>::ss(d, a_lo + kk * ksa, b_hi + kk * ksb, 1u);
    tc::Wg<N, 0>::ss(d, a_hi + kk * ksa, b_lo + kk * ksb, 1u);
  }
}

__device__ __forceinline__ void ra_split2(float a, float b, uint32_t& hi, uint32_t& lo) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  const float2 f = __bfloat1622float2(h2);
  const __nv_bfloat162 l2 = __floats2bfloat162_rn(a - f.x, b - f.y);
  hi = *reinterpret_cast<const uint32_t*>(&h2);
  lo = *reinterpret_cast<const uint32_t*>(&l2);
}

__global__ void __launch_bounds__(ra::THREADS, 1)
rel_attn_tc_kernel(const uint8_t* __restrict__ qimg, const uint8_t* __restrict__ kimg, const uint8_t* __restrict__ vimg,
                   const float* __restrict__ ek, const float* __restrict__ ev, const long long* __restrict__ lengths,
                   float* __restrict__ out, int H, int heads, int T, int nq, int nk) {
  using namespace ra;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t q_full, k_full[2], k_empty[2], v_full[2], v_empty[2];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int warp_u = tc::warp_uniform_idx();
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int bh = b * heads + h;
  float* qe_s = reinterpret_cast<float*>(smem + OFF_QE);   // [128][12]: q_i . Ek[r]
  float* pb_s = reinterpret_cast<float*>(smem + OFF_PB);   // [128][12]: p_{i, i+r-4}
  float* ev_s = reinterpret_cast<float*>(smem + OFF_EV);   // [9][96]

  // Ek as a B operand: [n = 16 rows (9 used)][k = 96] bf16 hi/lo panels; Ev in fp32
  for (int item = tid; item < KCD * 16; item += THREADS) {
    const int n = item % 16, kc = item / 16;
    float e8[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) e8[e] = n < NREL ? __ldg(ek + n * D + kc * 8 + e) : 0.f;
    uint4 hi, lo;
    ra_split8(e8, hi, lo);
    *reinterpret_cast<uint4*>(smem + OFF_E + (size_t)(kc * 16 + n) * 16) = hi;
    *reinterpret_cast<uint4*>(smem + OFF_E + E_PART + (size_t)(kc * 16 + n) * 16) = lo;
  }
  for (int i = tid; i < NREL * D; i += THREADS) ev_s[i] = __ldg(ev + i);
  for (int i = tid; i < TQ * 12; i += THREADS) pb_s[i] = 0.f;
  if (tid == 0) {
    tc::mbar_init(&q_full, 1);
    for (int i = 0; i < 2; ++i) {
      tc::mbar_init(&k_full[i], 1); tc::mbar_init(&k_empty[i], 2); tc::mbar_init(&v_full[i], 1); tc::mbar_init(&v_empty[i], 2);
    }
    tc::fence_barrier_init();
  }
  tc::fence_proxy_async_smem();     // the Ek panels were written through the generic proxy
  __syncthreads();
  const int ntile = 2 * nk;          // key tiles visited: pass 1 then pass 2

  if (warp_u == SM_WARPS) {
    // ------------------------------------------------------------------------------------ producer
    if (tc::elect_one()) {
      tc::mbar_arrive_expect_tx(&q_full, Q_TILE);
      tc::bulk_g2s(smem + OFF_Q, qimg + ((size_t)bh * nq + qt) * Q_TILE, Q_TILE, &q_full);
      for (int i = 0; i < ntile; ++i) {
        const int kt = i < nk ? i : i - nk, buf = i & 1;
        if (i >= 2) tc::mbar_wait_parked(&k_empty[buf], (uint32_t)(((i >> 1) - 1) & 1));
        tc::mbar_arrive_expect_tx(&k_full[buf], K_TILE);
        tc::bulk_g2s(smem + OFF_K + (size_t)buf * K_TILE, kimg + ((size_t)bh * nk + kt) * K_TILE, K_TILE, &k_full[buf]);
        if (i >= nk) {
          const int vb = kt & 1;
          if (kt >= 2) tc::mbar_wait_parked(&v_empty[vb], (uint32_t)(((kt >> 1) - 1) & 1));
          tc::mbar_arrive_expect_tx(&v_full[vb], V_TILE);
          tc::bulk_g2s(smem + OFF_V + (size_t)vb * V_TILE, vimg + ((size_t)bh * nk + kt) * V_TILE, V_TILE, &v_full[vb]);
        }
      }
    }
    return;
  }
  // ------------------------------------------------------------------------------------ two warpgroups of 64 rows
  const int wg = warp >> 2, t = tid & 127, w = t >> 5, g = lane >> 2, c = lane & 3;
  const uint32_t sb = tc::smem_u32(smem);
  const uint32_t qrow = (uint32_t)wg * 64u * 16u;
  const uint64_t q_hi = tc::smem_desc(sb + OFF_Q + qrow, TQ * 16), q_lo = tc::smem_desc(sb + OFF_Q + Q_PART + qrow, TQ * 16);
  const uint64_t e_hi = tc::smem_desc(sb + OFF_E, 16 * 16), e_lo = tc::smem_desc(sb + OFF_E + E_PART, 16 * 16);
  constexpr uint64_t KS_Q = (2 * TQ * 16) >> 4, KS_K = (2 * TK * 16) >> 4, KS_E = (2 * 16 * 16) >> 4, KS_V = (2 * D * 16) >> 4;
  const long long len = lengths ? lengths[b] : (long long)T;
  int lrow[2], gi[2];
  bool row_masked[2];
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    lrow[hh] = wg * 64 + 16 * w + g + 8 * hh;     // row of the CTA tile
    gi[hh] = qt * TQ + lrow[hh];
    row_masked[hh] = gi[hh] >= len;
  }
  tc::mbar_wait_parked(&q_full, 0);
  {   // relative-key logits q_i . Ek[r], r < 9
    float qe[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) qe[i] = 0.f;
    tc::wg_fence();
    ra_mma3<16>(qe, q_hi, q_lo, e_hi, e_lo, D / 16, KS_Q, KS_E);
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_hold(qe);
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int col = 8 * i + 2 * c + (e & 1);
        if (col < NREL) qe_s[lrow[e >> 1] * 12 + col] = qe[4 * i + e];
      }
    __syncwarp();                                           // a row's entries are read by the four threads that wrote them
  }
  float m[2] = {-1e30f, -1e30f}, l[2] = {0.f, 0.f}, inv_l[2] = {0.f, 0.f};
  float o[48];
#pragma unroll
  for (int i = 0; i < 48; ++i) o[i] = 0.f;
  for (int i = 0; i < ntile; ++i) {
    const bool pass2 = i >= nk;
    const int kt = pass2 ? i - nk : i, buf = i & 1;
    if (i == nk) {   // combine the four threads' (max, sum) of each row
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
#pragma unroll
        for (int x = 1; x <= 2; x <<= 1) {
          const float mo = __shfl_xor_sync(0xffffffffu, m[hh], x), lo_ = __shfl_xor_sync(0xffffffffu, l[hh], x);
          const float mn = fmaxf(m[hh], mo);
          l[hh] = l[hh] * __expf(m[hh] - mn) + lo_ * __expf(mo - mn);
          m[hh] = mn;
        }
        inv_l[hh] = 1.f / l[hh];
      }
    }
    float sc[32];
    {
      tc::mbar_wait_parked(&k_full[buf], (uint32_t)((i >> 1) & 1));
      const uint64_t k_hi = tc::smem_desc(sb + OFF_K + buf * K_TILE, TK * 16), k_lo = tc::smem_desc(sb + OFF_K + buf * K_TILE + K_PART, TK * 16);
#pragma unroll
      for (int j = 0; j < 32; ++j) sc[j] = 0.f;
      tc::wg_fence();
      ra_mma3<64>(sc, q_hi, q_lo, k_hi, k_lo, D / 16, KS_Q, KS_K);
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_hold(sc);
      if (t == 0) tc::mbar_arrive(&k_empty[buf]);
    }
#pragma unroll
    for (int q = 0; q < 8; ++q)
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hh = e >> 1, j = kt * TK + 8 * q + 2 * c + (e & 1);
        const int r = j - gi[hh] + W;
        float sv = sc[4 * q + e];
        if ((unsigned)r < (unsigned)NREL) sv += qe_s[lrow[hh] * 12 + r];
        if (row_masked[hh] || j >= len) sv = -1e4f;
        if (j >= T) sv = -INFINITY;
        sc[4 * q + e] = sv;
      }
    if (!pass2) {
#pragma unroll
      for (int hh = 0; hh < 2; ++hh) {
        float mx = -INFINITY;
#pragma unroll
        for (int q = 0; q < 8; ++q) mx = fmaxf(mx, fmaxf(sc[4 * q + 2 * hh], sc[4 * q + 2 * hh + 1]));
        const float m_new = fmaxf(m[hh], mx);
        float sum = 0.f;
#pragma unroll
        for (int q = 0; q < 8; ++q) sum += __expf(sc[4 * q + 2 * hh] - m_new) + __expf(sc[4 * q + 2 * hh + 1] - m_new);
        l[hh] = l[hh] * __expf(m[hh] - m_new) + sum;
        m[hh] = m_new;
      }
    } else {
      uint32_t ph[4][4], pl[4][4];
#pragma unroll
      for (int q = 0; q < 8; ++q) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int hh = e >> 1;
          sc[4 * q + e] = __expf(sc[4 * q + e] - m[hh]) * inv_l[hh];
          const int r = kt * TK + 8 * q + 2 * c + (e & 1) - gi[hh] + W;
          if ((unsigned)r < (unsigned)NREL) pb_s[lrow[hh] * 12 + r] = sc[4 * q + e];
        }
        ra_split2(sc[4 * q], sc[4 * q + 1], ph[q >> 1][(q & 1) * 2], pl[q >> 1][(q & 1) * 2]);
        ra_split2(sc[4 * q + 2], sc[4 * q + 3], ph[q >> 1][(q & 1) * 2 + 1], pl[q >> 1][(q & 1) * 2 + 1]);
      }
      const int vb = kt & 1;
      tc::mbar_wait_parked(&v_full[vb], (uint32_t)((kt >> 1) & 1));
      const uint64_t v_hi = tc::smem_desc(sb + OFF_V + vb * V_TILE, D * 16), v_lo = tc::smem_desc(sb + OFF_V + vb * V_TILE + V_PART, D * 16);
      tc::wg_fence();
#pragma unroll
      for (int kk = 0; kk < TK / 16; ++kk) {
        tc::Wg<96, 0>::rs(o, ph[kk], v_hi + kk * KS_V, 1u);
        tc::Wg<96, 0>::rs(o, pl[kk], v_hi + kk * KS_V, 1u);
        tc::Wg<96, 0>::rs(o, ph[kk], v_lo + kk * KS_V, 1u);
      }
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_hold(o);
      if (t == 0) tc::mbar_arrive(&v_empty[vb]);
    }
  }
  // epilogue: O (+ relative-value band) -> out[b, h*96 + col, t]
  __syncwarp();                                             // pb_s entries of a row were written by its four threads
#pragma unroll
  for (int hh = 0; hh < 2; ++hh) {
    if (gi[hh] >= T) continue;
    float pb[NREL];
#pragma unroll
    for (int r = 0; r < NREL; ++r) pb[r] = pb_s[lrow[hh] * 12 + r];
    float* ob = out + ((long long)b * H + (long long)h * D) * T + gi[hh];
#pragma unroll
    for (int q = 0; q < 12; ++q)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = 8 * q + 2 * c + e;
        float v = o[4 * q + 2 * hh + e];
#pragma unroll
        for (int r = 0; r < NREL; ++r) v = fmaf(pb[r], ev_s[r * D + col], v);
        ob[(long long)col * T] = v;
      }
  }
}

int launch_rel_attention_tc(const float* qkv, const float* ek, const float* ev, const long long* lengths, float* out,
                            void* ws, size_t ws_bytes, int B, int H, int heads, int window, int T, cudaStream_t s) {
  if (H % heads || H / heads != ra::D || window != ra::W) {
    set_error("rel_attention_tc: built for head dim 96 and window 4 (vits/models.py:220-238)");
    return SVCB_E_UNSUPPORTED;
  }
  if (B <= 0 || T <= 0) return SVCB_OK;
  SVCB_TRY(check_workspace(ws, ws_bytes, rel_attention_ws_bytes(B, heads, T), "rel_attention_tc"));
  const int nq = (T + ra::TQ - 1) / ra::TQ, nk = (T + ra::TK - 1) / ra::TK;
  uint8_t* qimg = static_cast<uint8_t*>(ws);
  uint8_t* kimg = qimg + (size_t)B * heads * nq * ra::Q_TILE;
  uint8_t* vimg = kimg + (size_t)B * heads * nk * ra::K_TILE;
  {
    KernelScope ks("rel_attn_pack", s, 0.0, 8.0 * 3 * B * H * (double)T);
    rel_attn_pack_kernel<<<dim3(nk, B * heads), 256, 0, s>>>(qkv, qimg, kimg, vimg, H, heads, T, nq, nk);
    SVCB_LAUNCH_CHECK("rel_attn_pack");
  }
  static DevSmemCache attr_cache;
  SVCB_CUDA_CHECK(ensure_dyn_smem(rel_attn_tc_kernel, ra::SMEM, attr_cache));
  // survey FLOPs: the reference's dense form, 4 * H * T^2 per item (q k^T and p v; the rel-pos products are extra)
  KernelScope ks("rel_attn_tc", s, 4.0 * B * H * (double)T * T, 4.0 * 4 * B * H * (double)T);
  rel_attn_tc_kernel<<<dim3(nq, heads, B), ra::THREADS, ra::SMEM, s>>>(qimg, kimg, vimg, ek, ev, lengths, out, H, heads, T, nq, nk);
  SVCB_LAUNCH_CHECK("rel_attn_tc");
  return SVCB_OK;
}

}  // namespace svcb

// Whisper encoder self-attention on the Hopper tensor cores (head dim 64, no mask).
//
// Replaces MultiHeadAttention.qkv_attention (whisper/model.py:88-101): q, k scaled by d^-1/4 each
// (= scores / 8), softmax in fp32, w @ v — SURVEY.md §8a row a15.  Both products are wgmma.
//
// Operands come straight from the QKV GEMM, whose epilogue 4 writes the head-major layout of
// common.cuh qkv_heads_off: per (item, q|k|v, head) the positions are tiled ([.][8 octets][128 or 64 rows][8]
// bf16, items padded to 128 positions), so every operand tile is one contiguous no-swizzle panel and one
// bulk copy.
//   S = Q K^T   A = Q panel [8][128][8] (shared memory), B = K tile [8][64 keys][8]   (K-major, 4 MMAs of K = 16)
//   O += P V    A = P, bf16, straight from the S accumulator registers (the m64nN accumulator fragment is the
//               m64k16 A fragment), B = V tile [8 d-octets][64 keys][8] read as an MN-major operand (no
//               transpose pass): 8 keys x 16 B = one core matrix, key groups 128 B apart (LBO), d-octets
//               TK * 16 B apart (SBO)
// One CTA = (item, head, 128 queries): two warpgroups of 64 query rows (online softmax over the 64-key tiles,
// four threads per row) and a producer warp (one 8 KB bulk copy per K / V tile into a 4-slot ring).
// The output is written as the tile image the out-projection consumes.
// Ragged batches (lens != null): item b attends over its first T_b = lens[b] keys only; its key loop stops at
// ceil(T_b / 64) tiles, as a lone run of T_b positions does, so each of its query rows gets the same bits.  Query
// tiles wholly past T_b write zeros: the next layers still read those rows (a masked key's P = 0 times its V row),
// so they must stay finite.
#include <cstdint>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

namespace wa {
constexpr int D = 64, TQ = 128, TK = 64, NS = 4;
constexpr uint32_t Q_BYTES = (D / 8) * TQ * 16;    // 16,384
constexpr uint32_t T_BYTES = (D / 8) * TK * 16;    //  8,192  (one ring slot: a K or a V tile)
constexpr uint32_t OFF_Q = 0, OFF_R = OFF_Q + Q_BYTES, SMEM = OFF_R + NS * T_BYTES;
constexpr int THREADS = 288;
constexpr int CTAS_PER_SM = 2;
}  // namespace wa

__device__ __forceinline__ float wa_ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t wa_pack(float a, float b) {
  const __nv_bfloat162 h2 = __floats2bfloat162_rn(a, b);
  return *reinterpret_cast<const uint32_t*>(&h2);
}

__global__ void __launch_bounds__(wa::THREADS, wa::CTAS_PER_SM)
whisper_attn_tc_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out_img, int T, int Dm,
                       int vswap, const int* __restrict__ lens) {
  using namespace wa;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t q_full, r_full[NS], r_empty[NS];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int warp_u = tc::warp_uniform_idx();
  const int qt = blockIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int heads = Dm / 64, Tp = qkv_heads_tp(T);
  const int Tb = lens ? __ldg(lens + b) : T;
  const int nk = qt * TQ < Tb ? (Tb + TK - 1) / TK : 0;   // 0: a query tile past the item's end, written as zeros
  const int m_item = b * T;                       // first flat row of the item
  if (tid == 0) {
    tc::mbar_init(&q_full, 1);
    for (int i = 0; i < NS; ++i) { tc::mbar_init(&r_full[i], 1); tc::mbar_init(&r_empty[i], 2); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp_u == 8) {
    // ---------------------------------------------------------------- producer: ring order K_0 V_0 K_1 V_1 ..
    if (tc::elect_one()) {
      const __nv_bfloat16* qb = qkv + qkv_heads_off(b, 0, h, 0, 0, heads, Tp);
      const __nv_bfloat16* kb = qkv + qkv_heads_off(b, 1, h, 0, 0, heads, Tp);
      const __nv_bfloat16* vb = qkv + qkv_heads_off(b, 2, h, 0, 0, heads, Tp);
      tc::mbar_arrive_expect_tx(&q_full, Q_BYTES);
      tc::bulk_g2s(smem + OFF_Q, qb + (size_t)qt * (TQ * D), Q_BYTES, &q_full);
      int slot = 0;
      uint32_t ph = 0;
      for (int n = 0; n < 2 * nk; ++n) {
        const __nv_bfloat16* src = ((n & 1) ? vb : kb) + (size_t)(n >> 1) * (TK * D);
        if (n >= NS) tc::mbar_wait_parked(&r_empty[slot], ph ^ 1u);
        tc::mbar_arrive_expect_tx(&r_full[slot], T_BYTES);
        tc::bulk_g2s(smem + OFF_R + (size_t)slot * T_BYTES, src, T_BYTES, &r_full[slot]);
        if (++slot == NS) { slot = 0; ph ^= 1u; }
      }
    }
    return;
  }
  // ------------------------------------------------------------------ two warpgroups of 64 query rows
  const int wg = warp >> 2, t = tid & 127, w = t >> 5, g = lane >> 2, c = lane & 3;
  const uint32_t sb = tc::smem_u32(smem);
  const uint64_t dq = tc::smem_desc(sb + OFF_Q + (uint32_t)wg * 64u * 16u, TQ * 16);
  constexpr uint64_t KS_Q = (2 * TQ * 16) >> 4, KS_K = (2 * TK * 16) >> 4;
  // V as the MN-major B operand: LBO between 8-key groups, SBO between d-octets (vswap exchanges them)
  const uint32_t v_lbo = vswap ? TK * 16 : 128, v_sbo = vswap ? 128 : TK * 16;
  constexpr float kC = 0.125f * 1.4426950408889634f;   // d^-1/4 on q and on k, and log2(e)
  float o[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;
  float m0 = -INFINITY, m1 = -INFINITY, l0 = 0.f, l1 = 0.f;   // rows g and g + 8 of this warp's 16
  tc::mbar_wait_parked(&q_full, 0);
  for (int kt = 0; kt < nk; ++kt) {
    float sc[32];
    {   // S = Q K_kt^T
      const int n = 2 * kt, slot = n % NS;
      tc::mbar_wait_parked(&r_full[slot], (uint32_t)((n / NS) & 1));
      const uint64_t dk = tc::smem_desc(sb + OFF_R + slot * T_BYTES, TK * 16);
      tc::wg_fence();
#pragma unroll
      for (int kk = 0; kk < D / 16; ++kk) tc::Wg<64, 0>::ss(sc, dq + kk * KS_Q, dk + kk * KS_K, kk ? 1u : 0u);
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_hold(sc);
      if (t == 0) tc::mbar_arrive(&r_empty[slot]);
    }
    const int nvalid = Tb - kt * TK;             // >= 64 except in the item's last tile
    if (nvalid < TK) {
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (8 * i + 2 * c + (e & 1) >= nvalid) sc[4 * i + e] = -INFINITY;
    }
    float a0 = -INFINITY, a1 = -INFINITY;
#pragma unroll
    for (int i = 0; i < 8; ++i) { a0 = fmaxf(a0, fmaxf(sc[4 * i], sc[4 * i + 1])); a1 = fmaxf(a1, fmaxf(sc[4 * i + 2], sc[4 * i + 3])); }
    a0 = fmaxf(a0, __shfl_xor_sync(0xffffffffu, a0, 1)); a0 = fmaxf(a0, __shfl_xor_sync(0xffffffffu, a0, 2));
    a1 = fmaxf(a1, __shfl_xor_sync(0xffffffffu, a1, 1)); a1 = fmaxf(a1, __shfl_xor_sync(0xffffffffu, a1, 2));
    const float n0 = fmaxf(m0, a0 * kC), n1 = fmaxf(m1, a1 * kC);
    const float al0 = wa_ex2(m0 - n0), al1 = wa_ex2(m1 - n1);
    m0 = n0; m1 = n1; l0 *= al0; l1 *= al1;
#pragma unroll
    for (int i = 0; i < 8; ++i) { o[4 * i] *= al0; o[4 * i + 1] *= al0; o[4 * i + 2] *= al1; o[4 * i + 3] *= al1; }
    uint32_t pa[4][4];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const float p0 = wa_ex2(fmaf(sc[4 * i], kC, -m0)), p1 = wa_ex2(fmaf(sc[4 * i + 1], kC, -m0));
      const float p2 = wa_ex2(fmaf(sc[4 * i + 2], kC, -m1)), p3 = wa_ex2(fmaf(sc[4 * i + 3], kC, -m1));
      l0 += p0 + p1; l1 += p2 + p3;
      pa[i >> 1][(i & 1) * 2] = wa_pack(p0, p1);
      pa[i >> 1][(i & 1) * 2 + 1] = wa_pack(p2, p3);
    }
    {   // O += P_kt V_kt
      const int n = 2 * kt + 1, slot = n % NS;
      tc::mbar_wait_parked(&r_full[slot], (uint32_t)((n / NS) & 1));
      const uint64_t dv = tc::smem_desc(sb + OFF_R + slot * T_BYTES, v_lbo, v_sbo);
      tc::wg_fence();
#pragma unroll
      for (int kk = 0; kk < TK / 16; ++kk) tc::Wg<64, 1>::rs(o, pa[kk], dv + (uint64_t)kk * 16u, 1u);   // 16 keys = 256 B
      tc::wg_commit();
      tc::wg_wait<0>();
      tc::wg_hold(o);
      if (t == 0) tc::mbar_arrive(&r_empty[slot]);
    }
  }
  l0 += __shfl_xor_sync(0xffffffffu, l0, 1); l0 += __shfl_xor_sync(0xffffffffu, l0, 2);
  l1 += __shfl_xor_sync(0xffffffffu, l1, 1); l1 += __shfl_xor_sync(0xffffffffu, l1, 2);
  const float i0 = nk ? 1.f / l0 : 0.f, i1 = nk ? 1.f / l1 : 0.f;
  // O / sum(p) -> bf16, written as the A tile image of the out-projection ([M/128][D/64][8][128][8])
#pragma unroll
  for (int half = 0; half < 2; ++half) {
    const int ti = qt * TQ + wg * 64 + 16 * w + g + 8 * half;
    if (ti < T) {
      const int mrow = m_item + ti;
      __nv_bfloat16* dst = out_img + ((size_t)(mrow >> 7) * heads + h) * 8192 + (size_t)(mrow & 127) * 8 + 2 * c;
      const float inv = half ? i1 : i0;
#pragma unroll
      for (int i = 0; i < 8; ++i)
        *reinterpret_cast<uint32_t*>(dst + (size_t)i * 1024) = wa_pack(o[4 * i + 2 * half] * inv, o[4 * i + 2 * half + 1] * inv);
    }
  }
}

// qkv: head-major layout of common.cuh (B x 3 x heads blocks of Tp x 64, pad rows finite);
// out_img: tile image of [B*T, D]
int launch_whisper_attention_tc(const void* qkv_img, void* out_img, int B, int T, int D, int heads, int vswap,
                                cudaStream_t s, const int* lens) {
  if (D != heads * 64 || D % 64) { set_error("whisper_attention_tc: head dim must be 64"); return SVCB_E_UNSUPPORTED; }
  if (B <= 0 || T <= 0) return SVCB_OK;
  static DevSmemCache attr_cache;
  SVCB_CUDA_CHECK(ensure_dyn_smem(whisper_attn_tc_kernel, wa::SMEM, attr_cache));
  KernelScope ks("whisper_attn_tc", s, 4.0 * B * (double)T * T * D, 2.0 * 4 * B * (double)T * D);
  whisper_attn_tc_kernel<<<dim3((T + wa::TQ - 1) / wa::TQ, heads, B), wa::THREADS, wa::SMEM, s>>>(
      static_cast<const __nv_bfloat16*>(qkv_img), static_cast<__nv_bfloat16*>(out_img), T, D, vswap, lens);
  SVCB_LAUNCH_CHECK("whisper_attn_tc");
  return SVCB_OK;
}

// row-major [B*T, 3D] (q | k | v) -> the head-major layout  (unit tests; the encoder's QKV GEMM writes it directly)
__global__ void qkv_rowmajor_to_heads_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int B, int T, int Dm) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int oct_per_row = 3 * Dm / 8;
  if (idx >= (size_t)B * T * oct_per_row) return;
  const int m = (int)(idx / oct_per_row), n = (int)(idx % oct_per_row) * 8;
  const int w = n / Dm, hd = (n - w * Dm) >> 6, d = n & 63, b = m / T, t = m - b * T;
  *reinterpret_cast<uint4*>(dst + qkv_heads_off(b, w, hd, t, d, Dm >> 6, qkv_heads_tp(T))) =
      *reinterpret_cast<const uint4*>(src + (size_t)m * 3 * Dm + n);
}
int launch_qkv_rowmajor_to_heads(const void* src, void* dst, int B, int T, int D, cudaStream_t s) {
  const size_t n = (size_t)B * T * (3 * D / 8);
  qkv_rowmajor_to_heads_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(static_cast<const __nv_bfloat16*>(src),
                                                                          static_cast<__nv_bfloat16*>(dst), B, T, D);
  SVCB_LAUNCH_CHECK("qkv_rowmajor_to_heads");
  return SVCB_OK;
}

// tile image ([R/128][K/64][8][128][8]) -> row-major [R, K]  (unit tests)
__global__ void image_to_rowmajor_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst, int R, int K) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int kc_per_row = K / 8;
  if (idx >= (size_t)R * kc_per_row) return;
  const int m = (int)(idx / kc_per_row), k = (int)(idx % kc_per_row) * 8;
  const size_t off = ((size_t)(m >> 7) * (K / 64) + (k >> 6)) * 8192 + (size_t)((k & 63) >> 3) * 1024 + (size_t)(m & 127) * 8;
  *reinterpret_cast<uint4*>(dst + (size_t)m * K + k) = *reinterpret_cast<const uint4*>(src + off);
}
int launch_image_to_rowmajor(const void* src, void* dst, int R, int K, cudaStream_t s) {
  const size_t n = (size_t)R * (K / 8);
  image_to_rowmajor_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(static_cast<const __nv_bfloat16*>(src),
                                                                       static_cast<__nv_bfloat16*>(dst), R, K);
  SVCB_LAUNCH_CHECK("image_to_rowmajor");
  return SVCB_OK;
}

}  // namespace svcb

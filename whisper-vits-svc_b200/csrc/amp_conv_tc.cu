// AMP-block link on the tensor cores, as two kernels that each stream at their own roofline:
//
//   snake_pack   SnakeAlias(x) -> bf16 hi/lo operand image in HBM            (CUDA cores, 8 B/element)
//   amp_conv_tc  Conv1d(C->C, K, dilation) + bias (+residual, stage mean)    (wgmma)
//
// Together they replace one `SnakeAlias -> Conv1d [-> + x]` link of AMPBlock.forward
// (vits_decoder/bigv.py:50-58; SnakeAlias = vits_decoder/alias/act.py:124-128), SURVEY.md §8a rows
// a9/a10.  Fusing both into one CTA-per-tile kernel leaves the tensor pipe idle behind a latency-bound
// per-tile Snake prologue (20 x load->sync->FIR->sync->FIR->sync with one resident CTA); split, the Snake
// pass runs with 32 warps/SM and the conv kernel feeds its A operand with bulk (TMA-engine) copies.
//
// Operand image ("P8" layout): hi/lo bf16 [B][Cp/8][Lp][8], Lp = 32 + roundup(L,128) + 32, row =
// 32 + t; rows outside the sequence and channels >= C are zero.  One (octet, row-range) of the A
// tile is therefore ONE contiguous run of R*16 bytes = one bulk copy straight into the K-major
// panel layout of tc.cuh, the zero rows are the conv's zero padding, and every tap is the same
// tile addressed through a row-shifted descriptor.
#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

constexpr int TC_M = 128;
constexpr int P8_PAD = 32;

__host__ __device__ inline int p8_rows_of(int L) { return P8_PAD + (L + 127) / 128 * 128 + P8_PAD; }
int p8_rows(int L) { return p8_rows_of(L); }

// ------------------------------------------------------------------------------------ snake_pack
// Register-resident (same scheme as amp_block_fused's ab_snake_run; the earlier version staged x and
// the 2x-rate Snake values of an 8 x 506 tile in shared memory across three CTA barriers and was
// issue/latency-bound at 1.9 TB/s, profiles/r01_notes.md): no CTA barrier, no v buffer.  A warp owns one octet of
// channels x 32 image rows: lane = 4*channel + run, a thread computes 8 consecutive samples of one
// channel from the 24 inputs around them (six 16-byte loads), then the warp transposes its 8 x 32
// tile through 1 KB of shared memory so that every lane packs ONE image row (8 channels -> 16 bytes
// of bf16 hi and 16 of lo) and the warp stores 512 contiguous bytes per part.
constexpr int SP3_ROWS = 256;  // image rows per CTA (8 warps x 32)

// wide: the interior test of the vector form (a dense batch: VEC; a ragged item: what a lone call of its own length
// would choose, so that the same runs take the packed and the clamped arithmetic)
template <bool VEC>
__device__ __forceinline__ void sp3_run(const float* __restrict__ xr, int n0, int L, bool wide, const SnakeTapsV& tp,
                                        const float* f_up, const float* f_dn, float a_, float b_, float (&o)[8]) {
  // (the vector loads touch xr[n0-8 .. n0+16): keep them inside the row)
  if (wide ? (n0 - 8 >= 0 && n0 + 16 <= L) : (n0 - 6 >= 0 && n0 + 13 <= L - 1)) {
    float x[24];  // xr[n0-8 .. n0+16)
    if (VEC && (wide || (n0 - 8 >= 0 && n0 + 16 <= L))) {   // (a dense batch: wide is the same test)
#pragma unroll
      for (int q = 0; q < 6; ++q) {
        const float4 t4 = __ldg(reinterpret_cast<const float4*>(xr + n0 - 8) + q);
        x[4 * q] = t4.x; x[4 * q + 1] = t4.y; x[4 * q + 2] = t4.z; x[4 * q + 3] = t4.w;
      }
    } else {
      x[0] = x[1] = x[22] = x[23] = 0.f;   // never read
#pragma unroll
      for (int q = 2; q < 22; ++q) x[q] = __ldg(xr + n0 - 8 + q);
    }
    snake8_packed(x, tp, a_, 0.5f * b_, o);
  } else {  // a tap crosses a sequence end: replicate-clamped scalar path; rows outside [0, L) are zero
    const int mhi = 2 * L - 1;
    for (int i = 0; i < 8; ++i) {
      const int n = n0 + i;
      float acc = 0.f;
      if (n >= 0 && n < L) {
        for (int k = 0; k < 12; ++k) {
          const int m = min(max(2 * n - 5 + k, 0), mhi);
          const int a = m >> 1, q = m & 1;
          float u = 0.f;
          for (int d = q; d < q + 6; ++d) u = fmaf(__ldg(xr + min(max(a - 3 + d, 0), L - 1)), f_up[11 + q - 2 * d], u);
          u *= 2.f;
          const float sn = snake_sin(u * a_);
          acc = fmaf(fmaf(b_, sn * sn, u), f_dn[k], acc);
        }
      }
      o[i] = acc;
    }
  }
}

// RAG: a ragged batch (lens): a separate instantiation, so that the dense ones fold `wide` and Lb at compile time
template <bool VEC, int MINB, bool RAG>
__global__ void __launch_bounds__(256, MINB)
snake_pack3_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                   const float* __restrict__ ea, const float* __restrict__ inv_b,
                   const float* __restrict__ fu_g, const float* __restrict__ fd_g, const SnakeTapsV tp, int C, int L, int Lp,
                   const int* __restrict__ lens, int lscale) {
  __shared__ float tile[8][32 * 9];   // per warp: [row][channel], row stride 9 -> conflict-free both ways
  __shared__ float f_up[12], f_dn[12];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int oc = blockIdx.y, b = blockIdx.z;
  if (tid < 12) { f_up[tid] = __ldg(fu_g + tid); f_dn[tid] = __ldg(fd_g + tid); }
  __syncthreads();
  const int row0 = blockIdx.x * SP3_ROWS + warp * 32;   // first image row of this warp
  if (row0 >= Lp) return;                               // warp-uniform
  const int c = lane >> 2, run = lane & 3;
  const int ch = oc * 8 + c;
  const int n0 = row0 - P8_PAD + 8 * run;
  // a ragged item ends at Lb <= L: its rows past Lb are zero, as in the image of a lone call
  const int Lb = RAG ? __ldg(lens + b) * lscale : L;
  const bool wide = RAG ? (Lb & 3) == 0 : VEC;
  float o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;
  if (ch < C && n0 < Lb && n0 + 8 > 0) {
    sp3_run<VEC>(x + ((long long)b * C + ch) * L, n0, Lb, wide, tp, f_up, f_dn, __ldg(ea + ch), __ldg(inv_b + ch), o);
  }
  float* tw = tile[warp];
#pragma unroll
  for (int i = 0; i < 8; ++i) tw[(8 * run + i) * 9 + c] = o[i];
  __syncwarp();
  float r[8];
#pragma unroll
  for (int k = 0; k < 8; ++k) r[k] = tw[lane * 9 + k];
  __align__(16) __nv_bfloat162 h2[4], l2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    h2[k] = __floats2bfloat162_rn(r[2 * k], r[2 * k + 1]);
    const float2 f = __bfloat1622float2(h2[k]);
    l2[k] = __floats2bfloat162_rn(r[2 * k] - f.x, r[2 * k + 1] - f.y);
  }
  const long long img = ((long long)b * gridDim.y + oc) * Lp + row0 + lane;
  *reinterpret_cast<uint4*>(hi + img * 8) = *reinterpret_cast<const uint4*>(h2);
  if (lo) *reinterpret_cast<uint4*>(lo + img * 8) = *reinterpret_cast<const uint4*>(l2);
}

int snake_taps_from_device(const float* fu_dev, const float* fd_dev, SnakeTapsV* out) {
  float h[24];
  SVCB_CUDA_CHECK(cudaMemcpy(h, fu_dev, 12 * sizeof(float), cudaMemcpyDeviceToHost));
  SVCB_CUDA_CHECK(cudaMemcpy(h + 12, fd_dev, 12 * sizeof(float), cudaMemcpyDeviceToHost));
  *out = snake_taps_pack(h, h + 12);
  return SVCB_OK;
}

size_t p8_image_bytes(int B, int C, int L) {  // one of hi / lo
  const int cp = (C + 15) / 16 * 16;
  return (size_t)B * (cp / 8) * p8_rows_of(L) * 16;
}

int launch_snake_pack(const float* x, void* hi, void* lo, const float* ea, const float* inv_b, const float* fu,
                      const float* fd, int B, int C, int L, cudaStream_t s, const SnakeTapsV* taps, const int* lens,
                      int lscale) {
  if (B <= 0 || C <= 0 || L <= 0) return SVCB_OK;
  SnakeTapsV tp;
  if (taps) tp = *taps;
  else SVCB_TRY(snake_taps_from_device(fu, fd, &tp));
  const int cp = (C + 15) / 16 * 16, Lp = p8_rows_of(L);
  char kname[64];
  snprintf(kname, sizeof(kname), "snake_pack_c%d", C);
  KernelScope ks(kname, s, 0.0, (lo ? 8.0 : 6.0) * B * C * (double)L, 70.0 * B * C * (double)L);
  {
    dim3 grid3((Lp + SP3_ROWS - 1) / SP3_ROWS, cp / 8, B);
    auto* h = static_cast<__nv_bfloat16*>(hi);
    auto* l = static_cast<__nv_bfloat16*>(lo);
    const bool vec = (L & 3) == 0 && (reinterpret_cast<uintptr_t>(x) & 15) == 0;
    // 64 registers -> four CTAs (32 warps) per SM: each warp lives for one tile, so residency is
    // what hides its initial load latency (10.8 vs 11.4 ms/step with two CTAs)
    if (lens && vec) snake_pack3_kernel<true, 4, true><<<grid3, 256, 0, s>>>(x, h, l, ea, inv_b, fu, fd, tp, C, L, Lp, lens, lscale);
    else if (lens) snake_pack3_kernel<false, 4, true><<<grid3, 256, 0, s>>>(x, h, l, ea, inv_b, fu, fd, tp, C, L, Lp, lens, lscale);
    else if (vec) snake_pack3_kernel<true, 4, false><<<grid3, 256, 0, s>>>(x, h, l, ea, inv_b, fu, fd, tp, C, L, Lp, lens, lscale);
    else snake_pack3_kernel<false, 4, false><<<grid3, 256, 0, s>>>(x, h, l, ea, inv_b, fu, fd, tp, C, L, Lp, lens, lscale);
    SVCB_LAUNCH_CHECK("snake_pack");
  }
  return SVCB_OK;
}

// ------------------------------------------------------------------------------------ amp_conv_tc
// Persistent and warp-specialised: each CTA walks tiles (item, 128 samples) with a static stride.
//   warp 0 (one lane)  the A image rows of each tile (bulk copies, one buffer per tile in flight)
//   warp 1 (one lane)  the weight matrices: all resident in shared memory when they fit, else a ring of 2-8 slots
//   warps 2-3 (a lane each)  the residual (and the stage sum y_old) of the tiles of A buffer 0 / 1, one channel octet
//                      per slot of a ring per buffer: one bulk copy of the tile's samples per channel (a contiguous
//                      run of [B][C][L])
//   warpgroups 1-2     all taps x split parts as wgmma m64nCpk16 into register accumulators, then
//                      + bias (+res, +stage accumulation, /3) stored straight from the accumulator fragments
// The residual copies of a tile start as soon as its buffer's previous epilogue has released their slots, so their HBM
// time runs under the MMAs.  They need 16-byte aligned channel rows (L % 4 == 0); other lengths load the residual with
// generic loads after the MMAs (AmpPlan::nr == 0).
// Two schedules (amp_plan):
//   ping-pong    (PP) each consumer warpgroup owns whole 128-row tiles, as two m64 accumulators: warpgroup 0 the even
//                tiles of the CTA's walk, warpgroup 1 the odd ones, each with its own A buffer.  One warpgroup's
//                epilogue runs while the other's MMAs keep the tensor pipe busy.
//   cooperative  both warpgroups on one tile, 64 rows each, when two A buffers and two weight slots do not fit
//                (C = 160) or two 128-row accumulators would not fit the registers.
// Either way every output row sees the same wgmma sequence (tap, weight part, A part, K step) into one accumulator.
struct AmpPlan { int pingpong, resident, nabuf, nw, nr; size_t smem; };
constexpr int AMP_WMAX = 8;       // weight ring depth (max) when the taps do not stay resident
constexpr int AMP_WKEEP = 4;      // ring slots a streamed shape keeps when the residual wants the room
constexpr int AMP_RMAX = 16;      // residual slots per A buffer (max)
constexpr int AMP_RSTRIDE = TC_M + 4;   // floats per staged channel row: the epilogue's 4 channels x 8 rows hit 32 banks
constexpr int AMP_THREADS = 384;
constexpr int AMP_PRODUCER_REGS = 40, AMP_CONSUMER_REGS = 232;   // 128 * 40 + 256 * 232 <= 64 K registers
constexpr int AMP_PP_MAX_C = 112;  // ping-pong: two 64 x C accumulators per warpgroup (at C = 128 they spill)

template <int NC, bool PP>
__global__ void __launch_bounds__(AMP_THREADS, 1)
amp_conv_tc_kernel(const AmpConvParams p, const int resident, const int nabuf, const int nw, const int nr) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t a_full[2], a_empty[2], w_full[AMP_WMAX], w_empty[AMP_WMAX], w_res, order[2];
  __shared__ __align__(8) uint64_t r_full[2 * AMP_RMAX], r_empty[2 * AMP_RMAX];
  constexpr int MB = PP ? 2 : 1;    // 64-row accumulators per consumer warpgroup

  const int tid = threadIdx.x, warp = tc::warp_uniform_idx();
  const int P = p.dil * (p.K - 1) / 2;
  const int R = TC_M + (p.K - 1) * p.dil;
  const int KC = NC / 8;
  const int parts = p.nsplit == 3 ? 2 : 1;
  const uint32_t a_part = (uint32_t)KC * R * 16u;
  const uint32_t a_buf = a_part * parts;
  const uint32_t wb = (uint32_t)NC * NC * 2u;
  const int nch = p.K * parts;
  uint8_t* Abase = smem;
  uint8_t* Wbase = smem + (size_t)nabuf * a_buf;
  const int tpi = (p.L + TC_M - 1) / TC_M;
  const int ntiles = p.B * tpi;
  // staged residual: per A buffer nr slots of one channel octet each, [array (res, y_old)][8 channels][AMP_RSTRIDE]
  const int nres = (p.res ? 1 : 0) + (p.accum ? 1 : 0);
  const int nu = (p.C + 7) / 8;   // octets per tile
  const uint32_t r_slot = (uint32_t)nres * 8u * AMP_RSTRIDE * 4u;
  float* Rbase = reinterpret_cast<float*>(Wbase + (size_t)(resident ? nch : nw) * wb);

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&a_full[i], 1); tc::mbar_init(&a_empty[i], PP ? 1 : 2); }
    for (int i = 0; i < AMP_WMAX; ++i) { tc::mbar_init(&w_full[i], 1); tc::mbar_init(&w_empty[i], PP ? 1 : 2); }
    tc::mbar_init(&w_res, 1);
    for (int i = 0; i < 2; ++i) tc::mbar_init(&order[i], 1);
    for (int b = 0; b < nabuf; ++b)
      for (int i = b * AMP_RMAX; i < b * AMP_RMAX + nr; ++i) { tc::mbar_init(&r_full[i], 1); tc::mbar_init(&r_empty[i], PP ? 4 : 8); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp < 4) {
    // ------------------------------------------------------------------ producers
    tc::setmaxnreg_dec<AMP_PRODUCER_REGS>();
    if (warp == 0 && tc::elect_one()) {
      const uint32_t run = (uint32_t)R * 16u;
      int it = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int buf = it % nabuf;   // ping-pong: the buffer of the warpgroup that owns the tile
        if (it >= nabuf) tc::mbar_wait(&a_empty[buf], (uint32_t)(((it / nabuf) - 1) & 1));
        const int b = tile / tpi, t0 = (tile - b * tpi) * TC_M;
        tc::mbar_arrive_expect_tx(&a_full[buf], run * KC * parts);
        const long long row = P8_PAD + t0 - P;
        for (int part = 0; part < parts; ++part) {
          const uint8_t* src = reinterpret_cast<const uint8_t*>(part == 0 ? p.a_hi : p.a_lo);
          uint8_t* dst = Abase + (size_t)buf * a_buf + (size_t)part * a_part;
          for (int kc = 0; kc < KC; ++kc)
            tc::bulk_g2s(dst + (size_t)kc * run, src + (((long long)b * KC + kc) * p.Lp + row) * 16, run, &a_full[buf]);
        }
      }
    } else if (warp == 1 && tc::elect_one()) {
      if (resident) {
        tc::mbar_arrive_expect_tx(&w_res, wb * (uint32_t)nch);
        for (int i = 0; i < nch; ++i)
          tc::bulk_g2s(Wbase + (size_t)i * wb, p.wpk + ((size_t)(i / parts) * 2 + (i % parts)) * wb, wb, &w_res);
      } else {
        // one pass over the nch matrices per tile, in the order the tiles' MMAs consume them
        int wi = 0;
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
          for (int i = 0; i < nch; ++i, ++wi) {
            const int st = wi % nw;
            if (wi >= nw) tc::mbar_wait(&w_empty[st], (uint32_t)(((wi / nw) - 1) & 1));
            tc::mbar_arrive_expect_tx(&w_full[st], wb);
            tc::bulk_g2s(Wbase + (size_t)st * wb, p.wpk + ((size_t)(i / parts) * 2 + (i % parts)) * wb, wb, &w_full[st]);
          }
        }
      }
    } else if (warp >= 2 && warp - 2 < nabuf && nr > 0 && tc::elect_one()) {
      // warp 2 + buf stages the tiles of A buffer buf: a lane that waits for its buffer's epilogue to free a slot then
      // does not hold back the copies of the other buffer's next tile
      const int buf = warp - 2;
      int g = 0;   // position in the buffer's residual stream
      for (int tile = blockIdx.x + buf * gridDim.x; tile < ntiles; tile += nabuf * gridDim.x, g += nu) {
        const int b = tile / tpi, t0 = (tile - b * tpi) * TC_M;
        const uint32_t run = (uint32_t)min(TC_M, p.L - t0) * 4u;
        for (int u = 0; u < nu; ++u) {
          const int q = g + u, s = buf * AMP_RMAX + q % nr;
          if (q >= nr) tc::mbar_wait(&r_empty[s], (uint32_t)(((q / nr) - 1) & 1));
          const int nc = min(8, p.C - 8 * u);
          tc::mbar_arrive_expect_tx(&r_full[s], run * (uint32_t)(nres * nc));
          float* slot = Rbase + (size_t)(buf * nr + q % nr) * (r_slot / 4u);
          for (int a = 0; a < nres; ++a) {
            const float* src = ((a == 0 && p.res) ? p.res : p.y) + ((long long)b * p.C + 8 * u) * p.L + t0;
            float* dst = slot + a * 8 * AMP_RSTRIDE;   // an octet's arrays are 8 rows apart even when it has fewer channels
            for (int c = 0; c < nc; ++c, src += p.L, dst += AMP_RSTRIDE) tc::bulk_g2s(dst, src, run, &r_full[s]);
          }
        }
      }
    }
    return;
  }

  // -------------------------------------------------------------------- MMA + epilogue (warpgroups 1-2)
  tc::setmaxnreg_inc<AMP_CONSUMER_REGS>();
  const int wg = (warp - 4) >> 2, t = tid & 127;
  const uint32_t a0 = tc::smem_u32(Abase), w0 = tc::smem_u32(Wbase);
  const uint32_t lbo_a = (uint32_t)R * 16u, lbo_b = (uint32_t)NC * 16u;
  const uint64_t ks_a = (2u * lbo_a) >> 4, ks_b = (2u * lbo_b) >> 4;
  constexpr int NK = NC / 16;
  const bool do_div = p.out_div != 0.f;
  if (resident) tc::mbar_wait(&w_res, 0);
  for (int it = PP ? wg : 0;; it += PP ? 2 : 1) {
    const int tile = blockIdx.x + it * gridDim.x;
    if (tile >= ntiles) break;
    const int buf = it % nabuf;
    const int b = tile / tpi, t0 = (tile - b * tpi) * TC_M;
    tc::mbar_wait(&a_full[buf], (uint32_t)((it / nabuf) & 1));
    // Ping-pong: wait until the other warpgroup has issued every MMA of tile it - 1 (its ((it - 1) / 2)-th arrival
    // here).  The two then do not share the tensor pipe, and they consume the weight stream strictly in tile order,
    // which its parity waits need: a warpgroup that ran a tile ahead could take a slot's earlier phase for its own.
    if (PP && it > 0) tc::mbar_wait(&order[wg], (uint32_t)(((it - 1) >> 1) & 1));
    const uint32_t a_hi = a0 + (uint32_t)buf * a_buf + (PP ? 0u : (uint32_t)wg * 64u * 16u), a_lo = a_hi + a_part;
    float acc[MB][NC / 2];
#pragma unroll
    for (int m = 0; m < MB; ++m)
#pragma unroll
      for (int i = 0; i < NC / 2; ++i) acc[m][i] = 0.f;
    int i = 0;
    for (int tap = 0; tap < p.K; ++tap) {
      const uint32_t tap_off = (uint32_t)(tap * p.dil) * 16u;
      for (int part = 0; part < parts; ++part, ++i) {
        uint32_t wbase;
        int st = 0;
        if (resident) {
          wbase = w0 + (uint32_t)i * wb;
        } else {
          const int wi = it * nch + i;   // position in the weight stream
          st = wi % nw;
          tc::mbar_wait(&w_full[st], (uint32_t)((wi / nw) & 1));
          wbase = w0 + (uint32_t)st * wb;
        }
        const int n_a = (part == 0 && parts == 2) ? 2 : 1;  // Wh meets Ah and Al; Wl meets Ah
        const uint64_t bd = tc::smem_desc(wbase, lbo_b);
        tc::wg_fence();
        for (int ap = 0; ap < n_a; ++ap) {
          const uint64_t ad = tc::smem_desc((ap == 0 ? a_hi : a_lo) + tap_off, lbo_a);
#pragma unroll
          for (int m = 0; m < MB; ++m)
#pragma unroll
            for (int kk = 0; kk < NK; ++kk) tc::Wg<NC, 0>::ss(acc[m], ad + 64u * m + kk * ks_a, bd + kk * ks_b, 1u);   // + 64 rows (address >> 4)
        }
        tc::wg_commit();
        if (!resident) {
          tc::wg_wait<0>();
          if (t == 0) tc::mbar_arrive(&w_empty[st]);
        }
      }
    }
    if (PP && t == 0) tc::mbar_arrive(&order[wg ^ 1]);
    tc::wg_wait<0>();
#pragma unroll
    for (int m = 0; m < MB; ++m) tc::wg_hold(acc[m]);
    if (t == 0) tc::mbar_arrive(&a_empty[buf]);

    // epilogue from the fragments: d[4 j + e] is row 16 w + l/4 + 8 (e/2), column 8 j + 2 (l%4) + e%2, so the 8 lanes
    // of a column cover 8 consecutive samples, one 32-byte sector of [B][C][L].
    const int w = t >> 5, l = t & 31;
    const long long yb = (long long)b * p.C * p.L;
    if (nr > 0) {
      // residual staged in shared memory: one octet (slot) at a time, released once all its rows are read
      const int g0 = (it / nabuf) * nu;
#pragma unroll
      for (int j = 0; j < NC / 8; ++j) {
        if (j >= nu) break;
        const int g = g0 + j, s = g % nr;
        tc::mbar_wait(&r_full[buf * AMP_RMAX + s], (uint32_t)((g / nr) & 1));
        const float* sr = Rbase + (size_t)(buf * nr + s) * (r_slot / 4u);
#pragma unroll
        for (int m = 0; m < MB; ++m) {
          const int r0 = (PP ? 64 * m : 64 * wg) + 16 * w + (l >> 2);   // row in the tile
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int c = 2 * (l & 3) + (e & 1), co = 8 * j + c, tr = r0 + 8 * (e >> 1), tt = t0 + tr;
            if (co < p.C && tt < p.L) {
              float a = p.res ? sr[c * AMP_RSTRIDE + tr] : 0.f;
              if (p.accum) a += sr[((nres - 1) * 8 + c) * AMP_RSTRIDE + tr];
              float o = acc[m][4 * j + e] + __ldg(p.bias + co) + a;
              // a real (uniform) branch: if-converted, the division would run its x/0 slow path per element
              if (do_div) { asm volatile(""); o = o / p.out_div; }
              p.y[yb + (long long)co * p.L + tt] = o;
            }
          }
        }
        __syncwarp();
        if (l == 0) tc::mbar_arrive(&r_empty[buf * AMP_RMAX + s]);
      }
      continue;
    }
    // generic loads: all residual / stage loads are issued before the first store
#pragma unroll
    for (int m = 0; m < MB; ++m) {
      const int r0 = t0 + (PP ? 64 * m : 64 * wg) + 16 * w + (l >> 2);
      float add[NC / 2];
#pragma unroll
      for (int j = 0; j < NC / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int co = 8 * j + 2 * (l & 3) + (e & 1), tt = r0 + 8 * (e >> 1);
          float a = 0.f;
          if (co < p.C && tt < p.L) {
            const long long off = yb + (long long)co * p.L + tt;
            if (p.res) a = p.res[off];
            if (p.accum) a += p.y[off];
          }
          add[4 * j + e] = a;
        }
#pragma unroll
      for (int j = 0; j < NC / 8; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int co = 8 * j + 2 * (l & 3) + (e & 1), tt = r0 + 8 * (e >> 1);
          if (co < p.C && tt < p.L) {
            float o = acc[m][4 * j + e] + __ldg(p.bias + co) + add[4 * j + e];
            // a real (uniform) branch: if-converted, the division would run its x/0 slow path per element
            if (do_div) { asm volatile(""); o = o / p.out_div; }
            p.y[yb + (long long)co * p.L + tt] = o;
          }
        }
    }
  }
}

// Resident weights when all nch matrices fit beside two A buffers; else a weight ring of as many slots as fit
// (2-8) beside two A buffers, or beside one (C = 160).  Ping-pong needs the two A buffers.
// nres (0-2) arrays are staged (residual, stage sum): each A buffer gets up to one slot per channel octet of a tile in
// the room left beside the resident weights or AMP_WKEEP ring slots; the ring takes what the residual leaves.
static AmpPlan amp_plan(int Cp, int K, int dil, int nsplit, int nres) {
  const int R = TC_M + (K - 1) * dil;
  const int parts = nsplit == 3 ? 2 : 1;
  const size_t a_buf = (size_t)(Cp / 8) * R * 16 * parts;
  const size_t wb = (size_t)Cp * Cp * 2;
  const size_t nch = (size_t)K * parts;
  const size_t r_slot = (size_t)nres * 8 * AMP_RSTRIDE * 4;
  const size_t limit = 227 * 1024 - 1024;
  AmpPlan pl;
  pl.resident = 2 * a_buf + nch * wb <= limit;
  pl.nabuf = (pl.resident || 2 * a_buf + 2 * wb <= limit) ? 2 : 1;
  const size_t left = limit - std::min(limit, pl.nabuf * a_buf);
  const size_t keep = pl.resident ? nch * wb : std::min<size_t>(AMP_WKEEP, left / wb) * wb;
  pl.nr = nres ? (int)std::min<size_t>(std::min(Cp / 8, AMP_RMAX), (left - std::min(left, keep)) / (pl.nabuf * r_slot)) : 0;
  const size_t r_bytes = pl.nabuf * pl.nr * r_slot;
  pl.nw = pl.resident ? 0 : (int)std::min<size_t>(AMP_WMAX, (left - std::min(left, r_bytes)) / wb);
  pl.pingpong = pl.nabuf == 2 && Cp <= AMP_PP_MAX_C;
  pl.smem = pl.nabuf * a_buf + (pl.resident ? nch : (size_t)pl.nw) * wb + r_bytes + 128;
  return pl;
}

size_t amp_conv_tc_smem_bytes(int Cp, int K, int dil, int nsplit) { return amp_plan(Cp, K, dil, nsplit, 0).smem; }

int launch_amp_conv_tc(const AmpConvParams& p, cudaStream_t s) {
  if (p.Cp % 16 || p.Cp < 16 || p.Cp > 256 || p.Cp < p.C || (p.nsplit != 1 && p.nsplit != 3)) {
    set_error("amp_conv_tc: bad channel padding / nsplit");
    return SVCB_E_BAD_SHAPE;
  }
  if (p.dil * (p.K - 1) / 2 > P8_PAD || p.Lp != p8_rows_of(p.L) || !p.a_hi || (p.nsplit == 3 && !p.a_lo)) {
    set_error("amp_conv_tc: operand image does not match (halo > 32 rows or wrong Lp)");
    return SVCB_E_BAD_SHAPE;
  }
  // the staged residual is bulk-copied by channel row: rows must start and end on 16 bytes
  const bool stage = (p.L % 4 == 0) && (reinterpret_cast<uintptr_t>(p.res) & 15) == 0 &&
                     (!p.accum || (reinterpret_cast<uintptr_t>(p.y) & 15) == 0);
  const AmpPlan pl = amp_plan(p.Cp, p.K, p.dil, p.nsplit, stage ? (p.res ? 1 : 0) + (p.accum ? 1 : 0) : 0);
  if ((!pl.resident && pl.nw < 1) || pl.smem > 227 * 1024 - 512) {
    set_error("amp_conv_tc: tile does not fit shared memory");
    return SVCB_E_UNSUPPORTED;
  }
  const int n_sm = device_sm_count();
  if (n_sm <= 0) { set_error("amp_conv_tc: cannot query the SM count"); return SVCB_E_CUDA; }
  const int ntiles = p.B * ((p.L + TC_M - 1) / TC_M);
  const int grid = std::min(ntiles, n_sm);
  const double macs = (double)p.B * p.L * p.C * p.C * p.K;
  char kname[64];
  snprintf(kname, sizeof(kname), "amp_conv_tc_%s_c%dk%d", p.nsplit == 3 ? "bf16x3" : "bf16", p.C, p.K);
  KernelScope ks(kname, s, 2.0 * macs,
                 (double)p.B * p.C * p.L * ((p.nsplit == 3 ? 4.0 : 2.0) + 4.0 * (p.res ? 2 : 1)));
  switch (p.Cp / 16 * 2 + pl.pingpong) {
#define SVCB_AMP_NC(nb, pp)                                                                                      \
  case nb * 2 + pp: {                                                                                            \
    static DevSmemCache attr_cache;                                                                              \
    SVCB_CUDA_CHECK(ensure_dyn_smem(amp_conv_tc_kernel<16 * nb, pp>, pl.smem, attr_cache));                      \
    amp_conv_tc_kernel<16 * nb, pp><<<grid, AMP_THREADS, pl.smem, s>>>(p, pl.resident, pl.nabuf, pl.nw, pl.nr); \
    break;                                                                                                       \
  }
    SVCB_AMP_NC(1, 0) SVCB_AMP_NC(2, 0) SVCB_AMP_NC(3, 0) SVCB_AMP_NC(4, 0) SVCB_AMP_NC(5, 0) SVCB_AMP_NC(6, 0)
    SVCB_AMP_NC(7, 0) SVCB_AMP_NC(8, 0) SVCB_AMP_NC(9, 0) SVCB_AMP_NC(10, 0) SVCB_AMP_NC(11, 0) SVCB_AMP_NC(12, 0)
    SVCB_AMP_NC(13, 0) SVCB_AMP_NC(14, 0) SVCB_AMP_NC(15, 0) SVCB_AMP_NC(16, 0)
    SVCB_AMP_NC(1, 1) SVCB_AMP_NC(2, 1) SVCB_AMP_NC(3, 1) SVCB_AMP_NC(4, 1) SVCB_AMP_NC(5, 1) SVCB_AMP_NC(6, 1)
    SVCB_AMP_NC(7, 1)
#undef SVCB_AMP_NC
  }
  SVCB_LAUNCH_CHECK("amp_conv_tc");
  return SVCB_OK;
}

}  // namespace svcb

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

template <bool VEC>
__device__ __forceinline__ void sp3_run(const float* __restrict__ xr, int n0, int L, const SnakeTapsV& tp,
                                        const float* f_up, const float* f_dn, float a_, float b_, float (&o)[8]) {
  // (the vector loads touch xr[n0-8 .. n0+16): keep them inside the row)
  if (VEC ? (n0 - 8 >= 0 && n0 + 16 <= L) : (n0 - 6 >= 0 && n0 + 13 <= L - 1)) {
    float x[24];  // xr[n0-8 .. n0+16)
    if (VEC) {
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

template <bool VEC, int MINB>
__global__ void __launch_bounds__(256, MINB)
snake_pack3_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                   const float* __restrict__ ea, const float* __restrict__ inv_b,
                   const float* __restrict__ fu_g, const float* __restrict__ fd_g, const SnakeTapsV tp, int C, int L, int Lp) {
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
  float o[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) o[i] = 0.f;
  if (ch < C && n0 < L && n0 + 8 > 0) {
    sp3_run<VEC>(x + ((long long)b * C + ch) * L, n0, L, tp, f_up, f_dn, __ldg(ea + ch), __ldg(inv_b + ch), o);
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
                      const float* fd, int B, int C, int L, cudaStream_t s, const SnakeTapsV* taps) {
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
    if (vec) snake_pack3_kernel<true, 4><<<grid3, 256, 0, s>>>(x, h, l, ea, inv_b, fu, fd, tp, C, L, Lp);
    else snake_pack3_kernel<false, 4><<<grid3, 256, 0, s>>>(x, h, l, ea, inv_b, fu, fd, tp, C, L, Lp);
    SVCB_LAUNCH_CHECK("snake_pack");
  }
  return SVCB_OK;
}

// ------------------------------------------------------------------------------------ amp_conv_tc
// Persistent: each CTA walks tiles (item, 128 samples) with a static stride.
//   producer thread  A image rows of tile i+1 (bulk copies, 1-2 buffers) and the weight tiles
//                    (all taps resident in shared memory when they fit, else a 2-slot ring per tile)
//   2 warpgroups     64 rows each: all taps x split parts of tile i as wgmma m64nCpk16 into register
//                    accumulators, then +bias (+res, +stage accumulation, /3) through a shared-memory strip
//                    (64 columns at a time) -> coalesced stores
struct AmpPlan { int resident, nabuf, nw; size_t smem; };
constexpr int AMP_WMAX = 2;     // weight ring depth when the taps do not stay resident
constexpr int AMP_EPI_LD = 72;  // floats per row of an epilogue strip
constexpr int AMP_THREADS = 288;
constexpr size_t AMP_STRIP_BYTES = 2 * 64 * AMP_EPI_LD * 4;

template <int NC>
__global__ void __launch_bounds__(AMP_THREADS, 1)
amp_conv_tc_kernel(const AmpConvParams p, const int resident, const int nabuf, const int nw) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t a_full[2], a_empty[2], w_full[AMP_WMAX], w_empty[AMP_WMAX], w_res;

  const int tid = threadIdx.x, warp = tid >> 5;
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
  float* Strips = reinterpret_cast<float*>(Wbase + (size_t)(resident ? nch : nw) * wb);
  const int tpi = (p.L + TC_M - 1) / TC_M;
  const int ntiles = p.B * tpi;

  if (tid == 0) {
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&a_full[i], 1); tc::mbar_init(&a_empty[i], 2); }
    for (int i = 0; i < AMP_WMAX; ++i) { tc::mbar_init(&w_full[i], 1); tc::mbar_init(&w_empty[i], 2); }
    tc::mbar_init(&w_res, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (tid == 256) {
    // ---------------------------------------------------------------- producer
    if (resident) {
      tc::mbar_arrive_expect_tx(&w_res, wb * (uint32_t)nch);
      for (int i = 0; i < nch; ++i)
        tc::bulk_g2s(Wbase + (size_t)i * wb, p.wpk + ((size_t)(i / parts) * 2 + (i % parts)) * wb, wb, &w_res);
    }
    const uint32_t run = (uint32_t)R * 16u;
    int it = 0, wi = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int buf = it % nabuf;
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
      if (!resident) {
        for (int i = 0; i < nch; ++i, ++wi) {
          const int st = wi % nw;
          if (wi >= nw) tc::mbar_wait(&w_empty[st], (uint32_t)(((wi / nw) - 1) & 1));
          tc::mbar_arrive_expect_tx(&w_full[st], wb);
          tc::bulk_g2s(Wbase + (size_t)st * wb, p.wpk + ((size_t)(i / parts) * 2 + (i % parts)) * wb, wb, &w_full[st]);
        }
      }
    }
  } else if (warp < 8) {
    // ---------------------------------------------------------------- MMA + epilogue (warpgroup wg: rows 64 wg ..)
    const int wg = warp >> 2, t = tid & 127;
    float* strip = Strips + wg * 64 * AMP_EPI_LD;
    const uint32_t a0 = tc::smem_u32(Abase), w0 = tc::smem_u32(Wbase);
    const uint32_t lbo_a = (uint32_t)R * 16u, lbo_b = (uint32_t)NC * 16u;
    const uint64_t ks_a = (2u * lbo_a) >> 4, ks_b = (2u * lbo_b) >> 4;
    constexpr int NK = NC / 16;
    const bool do_div = p.out_div != 0.f;
    if (resident) tc::mbar_wait(&w_res, 0);
    int it = 0, wi = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int buf = it % nabuf;
      const int b = tile / tpi, t0 = (tile - b * tpi) * TC_M;
      tc::mbar_wait(&a_full[buf], (uint32_t)((it / nabuf) & 1));
      const uint32_t a_hi = a0 + (uint32_t)buf * a_buf + (uint32_t)wg * 64u * 16u, a_lo = a_hi + a_part;
      float acc[NC / 2];
#pragma unroll
      for (int i = 0; i < NC / 2; ++i) acc[i] = 0.f;
      int i = 0;
      for (int tap = 0; tap < p.K; ++tap) {
        const uint32_t tap_off = (uint32_t)(tap * p.dil) * 16u;
        for (int part = 0; part < parts; ++part, ++i) {
          uint32_t wbase;
          int st = 0;
          if (resident) {
            wbase = w0 + (uint32_t)i * wb;
          } else {
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
            for (int kk = 0; kk < NK; ++kk) tc::Wg<NC, 0>::ss(acc, ad + kk * ks_a, bd + kk * ks_b, 1u);
          }
          tc::wg_commit();
          if (!resident) {
            tc::wg_wait<0>();
            if (t == 0) tc::mbar_arrive(&w_empty[st]);
            ++wi;
          }
        }
      }
      tc::wg_wait<0>();
      tc::wg_hold(acc);
      if (t == 0) tc::mbar_arrive(&a_empty[buf]);

      // epilogue: thread = (row t % 64, 32-column half t / 64) of every 64-column chunk
      const int tt = t0 + wg * 64 + (t & 63);
      const bool live = tt < p.L;
      const long long rowb = (long long)b * p.C * p.L + tt;
#pragma unroll 1
      for (int ch = 0; ch < (NC + 63) / 64; ++ch) {
        tc::named_sync(1 + wg, 128);
        tc::acc_to_smem<NC>(acc, strip, AMP_EPI_LD, 8 * ch, 8 * ch + 8);
        tc::named_sync(1 + wg, 128);
#pragma unroll 1
        for (int sub = 0; sub < 2; ++sub) {
          const int cl = (t >> 6) * 32 + sub * 16, c0 = ch * 64 + cl;
          if (c0 >= NC || !live) continue;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
            const int co = c0 + j;
            if (co < p.C) {
              const long long off = rowb + (long long)co * p.L;
              float a = 0.f;
              if (p.res) a = p.res[off];
              if (p.accum) a += p.y[off];
              float o = strip[(t & 63) * AMP_EPI_LD + cl + j] + __ldg(p.bias + co) + a;
              // a real (uniform) branch: if-converted, the division would run its x/0 slow path per element
              if (do_div) { asm volatile(""); o = o / p.out_div; }
              p.y[off] = o;
            }
          }
        }
      }
    }
  }
}

static AmpPlan amp_plan(int Cp, int K, int dil, int nsplit) {
  const int R = TC_M + (K - 1) * dil;
  const int parts = nsplit == 3 ? 2 : 1;
  const size_t a_buf = (size_t)(Cp / 8) * R * 16 * parts;
  const size_t wb = (size_t)Cp * Cp * 2;
  const size_t nch = (size_t)K * parts;
  const size_t limit = 227 * 1024 - 1024 - AMP_STRIP_BYTES;
  AmpPlan pl;
  pl.nw = 2;
  // resident weights + 2 A buffers when they fit, else a 2-slot weight ring with 2 (or 1) A buffers, else
  // (wide dilated taps: C = 160, k = 11, dilation 5) one A buffer and one weight slot
  if (2 * a_buf + nch * wb + 128 <= limit) { pl.resident = 1; pl.nabuf = 2; pl.smem = 2 * a_buf + nch * wb; }
  else {
    pl.resident = 0;
    pl.nabuf = (2 * a_buf + 2 * wb + 128 <= limit) ? 2 : 1;
    if (pl.nabuf == 1 && a_buf + 2 * wb + 128 > limit) pl.nw = 1;
    pl.smem = pl.nabuf * a_buf + pl.nw * wb;
  }
  pl.smem += AMP_STRIP_BYTES + 128;
  return pl;
}

size_t amp_conv_tc_smem_bytes(int Cp, int K, int dil, int nsplit) { return amp_plan(Cp, K, dil, nsplit).smem; }

int launch_amp_conv_tc(const AmpConvParams& p, cudaStream_t s) {
  if (p.Cp % 16 || p.Cp < 16 || p.Cp > 256 || p.Cp < p.C || (p.nsplit != 1 && p.nsplit != 3)) {
    set_error("amp_conv_tc: bad channel padding / nsplit");
    return SVCB_E_BAD_SHAPE;
  }
  if (p.dil * (p.K - 1) / 2 > P8_PAD || p.Lp != p8_rows_of(p.L) || !p.a_hi || (p.nsplit == 3 && !p.a_lo)) {
    set_error("amp_conv_tc: operand image does not match (halo > 32 rows or wrong Lp)");
    return SVCB_E_BAD_SHAPE;
  }
  const AmpPlan pl = amp_plan(p.Cp, p.K, p.dil, p.nsplit);
  if (pl.smem > 227 * 1024 - 512) { set_error("amp_conv_tc: tile does not fit shared memory"); return SVCB_E_UNSUPPORTED; }
  const int n_sm = device_sm_count();
  if (n_sm <= 0) { set_error("amp_conv_tc: cannot query the SM count"); return SVCB_E_CUDA; }
  const int ntiles = p.B * ((p.L + TC_M - 1) / TC_M);
  const int grid = std::min(ntiles, n_sm);
  const double macs = (double)p.B * p.L * p.C * p.C * p.K;
  char kname[64];
  snprintf(kname, sizeof(kname), "amp_conv_tc_%s_c%dk%d", p.nsplit == 3 ? "bf16x3" : "bf16", p.C, p.K);
  KernelScope ks(kname, s, 2.0 * macs,
                 (double)p.B * p.C * p.L * ((p.nsplit == 3 ? 4.0 : 2.0) + 4.0 * (p.res ? 2 : 1)));
  switch (p.Cp / 16) {
#define SVCB_AMP_NC(nb)                                                                                          \
  case nb: {                                                                                                     \
    static DevSmemCache attr_cache;                                                                              \
    SVCB_CUDA_CHECK(ensure_dyn_smem(amp_conv_tc_kernel<16 * nb>, pl.smem, attr_cache));                          \
    amp_conv_tc_kernel<16 * nb><<<grid, AMP_THREADS, pl.smem, s>>>(p, pl.resident, pl.nabuf, pl.nw);             \
    break;                                                                                                       \
  }
    SVCB_AMP_NC(1) SVCB_AMP_NC(2) SVCB_AMP_NC(3) SVCB_AMP_NC(4) SVCB_AMP_NC(5) SVCB_AMP_NC(6) SVCB_AMP_NC(7) SVCB_AMP_NC(8)
    SVCB_AMP_NC(9) SVCB_AMP_NC(10) SVCB_AMP_NC(11) SVCB_AMP_NC(12) SVCB_AMP_NC(13) SVCB_AMP_NC(14) SVCB_AMP_NC(15) SVCB_AMP_NC(16)
#undef SVCB_AMP_NC
  }
  SVCB_LAUNCH_CHECK("amp_conv_tc");
  return SVCB_OK;
}

}  // namespace svcb

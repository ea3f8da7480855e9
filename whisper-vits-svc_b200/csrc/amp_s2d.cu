// AMP-block links of the narrow generator stages on the tensor cores, in space-to-depth form.
//
// One launch = one `Conv1d(C->C, k, dilation) [+ x] -> SnakeAlias` link of AMPBlock.forward
// (vits_decoder/bigv.py:50-58; SnakeAlias = vits_decoder/alias/act.py:124-128), SURVEY.md §8a rows a9/a10.
//
// Why space-to-depth.  At N = C = 16..32 an MMA spends its time reading the A operand and the tensor
// pipe idles.  Folding r consecutive samples into the channel dimension (C * r = 160: r = 8 for C = 20,
// 16 for C = 10) turns the dilated conv into `ntaps` dense 160 x 160 block-Toeplitz products over rows of
// r samples (pack.py:conv_s2d_matrices): 2-8x more MACs, all of them at the wide N = 160 shape.
//
// Why the Snake lives in the epilogue.  In this layout an accumulator row holds r CONSECUTIVE samples of
// each channel: the epilogue thread that owns accumulator row tau has, per channel, exactly the register-resident
// run of samples the SnakeAlias code of round 1 works on.  It adds bias (+ residual), parks the run in a
// 4 KB shared strip so that neighbouring rows are visible, and computes the anti-aliased Snake of the
// NEXT link straight into that link's bf16 hi/lo operand image — no snake_pack pass, no fp32 round trip:
// 8-12 B of HBM traffic per element and link (was 20-24).
//
// Data layout ("S2D image"): bf16 hi and lo, [B][20 octets][Rp][8]; element (octet o, row, e) is
// snake(x)[b][c][r*(row - 16) + p] with 8*o + e = c*r + p.  Rows outside the sequence are zero (the
// conv's zero padding; the buffers are cleared once per stage and only valid rows are ever written).
// A tile = 128 consecutive rows of every octet = 20 bulk copies per split part, already in the K-major
// SWIZZLE_NONE panel layout of tc.cuh, and a Toeplitz tap is a row-shifted descriptor.
#include <algorithm>
#include <cstdint>
#include <cstdio>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

namespace s2d {
constexpr int N = 160;            // K' = N' = C * r
constexpr int KC = N / 8;         // octets
constexpr int RA = 144;           // rows of the A panel held in shared memory (128 + room for +-8 tap rows)
constexpr int A_OFF = 8;          // A-panel row of the tile's first output row
constexpr int PADR = 16;          // zero rows in front of every (item, octet) of an image
constexpr int TILE = 128;         // accumulator rows per tile
constexpr uint32_t A_PART = KC * RA * 16;       // 46,080 B
constexpr uint32_t W_SLOT = KC * N * 16;        // 51,200 B: one (tap, hi|lo) matrix
constexpr int GROUPS = 3;                       // epilogue column groups (x 4 row quadrants of 32 = 12 warps)
constexpr int STRIP = TILE * 8;                 // floats of one group's strip: 128 rows x (first 4 | last 4 samples) of one channel,
                                                // or 128 rows x 4 samples of two channels (r = 4)
constexpr uint32_t STG_BYTES = 64 + GROUPS * STRIP * 4 + 64 + GROUPS * 128 * 4;  // sample strips (+ guards) + edge buffers
constexpr uint32_t SMEM = 2 * A_PART + 2 * W_SLOT + STG_BYTES;
static_assert(SMEM + 1024 <= 227 * 1024, "A panel + weight ring + strips must fit the 227 KB of one CTA");
constexpr int EPI_WARPS = 4 * GROUPS;
constexpr int THREADS = (EPI_WARPS + 1) * 32;
constexpr int ACC_LD = N + 4;                   // floats per row of the staged accumulator (over the A panel)
static_assert(TILE * ACC_LD * 4 <= 2 * A_PART, "the staged accumulator must fit over the A panel");
}  // namespace s2d

int s2d_halo_rows(int r) { return r >= 8 ? 1 : 2; }                 // SnakeAlias reaches +-5 samples
int s2d_tile_stride(int r) { return s2d::TILE - 2 * s2d_halo_rows(r); }
int s2d_rows(int L, int r) {                                         // Rp of an image
  const int nrows = L / r, S = s2d_tile_stride(r);
  return ((nrows + S - 1) / S) * S + 160;
}
size_t s2d_image_bytes(int B, int L, int r) { return (size_t)B * s2d::KC * s2d_rows(L, r) * 16; }

__device__ __forceinline__ void s2d_store_octet(__nv_bfloat16* hi, __nv_bfloat16* lo, long long row_elem,
                                                const float (&o)[8]) {
  __align__(16) __nv_bfloat162 h2[4], l2[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    h2[k] = __floats2bfloat162_rn(o[2 * k], o[2 * k + 1]);
    const float2 f = __bfloat1622float2(h2[k]);
    l2[k] = __floats2bfloat162_rn(o[2 * k] - f.x, o[2 * k + 1] - f.y);
  }
  *reinterpret_cast<uint4*>(hi + row_elem) = *reinterpret_cast<const uint4*>(h2);
  *reinterpret_cast<uint4*>(lo + row_elem) = *reinterpret_cast<const uint4*>(l2);
}

// ------------------------------------------------------------------------------------------------ pack
// SnakeAlias(x[B,C,L]) -> S2D image (the first activation of every AMP block: its input is the stage
// input, not a convolution result).  One thread = one run of 8 samples = one image row of one octet.
__global__ void __launch_bounds__(256, 4)
snake_pack_s2d_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                      const float* __restrict__ ea, const float* __restrict__ inv_b,
                      const SnakeTapsV tp, int C, int L, int r, int Rp) {
  const int run = blockIdx.x * 256 + threadIdx.x;
  const int c = blockIdx.y, b = blockIdx.z;
  if (run * 8 >= L) return;
  const int opr = r >> 3;                       // octets per row of this channel (0 for r = 4: half an octet)
  const float* xr = x + ((long long)b * C + c) * L;
  const int n0 = run * 8;
  const float a_ = __ldg(ea + c), b_ = __ldg(inv_b + c);
  float out[8], xw[24];
  const bool first = n0 == 0, last = n0 + 8 == L;
  if (n0 - 8 >= 0 && n0 + 16 <= L) {
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      const float4 t4 = __ldg(reinterpret_cast<const float4*>(xr + n0 - 8) + q);
      xw[4 * q] = t4.x; xw[4 * q + 1] = t4.y; xw[4 * q + 2] = t4.z; xw[4 * q + 3] = t4.w;
    }
  } else {   // within 8 samples of a sequence end: replicate padding of x (alias/resample.py:28) = clamped loads
#pragma unroll
    for (int j = 0; j < 24; ++j) xw[j] = __ldg(xr + min(max(n0 - 8 + j, 0), L - 1));
  }
  snake8_packed(xw, tp, a_, 0.5f * b_, out, first, last);   // common.cuh: packed f32x2 FIRs
  if (opr) {
    const int row = run / opr, o = c * opr + run % opr;
    const long long row_elem = ((((long long)b * s2d::KC + o) * Rp) + s2d::PADR + row) * 8;
    s2d_store_octet(hi, lo, row_elem, out);
  } else {   // r = 4: the run covers rows 2*run, 2*run+1; this channel is half (4 elements) of octet c / 2
    __align__(8) __nv_bfloat162 h2[4], l2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      h2[k] = __floats2bfloat162_rn(out[2 * k], out[2 * k + 1]);
      const float2 f = __bfloat1622float2(h2[k]);
      l2[k] = __floats2bfloat162_rn(out[2 * k] - f.x, out[2 * k + 1] - f.y);
    }
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const long long e = ((((long long)b * s2d::KC + (c >> 1)) * Rp) + s2d::PADR + 2 * run + hrow) * 8 + (c & 1) * 4;
      *reinterpret_cast<uint2*>(hi + e) = *reinterpret_cast<const uint2*>(h2 + 2 * hrow);
      *reinterpret_cast<uint2*>(lo + e) = *reinterpret_cast<const uint2*>(l2 + 2 * hrow);
    }
  }
}

int launch_snake_pack_s2d(const float* x, void* hi, void* lo, const float* ea, const float* inv_b, const float* fu,
                          const float* fd, int B, int C, int L, cudaStream_t s, const SnakeTapsV* taps) {
  const int r = C > 0 ? s2d::N / C : 0;
  if (B <= 0 || L <= 0 || C * r != s2d::N || (r != 4 && r != 8 && r != 16) || L % 8 || (reinterpret_cast<uintptr_t>(x) & 15)) {
    set_error("snake_pack_s2d: unsupported shape");
    return SVCB_E_BAD_SHAPE;
  }
  SnakeTapsV tp;
  if (taps) tp = *taps;
  else SVCB_TRY(snake_taps_from_device(fu, fd, &tp));
  char kname[64];
  snprintf(kname, sizeof(kname), "snake_pack_s2d_c%d", C);
  KernelScope ks(kname, s, 0.0, 8.0 * B * C * (double)L, 70.0 * B * C * (double)L);
  dim3 grid((L / 8 + 255) / 256, C, B);
  snake_pack_s2d_kernel<<<grid, 256, 0, s>>>(x, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), ea,
                                             inv_b, tp, C, L, r, s2d_rows(L, r));
  SVCB_LAUNCH_CHECK("snake_pack_s2d");
  return SVCB_OK;
}

// S2D image (hi + lo) -> fp32 [B, C, L]: the unit tests read a link's output image through this.
__global__ void s2d_unpack_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
                                  float* __restrict__ y, int C, int L, int r, int Rp) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over C * L of item blockIdx.y
  if (i >= (long long)C * L) return;
  const int c = (int)(i / L), t = (int)(i % L);
  const int k = c * r + t % r, row = t / r;
  const long long e = ((((long long)blockIdx.y * s2d::KC + k / 8) * Rp) + s2d::PADR + row) * 8 + k % 8;
  y[(long long)blockIdx.y * C * L + i] = __bfloat162float(hi[e]) + __bfloat162float(lo[e]);
}
int launch_s2d_unpack(const void* hi, const void* lo, float* y, int B, int C, int L, cudaStream_t s) {
  const int r = s2d::N / C;
  dim3 grid((unsigned)(((long long)C * L + 255) / 256), B);
  s2d_unpack_kernel<<<grid, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(hi), static_cast<const __nv_bfloat16*>(lo), y, C, L, r,
                                         s2d_rows(L, r));
  SVCB_LAUNCH_CHECK("s2d_unpack");
  return SVCB_OK;
}

// ------------------------------------------------------------------------------------------------ link
// Persistent: every CTA walks tiles (item, 126 useful rows) with a static stride.
//   producer warp  A panel of the tile (40 bulk copies) and the (tap, hi|lo) weight matrices through a
//                  2-slot ring (four bulk copies each)
//   warpgroups 0-1 per tap: A_hi x W_hi, A_lo x W_hi, A_hi x W_lo — 30 wgmma m64n160k16 each for its 64 rows,
//                  register accumulators, then staged as fp32 rows over the (consumed) A panel
//   12 epilogue warps = 3 column groups x 4 row quadrants: group g owns units u = g (mod 3), a unit
//                  being one channel (r >= 8) or a channel pair (r = 4): 6-7 / 6-7 / 3-4 units per group for
//                  C = 20 / 40 / 10 (13 warps leave the MMA warpgroups the registers of 160 accumulator columns)
template <int R>
__global__ void __launch_bounds__(s2d::THREADS, 1)
amp_s2d_link_kernel(const AmpS2dParams p) {
  using namespace s2d;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t a_full, a_empty, w_full[2], w_empty[2];
  __shared__ float s_par[3][40];      // bias | exp(alpha) | 1 / (exp(beta) + 1e-9) of every channel (C <= 40)

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int warp_u = tc::warp_uniform_idx();
  if (tid < p.C) {
    s_par[0][tid] = __ldg(p.bias + tid);
    s_par[1][tid] = p.o_hi ? __ldg(p.ea + tid) : 0.f;
    s_par[2][tid] = p.o_hi ? __ldg(p.ib + tid) : 0.f;
  }
  constexpr int HS = R >= 8 ? 1 : 2;
  constexpr int S = TILE - 2 * HS;
  const int nrows = p.L / R;
  const int tpi = (nrows + S - 1) / S;
  const int ntiles = p.B * tpi;
  uint8_t* Abase = smem;
  uint8_t* Wbase = smem + 2 * A_PART;
  float* Stg = reinterpret_cast<float*>(smem + 2 * A_PART + 2 * W_SLOT);
  float* Acc = reinterpret_cast<float*>(smem);   // staged accumulator [TILE][ACC_LD], over the A panel

  if (tid == 0) {
    tc::mbar_init(&a_full, 1); tc::mbar_init(&a_empty, 1);
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&w_full[i], 1); tc::mbar_init(&w_empty[i], 2); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp_u == EPI_WARPS) {
    // ------------------------------------------------------------------------------------ producer
    if (tc::elect_one()) {
      const uint8_t* img[2] = {reinterpret_cast<const uint8_t*>(p.a_hi), reinterpret_cast<const uint8_t*>(p.a_lo)};
      int it = 0, wi = 0;
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int b = tile / tpi, t = tile - b * tpi;
        const long long row0 = (long long)t * S - HS - A_OFF + PADR;     // image row of A-panel row 0 (>= 6)
        if (it >= 1) tc::mbar_wait_parked(&a_empty, (uint32_t)((it - 1) & 1));
        tc::mbar_arrive_expect_tx(&a_full, 2 * A_PART);
        for (int part = 0; part < 2; ++part)
          for (int kc = 0; kc < KC; ++kc)
            tc::bulk_g2s(Abase + (size_t)part * A_PART + (size_t)kc * RA * 16,
                         img[part] + ((((long long)b * KC + kc) * p.Rp) + row0) * 16, RA * 16, &a_full);
        for (int c = 0; c < 2 * p.ntaps; ++c, ++wi) {
          const int st = wi & 1;
          if (wi >= 2) tc::mbar_wait_parked(&w_empty[st], (uint32_t)(((wi >> 1) - 1) & 1));
          tc::mbar_arrive_expect_tx(&w_full[st], W_SLOT);
#pragma unroll
          for (int piece = 0; piece < 4; ++piece)    // four requests in flight per matrix instead of one long one
            tc::bulk_g2s(Wbase + (size_t)st * W_SLOT + piece * (W_SLOT / 4), p.wpk + (size_t)c * W_SLOT + piece * (W_SLOT / 4),
                         W_SLOT / 4, &w_full[st]);
        }
      }
    }
    return;
  }
  {
    // ------------------------------------------------------------------------------------ epilogue
    const int q = warp & 3, g = warp >> 2;
    const int row = q * 32 + lane;
    const int wg = warp >> 2, tw = tid & 127;
    constexpr uint32_t LBO_A = RA * 16, LBO_B = N * 16;
    constexpr uint64_t KSA = (2 * LBO_A) >> 4, KSB = (2 * LBO_B) >> 4;      // descriptor step per K = 16
    const uint32_t a_h0 = tc::smem_u32(Abase) + (uint32_t)wg * 64u * 16u, a_l0 = a_h0 + A_PART, w_s0 = tc::smem_u32(Wbase);
    const float* arow = Acc + row * ACC_LD;
    int wi = 0;
    constexpr int CU = R >= 8 ? R : 8;            // accumulator columns per unit: whole channels, >= one image octet
    constexpr int NCH = CU / R;                   // channels per unit (2 for R = 4)
    const int NU = p.C / NCH;
    float* stg_g = Stg + 16 + (size_t)g * STRIP;                     // this group's strip (see the staging comment below)
    float* edge_g = Stg + 16 + GROUPS * STRIP + 16 + g * 128;        // [4 warps][<= 2 channels][lane 0: 5 | lane 31: 5] Snake values
    __nv_bfloat16* o_hi = static_cast<__nv_bfloat16*>(p.o_hi);
    __nv_bfloat16* o_lo = static_cast<__nv_bfloat16*>(p.o_lo);
    const bool do_div = p.out_div != 0.f;
    int it = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
      const int b = tile / tpi, t = tile - b * tpi;
      const int tau0 = t * S - HS;
      const int tau = tau0 + row;
      const bool valid = tau >= 0 && tau < nrows;
      const bool useful = valid && row >= HS && row < TILE - HS;
      // residual rows are independent of the accumulator: the first unit's are requested before the wait,
      // every later unit's one unit ahead (their latency was 19 % of all stall samples)
      const bool has_res = p.res != nullptr && valid;
      const long long xrow = (long long)b * p.C * p.L + (long long)tau * R;
      float4 rcur[CU / 4], rnext[CU / 4];
      auto load_res = [&](int u, float4 (&dst)[CU / 4]) {
        if (has_res) {
#pragma unroll
          for (int j = 0; j < CU / 4; ++j)
            dst[j] = __ldg(reinterpret_cast<const float4*>(p.res + xrow + (long long)(u * NCH + j / (R / 4)) * p.L) + j % (R / 4));
        }
      };
      load_res(g, rcur);
      if (wg < 2) {
        // ---------------------------------------------------------------- MMAs of this warpgroup's 64 rows
        tc::mbar_wait_parked(&a_full, (uint32_t)(it & 1));
        float acc[N / 2];
#pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
        for (int tap = 0; tap < p.ntaps; ++tap) {
          const uint32_t arow_off = (uint32_t)(A_OFF - p.mlo + tap) * 16u;   // row shift
          const uint64_t ah = tc::smem_desc(a_h0 + arow_off, LBO_A), al = tc::smem_desc(a_l0 + arow_off, LBO_A);
          for (int part = 0; part < 2; ++part, ++wi) {   // W_hi: A_hi x W_hi, A_lo x W_hi;  W_lo: A_hi x W_lo
            const int st = wi & 1;
            tc::mbar_wait_parked(&w_full[st], (uint32_t)((wi >> 1) & 1));
            const uint64_t bw = tc::smem_desc(w_s0 + (uint32_t)st * W_SLOT, LBO_B);
            tc::wg_fence();
#pragma unroll
            for (int kk = 0; kk < N / 16; ++kk) tc::Wg<N, 0>::ss(acc, ah + kk * KSA, bw + kk * KSB, 1u);
            if (part == 0) {
#pragma unroll
              for (int kk = 0; kk < N / 16; ++kk) tc::Wg<N, 0>::ss(acc, al + kk * KSA, bw + kk * KSB, 1u);
            }
            tc::wg_commit();
            tc::wg_wait<0>();
            if (tw == 0) tc::mbar_arrive(&w_empty[st]);
          }
        }
        tc::wg_hold(acc);
        tc::named_sync(6, 256);                   // both warpgroups' MMAs are done: the A panel is free
        tc::acc_to_smem<N>(acc, Acc + wg * 64 * ACC_LD, ACC_LD, 0, N / 8);
      }
      tc::named_sync(7, EPI_WARPS * 32);          // accumulator rows staged
      auto ld_acc = [&](int col, uint32_t* dst, int n) {
        for (int k = 0; k < n; k += 4) {
          const float4 q4 = *reinterpret_cast<const float4*>(arow + col + k);
          dst[k] = __float_as_uint(q4.x); dst[k + 1] = __float_as_uint(q4.y); dst[k + 2] = __float_as_uint(q4.z); dst[k + 3] = __float_as_uint(q4.w);
        }
      };
      uint32_t wpre[8];
      if constexpr (CU == 8) ld_acc(g * CU, wpre, 8);
      for (int u = g; u < NU; u += GROUPS) {                     // unit = one channel (R >= 8) or a channel pair (R = 4)
        if (u + GROUPS < NU) load_res(u + GROUPS, rnext);
        const int c0 = u * NCH;
        float v[CU];
        if constexpr (CU == 8) {
#pragma unroll
          for (int k = 0; k < NCH; ++k) {
            const float bias = s_par[0][c0 + k];
#pragma unroll
            for (int j = 0; j < R; ++j) v[k * R + j] = __uint_as_float(wpre[k * R + j]) + bias;
          }
          if (u + GROUPS < NU) ld_acc((u + GROUPS) * CU, wpre, 8);
        } else {
          uint32_t w[CU];
          ld_acc(u * CU, w, CU);
          const float bias = s_par[0][c0];
#pragma unroll
          for (int j = 0; j < R; ++j) v[j] = __uint_as_float(w[j]) + bias;
        }
        if (has_res) {
#pragma unroll
          for (int j = 0; j < CU / 4; ++j) {
            v[4 * j] += rcur[j].x; v[4 * j + 1] += rcur[j].y; v[4 * j + 2] += rcur[j].z; v[4 * j + 3] += rcur[j].w;
          }
        }
#pragma unroll
        for (int j = 0; j < CU / 4; ++j) rcur[j] = rnext[j];
        if (p.y && useful) {
#pragma unroll
          for (int j = 0; j < CU / 4; ++j) {
            float4* yp = reinterpret_cast<float4*>(p.y + xrow + (long long)(c0 + j / (R / 4)) * p.L) + j % (R / 4);
            float4 o4 = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
            if (p.accum) { const float4 y4 = *yp; o4.x += y4.x; o4.y += y4.y; o4.z += y4.z; o4.w += y4.w; }
            // a real (uniform) branch: if-converted, the division would run its x/0 slow path per element
            if (do_div) { asm volatile(""); o4.x = o4.x / p.out_div; o4.y = o4.y / p.out_div; o4.z = o4.z / p.out_div; o4.w = o4.w / p.out_div; }
            *yp = o4;
          }
        }
        if (p.o_hi) {
          // SnakeAlias of the result, written as the next link's operand image.  A row owns R consecutive
          // samples of a channel: it up-samples + applies Snake to ITS 2R values only (the 4 + 4 samples it
          // needs from the neighbouring rows come from the shared strip), then the 5 + 5 Snake values of
          // the neighbouring rows that its decimation filter reaches arrive by warp shuffle (lanes 0 / 31:
          // through a small edge buffer), so nothing is computed twice: 30 FMA + 2 sin per sample instead
          // of 46 + 3.5 for the register-run form with recomputed halos.  Sequence ends: the reference's
          // replicate padding of x (alias/resample.py:28) and of the 2x signal (alias/filter.py:90-91)
          // are two selects each — no scalar path.
          // strip layout per channel: [row][first 4 samples | last 4 samples] (for R = 4 both are the row's
          // 4 samples) — all a neighbouring row ever reads
          constexpr int RS = R == 4 ? 4 : 8;                         // strip floats per row and channel
#pragma unroll
          for (int k = 0; k < NCH; ++k) {
            float* strip = stg_g + k * (TILE * RS);
            *reinterpret_cast<float4*>(strip + row * RS) = make_float4(v[k * R], v[k * R + 1], v[k * R + 2], v[k * R + 3]);
            if constexpr (R > 4)
              *reinterpret_cast<float4*>(strip + row * RS + 4) =
                  make_float4(v[k * R + R - 4], v[k * R + R - 3], v[k * R + R - 2], v[k * R + R - 1]);
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
          // 2x-rate Snake values as (even, odd) pairs V[a + 3], a = position relative to the row's first sample:
          // own a = 0 .. R-1; the previous row's last five values are V[0].y, V[1], V[2], the next row's first five
          // V[R+3], V[R+4], V[R+5].x.  All FIR / range-reduction arithmetic runs as f32x2 pair operations (f2_fma /
          // FMUL2 / FADD2: one issue slot for the even and the odd phase), taps as uniform-register pairs.
          float2 V[NCH][R + 6];
#pragma unroll
          for (int k = 0; k < NCH; ++k) {
            const float a_ = s_par[1][c0 + k], hb_ = 0.5f * s_par[2][c0 + k];
            const float* strip = stg_g + k * (TILE * RS);
            float xw[R + 8];                                         // samples -4 .. R+3 relative to the row's first
            float4 l4 = *reinterpret_cast<const float4*>(strip + row * RS - 4);    // previous row's last four (row 0 / 127
            float4 r4 = *reinterpret_cast<const float4*>(strip + row * RS + RS);   //  read outside the strip: halo rows, unused)
            if (tau == 0) l4 = make_float4(v[k * R], v[k * R], v[k * R], v[k * R]);
            if (tau == nrows - 1) r4 = make_float4(v[k * R + R - 1], v[k * R + R - 1], v[k * R + R - 1], v[k * R + R - 1]);
            xw[0] = l4.x; xw[1] = l4.y; xw[2] = l4.z; xw[3] = l4.w;
#pragma unroll
            for (int j = 0; j < R; ++j) xw[4 + j] = v[k * R + j];
            xw[R + 4] = r4.x; xw[R + 5] = r4.y; xw[R + 6] = r4.z; xw[R + 7] = r4.w;
            // consecutive-sample pairs in both alignments, each held in its own (aligned) register pair so that
            // every FIR step is one f2_fma: XE[m] = (x[2m], x[2m+1]), XO[m] = (x[2m+1], x[2m+2])  (x = xw)
            float2 XE[(R + 8) / 2], XO[(R + 6) / 2];
#pragma unroll
            for (int m2 = 0; m2 < (R + 8) / 2; ++m2) XE[m2] = make_float2(xw[2 * m2], xw[2 * m2 + 1]);
#pragma unroll
            for (int m2 = 0; m2 < (R + 6) / 2; ++m2) XO[m2] = make_float2(xw[2 * m2 + 1], xw[2 * m2 + 2]);
#pragma unroll
            for (int a = 0; a < R; ++a) {
              // (u_even, u_odd)[a] = sum_i (x[a+1+i], x[a+2+i]) * (f[11-2i], f[10-2i])
              float2 U;
#pragma unroll
              for (int i = 0; i < 6; ++i) {
                const int j = a + 1 + i;
                const float2 pr = (j & 1) ? XO[(j - 1) / 2] : XE[j / 2];
                U = i == 0 ? f2_mul(pr, p.taps.fup[0]) : f2_fma(pr, p.taps.fup[i], U);
              }
              // u + sin^2(a u) / (e^beta + 1e-9) = (u + b/2) - (b/2) cos(2 a u); a u = k pi + r, |r| <= pi/2
              const float2 t = f2_mul(U, make_float2(a_, a_));
              const float2 kq = f2_add(f2_fma(t, make_float2(0.3183098861837907f, 0.3183098861837907f),
                                                      make_float2(12582912.f, 12582912.f)),
                                           make_float2(-12582912.f, -12582912.f));
              float2 rr = f2_fma(kq, make_float2(-3.140625f, -3.140625f), t);
              rr = f2_fma(kq, make_float2(-9.676535897932e-4f, -9.676535897932e-4f), rr);
              rr = f2_add(rr, rr);
              const float2 cs = make_float2(__cosf(rr.x), __cosf(rr.y));
              V[k][a + 3] = f2_fma(make_float2(-hb_, -hb_), cs, f2_add(U, make_float2(hb_, hb_)));
            }
            float* edge = edge_g + (q * NCH + k) * 16;
            if (lane == 0) {
              edge[0] = V[k][3].x; edge[1] = V[k][3].y; edge[2] = V[k][4].x; edge[3] = V[k][4].y; edge[4] = V[k][5].x;
            }
            if (lane == 31) {
              edge[8] = V[k][R].y; edge[9] = V[k][R + 1].x; edge[10] = V[k][R + 1].y; edge[11] = V[k][R + 2].x; edge[12] = V[k][R + 2].y;
            }
          }
          asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
          float out[CU];
#pragma unroll
          for (int k = 0; k < NCH; ++k) {
            float pv[5], nx[5];                                     // previous row's last five, next row's first five
            pv[0] = __shfl_up_sync(0xffffffffu, V[k][R].y, 1);     pv[1] = __shfl_up_sync(0xffffffffu, V[k][R + 1].x, 1);
            pv[2] = __shfl_up_sync(0xffffffffu, V[k][R + 1].y, 1); pv[3] = __shfl_up_sync(0xffffffffu, V[k][R + 2].x, 1);
            pv[4] = __shfl_up_sync(0xffffffffu, V[k][R + 2].y, 1);
            nx[0] = __shfl_down_sync(0xffffffffu, V[k][3].x, 1);   nx[1] = __shfl_down_sync(0xffffffffu, V[k][3].y, 1);
            nx[2] = __shfl_down_sync(0xffffffffu, V[k][4].x, 1);   nx[3] = __shfl_down_sync(0xffffffffu, V[k][4].y, 1);
            nx[4] = __shfl_down_sync(0xffffffffu, V[k][5].x, 1);
            if (lane == 0 && q > 0) {
#pragma unroll
              for (int i = 0; i < 5; ++i) pv[i] = edge_g[((q - 1) * NCH + k) * 16 + 8 + i];
            }
            if (lane == 31 && q < 3) {
#pragma unroll
              for (int i = 0; i < 5; ++i) nx[i] = edge_g[((q + 1) * NCH + k) * 16 + i];
            }
            if (tau == 0) {               // the 2x signal is replicate-padded before decimation (alias/filter.py:90-91)
#pragma unroll
              for (int i = 0; i < 5; ++i) pv[i] = V[k][3].x;
            }
            if (tau == nrows - 1) {
#pragma unroll
              for (int i = 0; i < 5; ++i) nx[i] = V[k][R + 2].y;
            }
            V[k][0] = make_float2(0.f, pv[0]); V[k][1] = make_float2(pv[1], pv[2]); V[k][2] = make_float2(pv[3], pv[4]);
            V[k][R + 3] = make_float2(nx[0], nx[1]); V[k][R + 4] = make_float2(nx[2], nx[3]); V[k][R + 5] = make_float2(nx[4], 0.f);
#pragma unroll
            for (int n = 0; n < R; ++n) {
              // out[n] = v[2n-5] f0 + sum_i (v[2n-4+2i], v[2n-3+2i]) . (f[2i+1], f[2i+2]) + v[2n+6] f11
              float2 acc2 = f2_mul(V[k][n + 1], p.taps.fdp[0]);
#pragma unroll
              for (int i = 1; i < 5; ++i) acc2 = f2_fma(V[k][n + 1 + i], p.taps.fdp[i], acc2);
              float o1 = acc2.x + acc2.y;
              o1 = fmaf(V[k][n].y, p.taps.fd0, o1);
              out[k * R + n] = fmaf(V[k][n + 6].x, p.taps.fd11, o1);
            }
          }
          if (useful) {
#pragma unroll
            for (int h = 0; h < CU / 8; ++h) {                       // 8 consecutive K' indices = one image octet row
              float oh[8];
#pragma unroll
              for (int i = 0; i < 8; ++i) oh[i] = out[8 * h + i];
              const int oc = u * (CU / 8) + h;
              const long long row_elem = ((((long long)b * KC + oc) * p.Rp) + PADR + tau) * 8;
              s2d_store_octet(o_hi, o_lo, row_elem, oh);
            }
          }
        }
      }
      tc::fence_proxy_async_smem();               // staged rows (generic proxy) -> the next tile's bulk copies
      tc::named_sync(7, EPI_WARPS * 32);
      if (tid == 0) tc::mbar_arrive(&a_empty);
    }
  }
}

int launch_amp_s2d_link(const AmpS2dParams& p, cudaStream_t s) {
  const int r = p.C > 0 ? s2d::N / p.C : 0;
  if (p.B <= 0 || p.L <= 0 || p.C * r != s2d::N || (r != 4 && r != 8 && r != 16) || p.L % r) {
    set_error("amp_s2d_link: unsupported shape (need C * r = 160 with r in {4, 8, 16} and L % r == 0)");
    return SVCB_E_BAD_SHAPE;
  }
  if (p.ntaps < 1 || p.mlo < 0 || p.mlo > s2d::A_OFF || p.ntaps - 1 - p.mlo > s2d::RA - s2d::TILE - s2d::A_OFF ||
      p.Rp != s2d_rows(p.L, r) || !p.a_hi || !p.a_lo || !p.wpk || !p.bias || (p.o_hi && (!p.o_lo || !p.ea || !p.ib || !p.fu || !p.fd))) {
    set_error("amp_s2d_link: tap range exceeds the A panel, wrong image rows or missing operand");
    return SVCB_E_BAD_SHAPE;
  }
  static DevSmemCache c4, c8, c16;
  const int n_sm = device_sm_count();
  if (n_sm <= 0) { set_error("amp_s2d_link: cannot query the SM count"); return SVCB_E_CUDA; }
  const int S = s2d_tile_stride(r);
  const int ntiles = p.B * ((p.L / r + S - 1) / S);
  const int grid = std::min(ntiles, n_sm);
  char kname[64];
  snprintf(kname, sizeof(kname), "amp_s2d_link_c%dk%dr%d", p.C, p.K, r);
  const double el = (double)p.B * p.C * p.L;
  KernelScope ks(kname, s, 2.0 * p.C * p.K * el, el * (4.0 + (p.o_hi ? 4.0 : 0.0) + (p.res ? 4.0 : 0.0) + (p.y ? (p.accum ? 8.0 : 4.0) : 0.0)),
                 p.o_hi ? 70.0 * el : 0.0);
  if (r == 4) {
    SVCB_CUDA_CHECK(ensure_dyn_smem(amp_s2d_link_kernel<4>, s2d::SMEM, c4));
    amp_s2d_link_kernel<4><<<grid, s2d::THREADS, s2d::SMEM, s>>>(p);
  } else if (r == 8) {
    SVCB_CUDA_CHECK(ensure_dyn_smem(amp_s2d_link_kernel<8>, s2d::SMEM, c8));
    amp_s2d_link_kernel<8><<<grid, s2d::THREADS, s2d::SMEM, s>>>(p);
  } else {
    SVCB_CUDA_CHECK(ensure_dyn_smem(amp_s2d_link_kernel<16>, s2d::SMEM, c16));
    amp_s2d_link_kernel<16><<<grid, s2d::THREADS, s2d::SMEM, s>>>(p);
  }
  SVCB_LAUNCH_CHECK("amp_s2d_link");
  return SVCB_OK;
}

}  // namespace svcb

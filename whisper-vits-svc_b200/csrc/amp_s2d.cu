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
// run of samples the SnakeAlias code of round 1 works on.  It adds bias (+ residual), writes the run back over
// its staged accumulator row so that neighbouring rows see it, and computes the anti-aliased Snake of the
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
constexpr uint32_t W_MAT = KC * N * 16;         // 51,200 B: one (tap, hi|lo) matrix
constexpr int KH = 10;                          // octets (K / 8) of one weight chunk: half a matrix
constexpr int WCH = KC / KH;                    // chunks per matrix
constexpr uint32_t W_SLOT = KH * N * 16;        // 25,600 B: one ring slot = one chunk
constexpr int NSLOT = 2;                        // weight ring depth
constexpr int GROUPS = 3;                       // epilogue column groups (x 4 row quadrants of 32 = 12 warps)
constexpr int ACC_LD = N + 4;                   // floats per row of the staged accumulator
constexpr uint32_t ACC_BYTES = TILE * ACC_LD * 4;           // 83,968 B
constexpr uint32_t EDGE_BYTES = GROUPS * 128 * 4;           // Snake values at the warps' row edges
constexpr uint32_t SMEM = 2 * A_PART + ACC_BYTES + NSLOT * W_SLOT + EDGE_BYTES;
static_assert(SMEM + 1024 <= 227 * 1024, "A panel + staged accumulator + weight ring must fit the 227 KB of one CTA");
static_assert(KC % KH == 0 && KH % 2 == 0, "a weight chunk is a whole number of K steps");
constexpr int EPI_WARPS = 4 * GROUPS;
constexpr int THREADS = (8 + EPI_WARPS) * 32;   // producer warpgroup, MMA warpgroup, 3 epilogue warpgroups
// 640 threads launch with 96 registers each (5 warps per SM sub-partition); the producers give theirs to the MMA
// warpgroup, which holds the 128 x 160 fp32 accumulator of a whole tile
constexpr int PRODUCER_REGS = 24, MMA_REGS = 192, EPI_REGS = 88;
static_assert(128 * PRODUCER_REGS + 128 * MMA_REGS + 32 * EPI_WARPS * EPI_REGS <= THREADS * 96, "register budget");
constexpr uint32_t LBO_A = RA * 16, LBO_B = N * 16;
constexpr uint64_t KSA = (2 * LBO_A) >> 4;      // A descriptor step per K = 16
constexpr int GCOLS = N / 4;                    // output columns of one phase group
}  // namespace s2d

int s2d_halo_rows(int r) { return r >= 8 ? 1 : 2; }                 // SnakeAlias reaches +-5 samples
int s2d_tile_stride(int r) { return s2d::TILE - 2 * s2d_halo_rows(r); }
int s2d_rows(int L, int r) {                                         // Rp of an image
  const int nrows = L / r, S = s2d_tile_stride(r);
  return ((nrows + S - 1) / S) * S + 160;
}
size_t s2d_image_bytes(int B, int L, int r) { return (size_t)B * s2d::KC * s2d_rows(L, r) * 16; }

// Output columns of the weights and the accumulator come in four slots of 40, n = 40 s + g c + j: slot s holds
// the g = r / 4 phases p = g q + j of every channel c of phase group q = {0, 1, 3, 2}[s] (pack.py:
// s2d_column_order).  Row tap m reaches the phases [max(0, r m - P), min(r - 1, r m + r - 1 + P)] only, so the
// matrix of an edge tap is zero outside the groups {0}, {0, 1} (m < 0) or {3}, {3, 2} (m > 0), that is outside
// columns [0, 40), [0, 80), [80, 120) or [80, 160).  Per tap 3 bits: code 1-4 = those ranges, 0 = all columns.
bool s2d_tap_plan(int k, int dil, int r, int& mlo, int& ntaps, uint64_t& tap_cols) {
  const int P = dil * (k - 1) / 2, g = r / 4;
  mlo = (P + r - 1) / r;
  ntaps = mlo + (r - 1 + P) / r + 1;
  tap_cols = 0;
  if (g < 1 || ntaps > 21) return false;
  for (int t = 0; t < ntaps; ++t) {
    const int m = t - mlo;
    const int q0 = std::max(0, r * m - P) / g, q1 = std::min(r - 1, r * m + r - 1 + P) / g;
    const int code = q0 == 0 && q1 <= 1 ? 1 + q1 : q1 == 3 && q0 >= 2 ? 3 + (3 - q0) : 0;
    tap_cols |= (uint64_t)code << (3 * t);
  }
  return true;
}

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
                      const SnakeTapsV tp, int C, int L, int r, int Rp, const int* __restrict__ lens, int lscale) {
  const int run = blockIdx.x * 256 + threadIdx.x;
  const int c = blockIdx.y, b = blockIdx.z;
  const int Lb = lens ? __ldg(lens + b) * lscale : L;   // a ragged item's end: its later rows stay zero
  if (run * 8 >= Lb) return;
  const int opr = r >> 3;                       // octets per row of this channel (0 for r = 4: half an octet)
  const float* xr = x + ((long long)b * C + c) * L;
  const int n0 = run * 8;
  const float a_ = __ldg(ea + c), b_ = __ldg(inv_b + c);
  float out[8], xw[24];
  const bool first = n0 == 0, last = n0 + 8 == Lb;
  if (n0 - 8 >= 0 && n0 + 16 <= Lb) {
#pragma unroll
    for (int q = 0; q < 6; ++q) {
      const float4 t4 = __ldg(reinterpret_cast<const float4*>(xr + n0 - 8) + q);
      xw[4 * q] = t4.x; xw[4 * q + 1] = t4.y; xw[4 * q + 2] = t4.z; xw[4 * q + 3] = t4.w;
    }
  } else {   // within 8 samples of a sequence end: replicate padding of x (alias/resample.py:28) = clamped loads
#pragma unroll
    for (int j = 0; j < 24; ++j) xw[j] = __ldg(xr + min(max(n0 - 8 + j, 0), Lb - 1));
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
                          const float* fd, int B, int C, int L, cudaStream_t s, const SnakeTapsV* taps, const int* lens,
                          int lscale) {
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
                                             inv_b, tp, C, L, r, s2d_rows(L, r), lens, lscale);
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
// One weight chunk (KH octets of K of one (tap, hi|lo) matrix) over the output columns [N0, N0 + W) it reaches: the
// accumulator registers of those columns (4j .. 4j+3 hold columns 8j .. 8j+7) and the B panel from its row N0 (16 B =
// one descriptor unit).  The skipped products are exact zeros.  ah / al point at the chunk's first K step.
template <int W, int N0, bool ALO>
__device__ __forceinline__ void s2d_mma(float (&acc)[s2d::N / 2], uint64_t ah, uint64_t al, uint64_t bw) {
  using namespace s2d;
  constexpr uint64_t KS = (2 * LBO_B) >> 4;
  float(&d)[W / 2] = *reinterpret_cast<float(*)[W / 2]>(acc + N0 / 2);
#pragma unroll
  for (int kk = 0; kk < KH / 2; ++kk) tc::Wg<W, 0>::ss(d, ah + kk * KSA, bw + N0 + kk * KS, 1u);
  if constexpr (ALO) {
#pragma unroll
    for (int kk = 0; kk < KH / 2; ++kk) tc::Wg<W, 0>::ss(d, al + kk * KSA, bw + N0 + kk * KS, 1u);
  }
}
// The accumulator is two independent 80-column halves, lower (slots 0, 1) and upper (slots 2, 3), each of which
// a wgmma only ever addresses from its first register: ptxas serialises every wgmma of the kernel once one of
// them starts inside another's register range.  A full tap is an m64n80 pair, never one m64n160: the 80
// accumulator registers of an m64n160 do not fit the 96 registers every thread launches with, and ptxas checks
// each instruction against that count.  `code` (s2d_tap_plan) is warp-uniform.
template <bool ALO>
__device__ __forceinline__ void s2d_mma_tap(float (&acc)[s2d::N / 2], uint64_t ah, uint64_t al, uint64_t bw, int code) {
  switch (code) {
    case 1: s2d_mma<40, 0, ALO>(acc, ah, al, bw); break;
    case 2: s2d_mma<80, 0, ALO>(acc, ah, al, bw); break;
    case 3: s2d_mma<40, 80, ALO>(acc, ah, al, bw); break;
    case 4: s2d_mma<80, 80, ALO>(acc, ah, al, bw); break;
    default: s2d_mma<80, 0, ALO>(acc, ah, al, bw); s2d_mma<80, 80, ALO>(acc, ah, al, bw); break;
  }
}

// Accumulator fragment (64 rows x 160 columns in slot order, see s2d_tap_plan; phase p = g q + j, g = R / 4) ->
// rows buf[row * ACC_LD + c * R + p] in the channel-major order the epilogue reads.  A thread holds the columns
// 8 i + 2 (l & 3) + {0, 1}, i = 5 s + i5, of rows rr and rr + 8: for R = 4 and 8 these are all R phases of its
// channels (float4 runs), for R = 16 pairs of phases (float2).  With the row stride of 164 floats (+4 banks per
// row) every store is free of bank conflicts.
template <int R>
__device__ __forceinline__ void s2d_stage_acc(const float (&d)[s2d::N / 2], float* buf) {
  using namespace s2d;
  const int t = threadIdx.x & 127, lq = t & 3;
  const int rr = 16 * (t >> 5) + ((t & 31) >> 2);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float* row = buf + (rr + 8 * h) * ACC_LD;
#pragma unroll
    for (int i5 = 0; i5 < 5; ++i5) {
      auto a = [&](int q, int e) { return d[4 * (5 * (q < 2 ? q : 5 - q) + i5) + 2 * h + e]; };   // group q, slot s
      if constexpr (R == 4) {          // channel 8 i5 + 2 lq + e, phase q
#pragma unroll
        for (int e = 0; e < 2; ++e)
          *reinterpret_cast<float4*>(row + 4 * (8 * i5 + 2 * lq + e)) = make_float4(a(0, e), a(1, e), a(2, e), a(3, e));
      } else if constexpr (R == 8) {   // channel 4 i5 + lq, phase 2 q + e
#pragma unroll
        for (int hh = 0; hh < 2; ++hh)
          *reinterpret_cast<float4*>(row + 8 * (4 * i5 + lq) + 4 * hh) =
              make_float4(a(2 * hh, 0), a(2 * hh, 1), a(2 * hh + 1, 0), a(2 * hh + 1, 1));
      } else {                         // channel 2 i5 + lq / 2, phase 4 q + 2 (lq & 1) + e
#pragma unroll
        for (int q = 0; q < 4; ++q)
          *reinterpret_cast<float2*>(row + 16 * (2 * i5 + (lq >> 1)) + 4 * q + 2 * (lq & 1)) = make_float2(a(q, 0), a(q, 1));
      }
    }
  }
}

// Persistent: every CTA walks tiles (item, 126 useful rows) with a static stride.  Tile i's epilogue runs while
// tile i+1's MMAs run: the accumulator is staged into a buffer of its own, not over the weight ring.
//   producer warpgroup  (24 registers) warp 0: the A panel of each tile in two K halves (20 bulk copies each), each
//                  requested as soon as the previous tile's MMAs of that half retire (a_empty[h]); warp 1: the weight
//                  chunks, half a (tap, hi|lo) matrix each, through a 2-slot ring (an edge tap's chunk: 10 runs of
//                  its reached columns)
//   MMA warpgroup  (192 registers) the whole 128-row tile as two m64 accumulators, in the order K half, tap,
//                  hi | lo: per chunk A_hi x W_hi and A_lo x W_hi (W_hi), or A_hi x W_lo (W_lo), over the chunk's 5 K
//                  steps, as m64n80 pairs (one per accumulator half) or m64n40 / m64n80 over the reached columns of
//                  an edge tap; one commit group per chunk.  The first K half of the panel is released halfway
//                  through the tile, so the next tile's copy of it runs under the second half's MMAs.  When the
//                  tile's last group retires the MMA warpgroup waits for the previous tile's epilogue to free the
//                  staging buffer (stg_free), stages the fp32 rows, arrives stg_full and goes on to the next tile
//   3 epilogue warpgroups = 3 column groups x 4 row quadrants (88 registers): group g owns units u = g (mod 3), a
//                  unit being one channel (r >= 8) or a channel pair (r = 4): 6-7 / 6-7 / 3-4 units per group for
//                  C = 20 / 40 / 10.  The staged rows double as the Snake's sample strips: a thread writes
//                  v = acc + bias (+ res) back over its row's unit, and the neighbouring rows read their 4 + 4
//                  samples from there
// RAG: a ragged batch (p.lens): a separate instantiation, so that the dense one keeps its registers
template <int R, bool RAG>
__global__ void __launch_bounds__(s2d::THREADS, 1)
amp_s2d_link_kernel(const AmpS2dParams p) {
  using namespace s2d;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t a_full[WCH], a_empty[WCH], w_full[NSLOT], w_empty[NSLOT], stg_full, stg_free;
  __shared__ float s_par[3][40];      // bias | exp(alpha) | 1 / (exp(beta) + 1e-9) of every channel (C <= 40)

  const int tid = threadIdx.x, lane = tid & 31;
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
  // the tile count p.B * tpi is computed in each role's loop: held across the role branches it was spilled
  uint8_t* Abase = smem;
  float* Acc = reinterpret_cast<float*>(smem + 2 * A_PART);           // staged accumulator [TILE][ACC_LD]
  uint8_t* Wbase = smem + 2 * A_PART + ACC_BYTES;
  float* Edge = reinterpret_cast<float*>(Wbase + NSLOT * W_SLOT);

  if (tid == 0) {
    for (int i = 0; i < WCH; ++i) { tc::mbar_init(&a_full[i], 1); tc::mbar_init(&a_empty[i], 1); }
    for (int i = 0; i < NSLOT; ++i) { tc::mbar_init(&w_full[i], 1); tc::mbar_init(&w_empty[i], 1); }
    tc::mbar_init(&stg_full, 128); tc::mbar_init(&stg_free, EPI_WARPS);
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp_u < 4) {
    // ------------------------------------------------------------------------------------ producers
    tc::setmaxnreg_dec<PRODUCER_REGS>();
    if (warp_u == 0 && tc::elect_one()) {
      const uint8_t* img[2] = {reinterpret_cast<const uint8_t*>(p.a_hi), reinterpret_cast<const uint8_t*>(p.a_lo)};
      int it = 0;
      for (int tile = blockIdx.x; tile < p.B * tpi; tile += gridDim.x, ++it) {
        const int b = tile / tpi, t = tile - b * tpi;
        const long long row0 = (long long)t * S - HS - A_OFF + PADR;     // image row of A-panel row 0 (>= 6)
        for (int h = 0; h < WCH; ++h) {   // K half h (hi and lo): free once the MMAs of the previous tile's half h retire
          if (it >= 1) tc::mbar_wait_parked(&a_empty[h], (uint32_t)((it - 1) & 1));
          tc::mbar_arrive_expect_tx(&a_full[h], 2 * KH * RA * 16);
          for (int part = 0; part < 2; ++part)
            for (int kc = h * KH; kc < h * KH + KH; ++kc)
              tc::bulk_g2s(Abase + (size_t)part * A_PART + (size_t)kc * RA * 16,
                           img[part] + ((((long long)b * KC + kc) * p.Rp) + row0) * 16, RA * 16, &a_full[h]);
        }
      }
    } else if (warp_u == 1 && tc::elect_one()) {
      int wi = 0;
      for (int tile = blockIdx.x; tile < p.B * tpi; tile += gridDim.x) {
        for (int h = 0; h < WCH; ++h) {              // the MMAs' order: K half, tap, hi | lo
          for (int c = 0; c < 2 * p.ntaps; ++c, ++wi) {
            const int code = (int)(p.tap_cols >> (3 * (c >> 1))) & 7;
            const int st = wi % NSLOT;
            if (wi >= NSLOT) tc::mbar_wait_parked(&w_empty[st], (uint32_t)(((wi / NSLOT) - 1) & 1));
            uint8_t* dst = Wbase + (size_t)st * W_SLOT;
            const uint8_t* src = p.wpk + (size_t)c * W_MAT + (size_t)h * W_SLOT;
            if (code) {        // an edge tap: only its reached columns, one run of w rows per octet
              const uint32_t w = (code & 1 ? 1u : 2u) * GCOLS, off = (code >= 3 ? 2u * GCOLS : 0u) * 16u;
              tc::mbar_arrive_expect_tx(&w_full[st], KH * w * 16);
              for (int kc = 0; kc < KH; ++kc) tc::bulk_g2s(dst + kc * LBO_B + off, src + kc * LBO_B + off, w * 16, &w_full[st]);
            } else {
              tc::mbar_arrive_expect_tx(&w_full[st], W_SLOT);
#pragma unroll
              for (int piece = 0; piece < 2; ++piece)    // two requests in flight per chunk instead of one long one
                tc::bulk_g2s(dst + piece * (W_SLOT / 2), src + piece * (W_SLOT / 2), W_SLOT / 2, &w_full[st]);
            }
          }
        }
      }
    }
    return;
  }
  if (warp_u >= 8) {
    // ------------------------------------------------------------------------------------ epilogue
    tc::setmaxnreg_dec<EPI_REGS>();
    const int ew = warp_u - 8;
    const int q = ew & 3, g = ew >> 2;
    const int row = q * 32 + lane;
    float* arow = Acc + row * ACC_LD;
    // the neighbouring rows (rows 0 and 127 are halo rows whose Snake values no useful row reads: clamped)
    const float* prow = Acc + max(row - 1, 0) * ACC_LD;
    const float* nrow = Acc + min(row + 1, TILE - 1) * ACC_LD;
    constexpr int CU = R >= 8 ? R : 8;            // accumulator columns per unit: whole channels, >= one image octet
    constexpr int NCH = CU / R;                   // channels per unit (2 for R = 4)
    const int NU = p.C / NCH;
    float* edge_g = Edge + g * 128;               // [4 warps][<= 2 channels][lane 0: 5 | lane 31: 5] Snake values
    __nv_bfloat16* o_hi = static_cast<__nv_bfloat16*>(p.o_hi);
    __nv_bfloat16* o_lo = static_cast<__nv_bfloat16*>(p.o_lo);
    const bool do_div = p.out_div != 0.f;
    int it = 0;
    for (int tile = blockIdx.x; tile < p.B * tpi; tile += gridDim.x, ++it) {
      const int b = tile / tpi, t = tile - b * tpi;
      const int tau0 = t * S - HS;
      const int tau = tau0 + row;
      // a ragged item's last row: its later rows are neither read as residual, stored, nor written to the image
      const int nrows_b = RAG ? __ldg(p.lens + b) * p.lscale / R : nrows;
      const bool valid = tau >= 0 && tau < nrows_b, at_end = tau == nrows_b - 1;
      const bool useful = valid && row >= HS && row < TILE - HS;
      // residual rows are independent of the accumulator: the first unit's are requested before the wait,
      // every later unit's one unit ahead
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
      tc::mbar_wait_parked(&stg_full, (uint32_t)(it & 1));      // this tile's accumulator rows are staged
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
          // needs from the neighbouring rows are read from their staged rows, where each row has written its
          // v back over its accumulator columns), then the 5 + 5 Snake values of the neighbouring rows that its
          // decimation filter reaches arrive by warp shuffle (lanes 0 / 31: through a small edge buffer), so
          // nothing is computed twice: 30 FMA + 2 sin per sample instead of 46 + 3.5 for the register-run form
          // with recomputed halos.  Sequence ends: the reference's replicate padding of x
          // (alias/resample.py:28) and of the 2x signal (alias/filter.py:90-91) are two selects each — no scalar path.
#pragma unroll
          for (int j = 0; j < CU / 4; ++j)
            *reinterpret_cast<float4*>(arow + u * CU + 4 * j) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
          asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
          // 2x-rate Snake values as (even, odd) pairs V[a + 3], a = position relative to the row's first sample:
          // own a = 0 .. R-1; the previous row's last five values are V[0].y, V[1], V[2], the next row's first five
          // V[R+3], V[R+4], V[R+5].x.  All FIR / range-reduction arithmetic runs as f32x2 pair operations (f2_fma /
          // FMUL2 / FADD2: one issue slot for the even and the odd phase), taps as uniform-register pairs.
          float2 V[NCH][R + 6];
#pragma unroll
          for (int k = 0; k < NCH; ++k) {
            const float a_ = s_par[1][c0 + k], hb_ = 0.5f * s_par[2][c0 + k];
            const int col = (c0 + k) * R;
            float xw[R + 8];                                         // samples -4 .. R+3 relative to the row's first
            float4 l4 = *reinterpret_cast<const float4*>(prow + col + R - 4);   // previous row's last four
            float4 r4 = *reinterpret_cast<const float4*>(nrow + col);           // next row's first four
            if (tau == 0) l4 = make_float4(v[k * R], v[k * R], v[k * R], v[k * R]);
            if (at_end) r4 = make_float4(v[k * R + R - 1], v[k * R + R - 1], v[k * R + R - 1], v[k * R + R - 1]);
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
            if (at_end) {
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
      // every row of this warp has been read: once all twelve warps have arrived, the MMA warpgroup may stage
      // the next tile over the buffer
      __syncwarp();
      if (lane == 0) tc::mbar_arrive(&stg_free);
    }
    return;
  }
  // ------------------------------------------------------------------------------------ MMAs
  tc::setmaxnreg_inc<MMA_REGS>();
  const int tw = tid & 127;
  const uint32_t a_h0 = tc::smem_u32(Abase), a_l0 = a_h0 + A_PART, w_s0 = tc::smem_u32(Wbase);
  int wi = 0, it = 0;
  for (int tile = blockIdx.x; tile < p.B * tpi; tile += gridDim.x, ++it) {
    float acc0[N / 2], acc1[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) { acc0[i] = 0.f; acc1[i] = 0.f; }
#pragma unroll   // part and h are constants: each chunk is one branch-free commit group
    for (int h = 0; h < WCH; ++h) {
      // K half h of every tap: the panel's other half may still be loading, and once this loop's last chunk has
      // retired the half is released for the next tile's copies
      tc::mbar_wait_parked(&a_full[h], (uint32_t)(it & 1));
      for (int tap = 0; tap < p.ntaps; ++tap) {
        const uint32_t arow_off = (uint32_t)(A_OFF - p.mlo + tap) * 16u;   // row shift
        const int code = (int)(p.tap_cols >> (3 * tap)) & 7;
#pragma unroll
        for (int part = 0; part < 2; ++part) {   // W_hi: A_hi x W_hi, A_lo x W_hi;  W_lo: A_hi x W_lo
          const uint32_t koff = arow_off + (uint32_t)h * (KH / 2) * 2u * LBO_A;
          const uint64_t ah0 = tc::smem_desc(a_h0 + koff, LBO_A), al0 = tc::smem_desc(a_l0 + koff, LBO_A);
          const uint64_t ah1 = tc::smem_desc(a_h0 + koff + 64u * 16u, LBO_A), al1 = tc::smem_desc(a_l0 + koff + 64u * 16u, LBO_A);
          const int st = wi % NSLOT;
          tc::mbar_wait_parked(&w_full[st], (uint32_t)((wi / NSLOT) & 1));
          const uint64_t bw = tc::smem_desc(w_s0 + (uint32_t)st * W_SLOT, LBO_B);
          tc::wg_fence();
          if (part == 0) { s2d_mma_tap<true>(acc0, ah0, al0, bw, code); s2d_mma_tap<true>(acc1, ah1, al1, bw, code); }
          else { s2d_mma_tap<false>(acc0, ah0, al0, bw, code); s2d_mma_tap<false>(acc1, ah1, al1, bw, code); }
          tc::wg_commit();
          // drain before the next chunk: the ring is fed from L2 about as fast as the MMAs consume it, so the
          // slot is released the moment its MMAs retire
          tc::wg_wait<0>();
          if (tw == 0) tc::mbar_arrive(&w_empty[st]);
          ++wi;
        }
      }
      if (tw == 0) tc::mbar_arrive(&a_empty[h]);
    }
    tc::wg_hold(acc0);
    tc::wg_hold(acc1);
    if (it >= 1) tc::mbar_wait_parked(&stg_free, (uint32_t)((it - 1) & 1));
    s2d_stage_acc<R>(acc0, Acc);
    s2d_stage_acc<R>(acc1, Acc + 64 * ACC_LD);
    tc::mbar_arrive(&stg_full);
  }
}

// ------------------------------------------------------------------------------------------------ serial link
constexpr int S2D_SERIAL_TAPS = 7;   // links of this many taps or more run the serial kernel below
// The links of 7 or more taps keep the schedule the overlapped kernel replaced: MMAs, staging and epilogue one after
// the other per tile, two MMA warpgroups of 64 rows, and whole weight matrices through a 2 x 51,200 B ring with the
// staged accumulator over it.  Their tap loop is long enough that the epilogue is the smaller share, and the
// half-matrix ring of the overlapped kernel starves it (DESIGN.md, "Overlapped epilogue").
namespace s2d_serial {
using namespace s2d;
constexpr uint32_t W_SLOT = KC * N * 16;        // 51,200 B: one (tap, hi|lo) matrix
constexpr int STRIP = TILE * 8;                 // floats of one group's strip: 128 rows x (first 4 | last 4 samples) of one channel,
                                                // or 128 rows x 4 samples of two channels (r = 4)
constexpr uint32_t STG_BYTES = 64 + GROUPS * STRIP * 4 + 64 + GROUPS * 128 * 4;  // sample strips (+ guards) + edge buffers
constexpr uint32_t RES_W = 20 * 40 * 16;       // 12,800 B: the first tap's W_hi over its 40 reached columns, packed
constexpr uint32_t SMEM = 2 * A_PART + 2 * W_SLOT + STG_BYTES + RES_W;
static_assert(SMEM + 1024 <= 227 * 1024, "A panel + weight ring + strips + resident matrix must fit the 227 KB of one CTA");
constexpr int THREADS = (EPI_WARPS + 1) * 32;
static_assert(TILE * ACC_LD * 4 <= 2 * W_SLOT, "the staged accumulator must fit over the weight ring");
// One (tap, hi|lo) matrix over the output columns [N0, N0 + W) it reaches: the accumulator registers of those
// columns (4j .. 4j+3 hold columns 8j .. 8j+7) and the B panel from its row N0 (16 B = one descriptor unit).
// The skipped products are exact zeros, so every output sums the same products in the same order as at W = 160.
// LB: bytes between the K-chunks of the B panel (LBO_B in the ring; W * 16 for a matrix packed to its columns).
template <int W, int N0, bool ALO, uint32_t LB = LBO_B>
__device__ __forceinline__ void s2d_mma(float (&acc)[N / 2], uint64_t ah, uint64_t al, uint64_t bw) {
  using namespace s2d;
  constexpr uint64_t KS = (2 * LB) >> 4;
  float(&d)[W / 2] = *reinterpret_cast<float(*)[W / 2]>(acc + N0 / 2);
#pragma unroll
  for (int kk = 0; kk < N / 16; ++kk) tc::Wg<W, 0>::ss(d, ah + kk * KSA, bw + N0 + kk * KS, 1u);
  if constexpr (ALO) {
#pragma unroll
    for (int kk = 0; kk < N / 16; ++kk) tc::Wg<W, 0>::ss(d, al + kk * KSA, bw + N0 + kk * KS, 1u);
  }
}
// The accumulator is two independent 80-column halves, lower (slots 0, 1) and upper (slots 2, 3), each of which
// a wgmma only ever addresses from its first register: ptxas serialises every wgmma of the kernel once one of
// them starts inside another's register range.  `code` (s2d_tap_plan) is warp-uniform.
// TRIM = false (a link without edge taps to trim): one m64n160 over the whole accumulator per K step.
template <bool ALO, bool TRIM>
__device__ __forceinline__ void s2d_mma_tap(float (&acc)[N / 2], uint64_t ah, uint64_t al, uint64_t bw, int code) {
  if constexpr (!TRIM) {
    s2d_mma<s2d::N, 0, ALO>(acc, ah, al, bw);
    return;
  }
  switch (code) {
    case 1: s2d_mma<40, 0, ALO>(acc, ah, al, bw); break;
    case 2: s2d_mma<80, 0, ALO>(acc, ah, al, bw); break;
    case 3: s2d_mma<40, 80, ALO>(acc, ah, al, bw); break;
    case 4: s2d_mma<80, 80, ALO>(acc, ah, al, bw); break;
    default: s2d_mma<80, 0, ALO>(acc, ah, al, bw); s2d_mma<80, 80, ALO>(acc, ah, al, bw); break;
  }
}

// Persistent: every CTA walks tiles (item, 126 useful rows) with a static stride.
//   producer warp  A panel of the tile (40 bulk copies) and the (tap, hi|lo) weight matrices through a
//                  2-slot ring (four bulk copies each; an edge tap's 20 runs of its reached columns).  The next
//                  tile's A panel is requested as soon as this tile's MMAs retire (a_empty), so it loads under
//                  this tile's epilogue; its weights wait for the epilogue to release the ring (ring_free)
//   warpgroups 0-1 per tap: A_hi x W_hi, A_lo x W_hi, A_hi x W_lo — 30 pairs of wgmma m64n80k16 (one per
//                  accumulator half; one m64n160 when the link has no edge tap to trim) each for its 64 rows, or
//                  30 m64n40 / m64n80 over the reached columns of an edge tap; register accumulators (the wgmma of one matrix form one commit group), then
//                  staged as fp32 rows over the (consumed) weight ring
//   12 epilogue warps = 3 column groups x 4 row quadrants: group g owns units u = g (mod 3), a unit
//                  being one channel (r >= 8) or a channel pair (r = 4): 6-7 / 6-7 / 3-4 units per group for
//                  C = 20 / 40 / 10 (13 warps leave the MMA warpgroups the registers of 160 accumulator columns)
// RAG: a ragged batch (p.lens): a separate instantiation, so that the dense one keeps its registers
// TRIM: the link has edge taps to trim (p.tap_cols != 0); without, one m64n160 per K step as before
template <int R, bool RAG, bool TRIM>
__global__ void __launch_bounds__(THREADS, 1)
amp_s2d_link_serial_kernel(const AmpS2dParams p) {
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t a_full, a_empty, ring_free, w_full[2], w_empty[2], res_full;
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
  uint8_t* Res = smem + 2 * A_PART + 2 * W_SLOT + STG_BYTES;
  // The first matrix of every tile waits for the epilogue to release the ring, and its L2 fetch is exposed.
  // When it is a 40-column edge tap (tap 0 reaching phase group 0 only) its W_hi is the same 12,800 B for every
  // tile: it is loaded once, packed to its columns, and stays resident outside the ring.
  const bool res0 = TRIM && (p.tap_cols & 7) == 1;
  float* Acc = reinterpret_cast<float*>(Wbase);  // staged accumulator [TILE][ACC_LD], over the weight ring

  if (tid == 0) {
    tc::mbar_init(&a_full, 1); tc::mbar_init(&a_empty, 1); tc::mbar_init(&ring_free, 1);
    for (int i = 0; i < 2; ++i) { tc::mbar_init(&w_full[i], 1); tc::mbar_init(&w_empty[i], 2); }
    tc::mbar_init(&res_full, 1);
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (warp_u == EPI_WARPS) {
    // ------------------------------------------------------------------------------------ producer
    if (tc::elect_one()) {
      const uint8_t* img[2] = {reinterpret_cast<const uint8_t*>(p.a_hi), reinterpret_cast<const uint8_t*>(p.a_lo)};
      int it = 0, wi = 0;
      if (res0) {
        tc::mbar_arrive_expect_tx(&res_full, RES_W);
        for (int kc = 0; kc < KC; ++kc) tc::bulk_g2s(Res + kc * GCOLS * 16, p.wpk + kc * LBO_B, GCOLS * 16, &res_full);
      }
      for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
        const int b = tile / tpi, t = tile - b * tpi;
        const long long row0 = (long long)t * S - HS - A_OFF + PADR;     // image row of A-panel row 0 (>= 6)
        // the A panel is free once the previous tile's MMAs have retired: its copies run under that tile's
        // epilogue; the ring holds that epilogue's staged accumulator until the epilogue has read it
        if (it >= 1) tc::mbar_wait_parked(&a_empty, (uint32_t)((it - 1) & 1));
        tc::mbar_arrive_expect_tx(&a_full, 2 * A_PART);
        for (int part = 0; part < 2; ++part)
          for (int kc = 0; kc < KC; ++kc)
            tc::bulk_g2s(Abase + (size_t)part * A_PART + (size_t)kc * RA * 16,
                         img[part] + ((((long long)b * KC + kc) * p.Rp) + row0) * 16, RA * 16, &a_full);
        if (it >= 1) tc::mbar_wait_parked(&ring_free, (uint32_t)((it - 1) & 1));
        for (int c = res0 ? 1 : 0; c < 2 * p.ntaps; ++c, ++wi) {
          const int st = wi & 1;
          if (wi >= 2) tc::mbar_wait_parked(&w_empty[st], (uint32_t)(((wi >> 1) - 1) & 1));
          const int code = (int)(p.tap_cols >> (3 * (c >> 1))) & 7;
          uint8_t* dst = Wbase + (size_t)st * W_SLOT;
          const uint8_t* src = p.wpk + (size_t)c * W_SLOT;
          if (code) {        // an edge tap: only its reached columns, one run of w rows per octet
            const uint32_t w = (code & 1 ? 1u : 2u) * GCOLS, off = (code >= 3 ? 2u * GCOLS : 0u) * 16u;
            tc::mbar_arrive_expect_tx(&w_full[st], KC * w * 16);
            for (int kc = 0; kc < KC; ++kc) tc::bulk_g2s(dst + kc * LBO_B + off, src + kc * LBO_B + off, w * 16, &w_full[st]);
          } else {
            tc::mbar_arrive_expect_tx(&w_full[st], W_SLOT);
#pragma unroll
            for (int piece = 0; piece < 4; ++piece)    // four requests in flight per matrix instead of one long one
              tc::bulk_g2s(dst + piece * (W_SLOT / 4), src + piece * (W_SLOT / 4), W_SLOT / 4, &w_full[st]);
          }
        }
      }
    }
    return;
  }
  {
    // ------------------------------------------------------------------------------------ epilogue
    const int q = warp & 3, g = warp >> 2;
    const int row = q * 32 + lane;
    // warp_u, not warp: ptxas must see the MMA branch (wg < 2) as warp-uniform, or it serialises every wgmma
    const int wg = warp_u >> 2, tw = tid & 127;
    const uint32_t a_h0 = tc::smem_u32(Abase) + (uint32_t)wg * 64u * 16u, a_l0 = a_h0 + A_PART, w_s0 = tc::smem_u32(Wbase);
    const uint64_t b_res = tc::smem_desc(tc::smem_u32(Res), GCOLS * 16);
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
      // a ragged item's last row: its later rows are neither read as residual, stored, nor written to the image
      const int nrows_b = RAG ? __ldg(p.lens + b) * p.lscale / R : nrows;
      const bool valid = tau >= 0 && tau < nrows_b, at_end = tau == nrows_b - 1;
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
          const int code = (int)(p.tap_cols >> (3 * tap)) & 7;
#pragma unroll   // part is a constant: each matrix is one branch-free commit group
          for (int part = 0; part < 2; ++part) {   // W_hi: A_hi x W_hi, A_lo x W_hi;  W_lo: A_hi x W_lo
            if (part == 0 && tap == 0 && res0) {     // the resident first matrix: no ring slot
              tc::mbar_wait_parked(&res_full, 0u);
              tc::wg_fence();
              s2d_mma<GCOLS, 0, true, GCOLS * 16>(acc, ah, al, b_res);
              tc::wg_commit();
              tc::wg_wait<0>();
              continue;
            }
            const int st = wi & 1;
            tc::mbar_wait_parked(&w_full[st], (uint32_t)((wi >> 1) & 1));
            const uint64_t bw = tc::smem_desc(w_s0 + (uint32_t)st * W_SLOT, LBO_B);
            tc::wg_fence();
            if (part == 0) s2d_mma_tap<true, TRIM>(acc, ah, al, bw, code);
            else s2d_mma_tap<false, TRIM>(acc, ah, al, bw, code);
            tc::wg_commit();
            // drain before the next matrix: the ring is fed from L2 about as fast as the MMAs consume it, so
            // the slot is released the moment its MMAs retire (releasing it one matrix later, under
            // wgmma.wait_group 1, made the links 2-33 % slower on an H100 SXM at 700 W)
            tc::wg_wait<0>();
            if (tw == 0) tc::mbar_arrive(&w_empty[st]);
            ++wi;
          }
        }
        tc::wg_hold(acc);
        tc::named_sync(6, 256);                   // both warpgroups' MMAs have retired: A panel and ring are free
        if (tid == 0) tc::mbar_arrive(&a_empty);
        s2d_stage_acc<R>(acc, Acc + wg * 64 * ACC_LD);
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
            if (at_end) r4 = make_float4(v[k * R + R - 1], v[k * R + R - 1], v[k * R + R - 1], v[k * R + R - 1]);
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
            if (at_end) {
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
      tc::fence_proxy_async_smem();               // staged rows (generic proxy) -> the next tile's weight copies
      tc::named_sync(7, EPI_WARPS * 32);
      if (tid == 0) tc::mbar_arrive(&ring_free);
    }
  }
}
}  // namespace s2d_serial

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
  for (int t = 0; t < p.ntaps; ++t)
    if (((p.tap_cols >> (3 * t)) & 7) > 4) {
      set_error("amp_s2d_link: a tap's column range is empty");
      return SVCB_E_BAD_SHAPE;
    }
  static DevSmemCache c4, c8, c16, g4, g8, g16;
  static DevSmemCache sc4, sc8, sc16, sg4, sg8, sg16, su4, su8, su16, sv4, sv8, sv16;
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
#define SVCB_S2D_LINK(r_, rag, cache)                                                 \
  do {                                                                                \
    SVCB_CUDA_CHECK(ensure_dyn_smem(amp_s2d_link_kernel<r_, rag>, s2d::SMEM, cache)); \
    amp_s2d_link_kernel<r_, rag><<<grid, s2d::THREADS, s2d::SMEM, s>>>(p);            \
  } while (0)
#define SVCB_S2D_SERIAL(r_, rag, trim, cache)                                                                      \
  do {                                                                                                             \
    SVCB_CUDA_CHECK(ensure_dyn_smem(s2d_serial::amp_s2d_link_serial_kernel<r_, rag, trim>, s2d_serial::SMEM, cache)); \
    s2d_serial::amp_s2d_link_serial_kernel<r_, rag, trim><<<grid, s2d_serial::THREADS, s2d_serial::SMEM, s>>>(p);  \
  } while (0)
  if (p.ntaps >= S2D_SERIAL_TAPS) {
    // links without a trimmed tap keep the single 160-column accumulator (one m64n160 per K step)
    const bool trim = p.tap_cols != 0;
    if (p.lens && trim) {
      if (r == 4) SVCB_S2D_SERIAL(4, true, true, sg4);
      else if (r == 8) SVCB_S2D_SERIAL(8, true, true, sg8);
      else SVCB_S2D_SERIAL(16, true, true, sg16);
    } else if (p.lens) {
      if (r == 4) SVCB_S2D_SERIAL(4, true, false, sv4);
      else if (r == 8) SVCB_S2D_SERIAL(8, true, false, sv8);
      else SVCB_S2D_SERIAL(16, true, false, sv16);
    } else if (trim) {
      if (r == 4) SVCB_S2D_SERIAL(4, false, true, sc4);
      else if (r == 8) SVCB_S2D_SERIAL(8, false, true, sc8);
      else SVCB_S2D_SERIAL(16, false, true, sc16);
    } else {
      if (r == 4) SVCB_S2D_SERIAL(4, false, false, su4);
      else if (r == 8) SVCB_S2D_SERIAL(8, false, false, su8);
      else SVCB_S2D_SERIAL(16, false, false, su16);
    }
  } else if (p.lens) {
    if (r == 4) SVCB_S2D_LINK(4, true, g4);
    else if (r == 8) SVCB_S2D_LINK(8, true, g8);
    else SVCB_S2D_LINK(16, true, g16);
  } else {
    if (r == 4) SVCB_S2D_LINK(4, false, c4);
    else if (r == 8) SVCB_S2D_LINK(8, false, c8);
    else SVCB_S2D_LINK(16, false, c16);
  }
#undef SVCB_S2D_SERIAL
#undef SVCB_S2D_LINK
  SVCB_LAUNCH_CHECK("amp_s2d_link");
  return SVCB_OK;
}

}  // namespace svcb

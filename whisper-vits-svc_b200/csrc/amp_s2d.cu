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
// conv's zero padding).  A tile = 128 consecutive rows of every octet = 20 bulk copies per split part, already in
// the K-major SWIZZLE_NONE panel layout of tc.cuh, and a Toeplitz tap is a row-shifted descriptor.
//
// Folded image (fold f = the dilation d of the link that reads it, f > 1): a conv of dilation d is d independent
// undilated convs, one per stream x[q], x[q+d], ...  Row b*f + q (after the 16 zero rows) holds the r samples
// b*r*f + q + j*f, j = 0 .. r-1, of stream q: the standard image permuted inside blocks of r*f samples.  The link
// then runs the undilated conv's matrices, tap m shifted by m*f rows, over tiles of whole blocks.  Every writer
// stores every position of an item's first nrows + S2D_TAIL rows (zeros past the item's end), because the two
// ping-pong images are reused by links of folds 1, 3 and 5 and an "outside" position of one fold held a sample in
// another; rows after those are never written and stay as cleared once per stage.
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

// rows every writer stores past an item's last row, zeros: they cover the last block of every fold up to FOLD_MAX
constexpr int S2D_FOLD_MAX = 5, S2D_TAIL = S2D_FOLD_MAX - 1;

int s2d_rows(int L, int r) {                                         // Rp of an image (any fold; see s2d_tile)
  const int nrows = L / r, S = s2d::TILE - 2 * (r >= 8 ? 1 : 2);
  return ((nrows + S - 1) / S) * S + 160;
}
size_t s2d_image_bytes(int B, int L, int r) { return (size_t)B * s2d::KC * s2d_rows(L, r) * 16; }

// Tile geometry of a link whose input image has fold fin and output image fold fout (at most one of them > 1).
// Useful rows per tile `stride`, `halo` rows on each side (SnakeAlias reaches +-5 samples); a_off = A-panel row of
// the tile's first accumulator row.  A folded input: tiles of whole blocks, a halo of one block, and as many rows as
// fit the A panel with the taps' reach of +-m*fin rows (rows past them are computed from the next octet's rows and
// never used).  A folded output: whole output blocks of useful rows.  Twin: pack.py:s2d_tile.
S2dTile s2d_tile(int r, int fin, int fout, int mlo, int mhi) {
  S2dTile t;
  if (fin > 1) {
    const int rows = std::min(s2d::TILE, s2d::RA - (mlo + mhi) * fin) / fin * fin;
    t.halo = fin; t.stride = rows - 2 * fin; t.a_off = mlo * fin;
  } else {
    t.halo = r >= 8 ? 1 : 2; t.stride = (s2d::TILE - 2 * t.halo) / fout * fout; t.a_off = s2d::A_OFF;
  }
  return t;
}

// Output columns of the weights and the accumulator come in four slots of 40, n = 40 s + g c + j: slot s holds
// the g = r / 4 phases p = g q + j of every channel c of phase group q = {0, 1, 3, 2}[s] (pack.py:
// s2d_column_order).  Row tap m reaches the phases [max(0, r m - P), min(r - 1, r m + r - 1 + P)] only, so the
// matrix of an edge tap is zero outside the groups {0}, {0, 1} (m < 0) or {3}, {3, 2} (m > 0), that is outside
// columns [0, 40), [0, 80), [80, 120) or [80, 160).  Per tap 3 bits: code 1-4 = those ranges, 0 = all columns.
static bool s2d_taps(int k, int dil, int r, S2dPlan& pl) {
  const int P = dil * (k - 1) / 2, g = r / 4;
  pl.mlo = (P + r - 1) / r;
  pl.ntaps = pl.mlo + (r - 1 + P) / r + 1;
  pl.tap_cols = 0;
  if (g < 1 || pl.ntaps > 21) return false;
  for (int t = 0; t < pl.ntaps; ++t) {
    const int m = t - pl.mlo;
    const int q0 = std::max(0, r * m - P) / g, q1 = std::min(r - 1, r * m + r - 1 + P) / g;
    const int code = q0 == 0 && q1 <= 1 ? 1 + q1 : q1 == 3 && q0 >= 2 ? 3 + (3 - q0) : 0;
    pl.tap_cols |= (uint64_t)code << (3 * t);
  }
  return true;
}
// 40-column units a link multiplies per tile row (a full tap 4, an edge tap 1 or 2)
static int s2d_col_units(const S2dPlan& pl) {
  int u = 0;
  for (int t = 0; t < pl.ntaps; ++t) {
    const int code = (int)(pl.tap_cols >> (3 * t)) & 7;
    u += code == 0 ? 4 : code & 1 ? 1 : 2;
  }
  return u;
}
// The fold a c1 link reads its input in: its dilation when the link has more than 3 full taps of column work and the
// undilated conv's column work per useful row (tap work over the tile stride, which the one-block halo shortens) is
// lower, else 1.  Twin: pack.py:s2d_fold.
bool s2d_tap_plan(int k, int dil, int r, S2dPlan& pl) {
  pl.fold = 1;
  if (!s2d_taps(k, dil, r, pl)) return false;
  S2dPlan u;
  if (dil < 2 || dil > S2D_FOLD_MAX || !s2d_taps(k, 1, r, u)) return true;
  const S2dTile t1 = s2d_tile(r, 1, 1, pl.mlo, pl.ntaps - 1 - pl.mlo), td = s2d_tile(r, dil, 1, u.mlo, u.ntaps - 1 - u.mlo);
  if (td.stride <= 0 || td.halo + td.a_off > s2d::PADR) return true;
  // A link of at most 3 full taps of column work is bound by its Snake epilogue, which reads a folded tile's
  // samples one by one through the permutation: folded, such links measured up to 20 % slower (DESIGN.md §5)
  const int cu = s2d_col_units(pl);
  if (cu > 12 && (long long)s2d_col_units(u) * t1.stride < (long long)cu * td.stride) { pl = u; pl.fold = dil; }
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
// SnakeAlias(x[B,C,L]) -> S2D image of fold f (the first activation of every AMP block: its input is the stage
// input, not a convolution result).  One thread = one run of 8 samples; runs past the item's end up to its last
// written row (S2D_TAIL, whole blocks of f) store zeros.  Fold 1: the run is one image row of one octet (half an
// octet in two rows for r = 4).  Fold f > 1: its samples lie in 8 different rows, 2-byte stores (no link of
// configs/base.yaml reads a folded image written here: its first dilation is 1).
// One run of 8 samples of channel c from sample n0 into the image of fold f
template <bool FOLDED>
__device__ __forceinline__ void s2d_pack_store(__nv_bfloat16* hi, __nv_bfloat16* lo, const float (&out)[8], long long item,
                                               int c, int n0, int r, int Rp, int f) {
  if constexpr (FOLDED) {
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int s = n0 + j, blk = s / (r * f), w = s - blk * r * f;
      const int k = c * r + w / f, row = blk * f + w % f;
      const long long e = (item + (long long)(k >> 3) * Rp + s2d::PADR + row) * 8 + (k & 7);
      const __nv_bfloat16 h = __float2bfloat16_rn(out[j]);
      hi[e] = h;
      lo[e] = __float2bfloat16_rn(out[j] - __bfloat162float(h));
    }
  } else if (r >= 8) {
    const int opr = r >> 3, run = n0 >> 3;       // octets per row of this channel
    const int row = run / opr, o = c * opr + run % opr;
    s2d_store_octet(hi, lo, (item + (long long)o * Rp + s2d::PADR + row) * 8, out);
  } else {   // r = 4: the run covers rows 2*run, 2*run+1; this channel is half (4 elements) of octet c / 2
    __align__(8) __nv_bfloat162 h2[4], l2[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      h2[k] = __floats2bfloat162_rn(out[2 * k], out[2 * k + 1]);
      const float2 f2 = __bfloat1622float2(h2[k]);
      l2[k] = __floats2bfloat162_rn(out[2 * k] - f2.x, out[2 * k + 1] - f2.y);
    }
#pragma unroll
    for (int hrow = 0; hrow < 2; ++hrow) {
      const long long e = (item + (long long)(c >> 1) * Rp + s2d::PADR + n0 / 4 + hrow) * 8 + (c & 1) * 4;
      *reinterpret_cast<uint2*>(hi + e) = *reinterpret_cast<const uint2*>(h2 + 2 * hrow);
      *reinterpret_cast<uint2*>(lo + e) = *reinterpret_cast<const uint2*>(l2 + 2 * hrow);
    }
  }
}

template <bool FOLDED>
__global__ void __launch_bounds__(256, 4)
snake_pack_s2d_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ hi, __nv_bfloat16* __restrict__ lo,
                      const float* __restrict__ ea, const float* __restrict__ inv_b,
                      const SnakeTapsV tp, int C, int L, int r, int Rp, const int* __restrict__ lens, int lscale, int f) {
  const int run = blockIdx.x * 256 + threadIdx.x;
  const int c = blockIdx.y, b = blockIdx.z;
  const int Lb = lens ? __ldg(lens + b) * lscale : L;   // a ragged item's end
  const long long item = (long long)b * s2d::KC * Rp;
  const int n0 = run * 8;
  if (n0 >= Lb) {   // past the item's end, up to its last written row (S2D_TAIL, whole blocks of f): zeros
    if (n0 < (Lb / r + S2D_TAIL + f - 1) / f * f * r) {
      const float zero[8] = {};
      s2d_pack_store<FOLDED>(hi, lo, zero, item, c, n0, r, Rp, f);
    }
    return;
  }
  const float* xr = x + ((long long)b * C + c) * L;
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
  s2d_pack_store<FOLDED>(hi, lo, out, item, c, n0, r, Rp, f);
}

int launch_snake_pack_s2d(const float* x, void* hi, void* lo, const float* ea, const float* inv_b, const float* fu,
                          const float* fd, int B, int C, int L, cudaStream_t s, const SnakeTapsV* taps, const int* lens,
                          int lscale, int fold) {
  const int r = C > 0 ? s2d::N / C : 0;
  if (B <= 0 || L <= 0 || C * r != s2d::N || (r != 4 && r != 8 && r != 16) || L % 8 || L % r || fold < 1 ||
      fold > S2D_FOLD_MAX || (reinterpret_cast<uintptr_t>(x) & 15)) {
    set_error("snake_pack_s2d: unsupported shape");
    return SVCB_E_BAD_SHAPE;
  }
  SnakeTapsV tp;
  if (taps) tp = *taps;
  else SVCB_TRY(snake_taps_from_device(fu, fd, &tp));
  char kname[64];
  snprintf(kname, sizeof(kname), "snake_pack_s2d_c%d", C);
  KernelScope ks(kname, s, 0.0, 8.0 * B * C * (double)L, 70.0 * B * C * (double)L);
  const int ext = (L / r + S2D_TAIL + fold - 1) / fold * fold * r;
  dim3 grid((ext / 8 + 1 + 255) / 256, C, B);
  auto kern = fold > 1 ? snake_pack_s2d_kernel<true> : snake_pack_s2d_kernel<false>;
  kern<<<grid, 256, 0, s>>>(x, static_cast<__nv_bfloat16*>(hi), static_cast<__nv_bfloat16*>(lo), ea, inv_b, tp, C, L, r,
                            s2d_rows(L, r), lens, lscale, fold);
  SVCB_LAUNCH_CHECK("snake_pack_s2d");
  return SVCB_OK;
}

// S2D image of fold f (hi + lo) -> fp32 [B, C, L]: the unit tests read a link's output image through this.
__global__ void s2d_unpack_kernel(const __nv_bfloat16* __restrict__ hi, const __nv_bfloat16* __restrict__ lo,
                                  float* __restrict__ y, int C, int L, int r, int Rp, int f) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;     // over C * L of item blockIdx.y
  if (i >= (long long)C * L) return;
  const int c = (int)(i / L), t = (int)(i % L);
  const int blk = t / (r * f), w = t - blk * r * f;
  const int k = c * r + w / f, row = blk * f + w % f;
  const long long e = ((((long long)blockIdx.y * s2d::KC + k / 8) * Rp) + s2d::PADR + row) * 8 + k % 8;
  y[(long long)blockIdx.y * C * L + i] = __bfloat162float(hi[e]) + __bfloat162float(lo[e]);
}
int launch_s2d_unpack(const void* hi, const void* lo, float* y, int B, int C, int L, cudaStream_t s, int fold) {
  const int r = s2d::N / C;
  dim3 grid((unsigned)(((long long)C * L + 255) / 256), B);
  s2d_unpack_kernel<<<grid, 256, 0, s>>>(static_cast<const __nv_bfloat16*>(hi), static_cast<const __nv_bfloat16*>(lo), y, C, L, r,
                                         s2d_rows(L, r), fold);
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

// Persistent: every CTA walks tiles (item, p.stride useful rows, s2d_tile) with a static stride.  Tile i's epilogue
// runs while tile i+1's MMAs run: the accumulator is staged into a buffer of its own, not over the weight ring.
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
// MODE: FOLD_STD (input and output standard), FOLD_IN (the input image is folded, p.fin > 1: the epilogue thread of
//   row rho reads the r samples rho*r + j from the staged rows through the fold's permutation, s_tab), FOLD_OUT (the
//   output image is folded, p.fout > 1: the thread writes its Snake values back over its row and, after a barrier,
//   gathers the 8 samples of one octet of the folded row it owns, so the stores stay 16 B wide)
enum { FOLD_STD = 0, FOLD_IN = 1, FOLD_OUT = 2 };
template <int R, bool RAG, int MODE>
__global__ void __launch_bounds__(s2d::THREADS, 1)
amp_s2d_link_kernel(const AmpS2dParams p) {
  using namespace s2d;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t a_full[WCH], a_empty[WCH], w_full[NSLOT], w_empty[NSLOT], stg_full, stg_free;
  __shared__ float s_par[3][40];      // bias | exp(alpha) | 1 / (exp(beta) + 1e-9) of every channel (C <= 40)
  // FOLD_IN: staged-buffer offset of sample a = -4 .. R+3 of a row rho = blk * fin + e, relative to row blk * fin:
  // row e = 0 .. fin-1 of a tile's blocks, row fin = the identity (rows past the tile's blocks)
  constexpr int TW = R + 8;
  __shared__ __align__(16) int s_tab[MODE == FOLD_IN ? (S2D_FOLD_MAX + 1) * TW : 4];

  const int tid = threadIdx.x, lane = tid & 31;
  const int warp_u = tc::warp_uniform_idx();
  if (tid < p.C) {
    s_par[0][tid] = __ldg(p.bias + tid);
    s_par[1][tid] = p.o_hi ? __ldg(p.ea + tid) : 0.f;
    s_par[2][tid] = p.o_hi ? __ldg(p.ib + tid) : 0.f;
  }
  if constexpr (MODE == FOLD_IN) {
    const int f = p.fin;
    for (int i = tid; i < (f + 1) * TW; i += blockDim.x) {
      const int e = i / TW, a = i % TW - 4;
      int off;
      if (e == f) {
        off = a < 0 ? a + R - ACC_LD : a >= R ? a - R + ACC_LD : a;
      } else {
        int w = e * R + a;
        const int bb = w < 0 ? -1 : w >= R * f ? 1 : 0;
        w -= bb * R * f;
        off = (bb * f + w % f) * ACC_LD + w / f;
      }
      s_tab[i] = off;
    }
  }
  const int HS = p.halo, S = p.stride;
  const int nrows = p.L / R;
  const int tpi = (nrows + S2D_TAIL + S - 1) / S;     // the writers' rows past an item's end are in some tile
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
        const long long row0 = (long long)t * S - HS - p.a_off + PADR;   // image row of A-panel row 0 (>= 1)
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
    // FOLD_IN: the thread still owns standard row tau = tile start + row (tiles start at a block), whose samples
    // sit at frow + s_tab[e][a] of the staged rows; rows past the tile's blocks read and write their own row
    int fe = 0, fbase = row;
    if constexpr (MODE == FOLD_IN) {
      if (row < S + 2 * HS) { fe = row % p.fin; fbase = row - fe; }
      else fe = p.fin;
    }
    float* frow = Acc + fbase * ACC_LD;
    const int* ftab = s_tab + fe * TW + 4;
    // FOLD_OUT: the folded row this thread writes is block blk, stream q of the tile's useful rows: its element j
    // is sample osb + j * fout after the first useful row
    int osb = 0;
    if constexpr (MODE == FOLD_OUT) {
      const int rl = max(row - HS, 0), blk = rl / p.fout;
      osb = blk * R * p.fout + rl - blk * p.fout;
    }
    int it = 0;
    for (int tile = blockIdx.x; tile < p.B * tpi; tile += gridDim.x, ++it) {
      const int b = tile / tpi, t = tile - b * tpi;
      const int tau0 = t * S - HS;
      const int tau = tau0 + row;
      // a ragged item's last row: its later rows are neither read as residual nor stored; the image gets zeros there
      const int nrows_b = RAG ? __ldg(p.lens + b) * p.lscale / R : nrows;
      const bool valid = tau >= 0 && tau < nrows_b, at_end = tau == nrows_b - 1;
      const bool inner = row >= HS && row < HS + S;
      const bool useful = valid && inner;
      const bool img_row = inner && tau < nrows_b + S2D_TAIL;     // the image rows this thread writes
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
          if constexpr (MODE == FOLD_IN) {
#pragma unroll
            for (int i = 0; i < 4; ++i) dst[k + i] = __float_as_uint(frow[col + k + i - (k + i) % R + ftab[(k + i) % R]]);
          } else {
            const float4 q4 = *reinterpret_cast<const float4*>(arow + col + k);
            dst[k] = __float_as_uint(q4.x); dst[k + 1] = __float_as_uint(q4.y); dst[k + 2] = __float_as_uint(q4.z); dst[k + 3] = __float_as_uint(q4.w);
          }
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
          if constexpr (MODE == FOLD_IN) {
#pragma unroll
            for (int k = 0; k < CU; ++k) frow[u * CU + k - k % R + ftab[k % R]] = v[k];
          } else {
#pragma unroll
            for (int j = 0; j < CU / 4; ++j)
              *reinterpret_cast<float4*>(arow + u * CU + 4 * j) = make_float4(v[4 * j], v[4 * j + 1], v[4 * j + 2], v[4 * j + 3]);
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
            const int col = (c0 + k) * R;
            float xw[R + 8];                                         // samples -4 .. R+3 relative to the row's first
            float4 l4, r4;                                           // previous row's last four, next row's first four
            if constexpr (MODE == FOLD_IN) {
              l4 = make_float4(frow[col + ftab[-4]], frow[col + ftab[-3]], frow[col + ftab[-2]], frow[col + ftab[-1]]);
              r4 = make_float4(frow[col + ftab[R]], frow[col + ftab[R + 1]], frow[col + ftab[R + 2]], frow[col + ftab[R + 3]]);
            } else {
              l4 = *reinterpret_cast<const float4*>(prow + col + R - 4);
              r4 = *reinterpret_cast<const float4*>(nrow + col);
            }
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
          if (tau >= nrows_b) {                                     // past the item's end: zeros
#pragma unroll
            for (int i = 0; i < CU; ++i) out[i] = 0.f;
          }
          if constexpr (MODE == FOLD_OUT) {
            // every Snake value of the unit has been read (second barrier): the row's values go back over its
            // columns, and the octet of folded row tau gathers its 8 samples from the d rows of its block
#pragma unroll
            for (int j = 0; j < CU / 4; ++j)
              *reinterpret_cast<float4*>(arow + u * CU + 4 * j) = make_float4(out[4 * j], out[4 * j + 1], out[4 * j + 2], out[4 * j + 3]);
            asm volatile("bar.sync %0, 128;" ::"r"(1 + g) : "memory");
            if (img_row) {
#pragma unroll
              for (int i = 0; i < CU; ++i) {
                const int s = osb + (i % R) * p.fout;             // channel c0 + i / R, phase i % R of the folded row
                out[i] = Acc[(HS + s / R) * ACC_LD + (c0 + i / R) * R + s % R];
              }
            }
          }
          if (img_row) {
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
        const uint32_t arow_off = (uint32_t)(p.a_off + (tap - p.mlo) * p.fin) * 16u;   // row shift
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

int launch_amp_s2d_link(const AmpS2dParams& p_in, cudaStream_t s) {
  AmpS2dParams p = p_in;
  const int r = p.C > 0 ? s2d::N / p.C : 0;
  if (p.B <= 0 || p.L <= 0 || p.C * r != s2d::N || (r != 4 && r != 8 && r != 16) || p.L % r) {
    set_error("amp_s2d_link: unsupported shape (need C * r = 160 with r in {4, 8, 16} and L % r == 0)");
    return SVCB_E_BAD_SHAPE;
  }
  if (p.fin < 1 || p.fout < 1 || p.fin > S2D_FOLD_MAX || p.fout > S2D_FOLD_MAX || (p.fin > 1 && p.fout > 1) ||
      (p.fout > 1 && !p.o_hi)) {
    set_error("amp_s2d_link: folds must be in [1, 5], at most one of input and output folded, a folded output written");
    return SVCB_E_BAD_SHAPE;
  }
  const int mhi = p.ntaps - 1 - p.mlo;
  const S2dTile tg = s2d_tile(r, p.fin, p.fout, p.mlo, mhi);
  p.halo = tg.halo; p.stride = tg.stride; p.a_off = tg.a_off;
  const int tpi = (p.L / r + S2D_TAIL + p.stride - 1) / max(p.stride, 1);
  // the A panel of every tap of every tile, and every image row written, lie inside the image
  const int rows_used = p.fin > 1 ? p.stride + 2 * p.halo : s2d::TILE;   // accumulator rows the epilogue reads
  if (p.ntaps < 1 || p.mlo < 0 || mhi < 0 || p.stride <= 0 || p.a_off < p.mlo * p.fin ||
      p.a_off + mhi * p.fin + rows_used > s2d::RA || p.halo + p.a_off > s2d::PADR || (long long)(tpi - 1) * p.stride - p.halo - p.a_off + s2d::PADR + s2d::RA > p.Rp ||
      p.Rp != s2d_rows(p.L, r) || !p.a_hi || !p.a_lo || !p.wpk || !p.bias || (p.o_hi && (!p.o_lo || !p.ea || !p.ib || !p.fu || !p.fd))) {
    set_error("amp_s2d_link: tap range exceeds the A panel, wrong image rows or missing operand");
    return SVCB_E_BAD_SHAPE;
  }
  for (int t = 0; t < p.ntaps; ++t)
    if (((p.tap_cols >> (3 * t)) & 7) > 4) {
      set_error("amp_s2d_link: a tap's column range is empty");
      return SVCB_E_BAD_SHAPE;
    }
  static DevSmemCache cache[3][2][3];   // r, ragged, mode
  const int n_sm = device_sm_count();
  if (n_sm <= 0) { set_error("amp_s2d_link: cannot query the SM count"); return SVCB_E_CUDA; }
  const int ntiles = p.B * tpi;
  const int grid = std::min(ntiles, n_sm);
  char kname[64];
  snprintf(kname, sizeof(kname), "amp_s2d_link_c%dk%dr%d", p.C, p.K, r);
  const double el = (double)p.B * p.C * p.L;
  KernelScope ks(kname, s, 2.0 * p.C * p.K * el, el * (4.0 + (p.o_hi ? 4.0 : 0.0) + (p.res ? 4.0 : 0.0) + (p.y ? (p.accum ? 8.0 : 4.0) : 0.0)),
                 p.o_hi ? 70.0 * el : 0.0);
  const int mode = p.fin > 1 ? FOLD_IN : p.fout > 1 ? FOLD_OUT : FOLD_STD;
  const int ri = r == 4 ? 0 : r == 8 ? 1 : 2;
  auto launch = [&](auto kern) -> int {
    SVCB_CUDA_CHECK(ensure_dyn_smem(kern, s2d::SMEM, cache[ri][p.lens ? 1 : 0][mode]));
    kern<<<grid, s2d::THREADS, s2d::SMEM, s>>>(p);
    return SVCB_OK;
  };
#define SVCB_S2D_MODES(r_, rag)                                                       \
  (mode == FOLD_IN    ? launch(amp_s2d_link_kernel<r_, rag, FOLD_IN>)                 \
   : mode == FOLD_OUT ? launch(amp_s2d_link_kernel<r_, rag, FOLD_OUT>)                \
                      : launch(amp_s2d_link_kernel<r_, rag, FOLD_STD>))
  int rc;
  if (p.lens) rc = r == 4 ? SVCB_S2D_MODES(4, true) : r == 8 ? SVCB_S2D_MODES(8, true) : SVCB_S2D_MODES(16, true);
  else rc = r == 4 ? SVCB_S2D_MODES(4, false) : r == 8 ? SVCB_S2D_MODES(8, false) : SVCB_S2D_MODES(16, false);
#undef SVCB_S2D_MODES
  SVCB_TRY(rc);
  SVCB_LAUNCH_CHECK("amp_s2d_link");
  return SVCB_OK;
}

}  // namespace svcb

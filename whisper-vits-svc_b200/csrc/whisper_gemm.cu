// Dense bf16 GEMM on wgmma for the Whisper encoder's linear layers, with fused epilogues.
//
//   C[M,N] = A[M,K] . W[N,K]^T + bias        replaces the F.linear calls of whisper/model.py:66-82
//                                            (query/key/value/out) and :116 (Linear -> GELU -> Linear)
//                                            including bias, GELU and the residual adds.
//
// Operands live in HBM as *tile images*: A (activations, written by the producing kernels) and W
// (packed by the host) are stored tile by tile — [row-tile][k-tile] blocks of 128 (or BN) rows x 64
// k, each block already in the K-major panel order of tc.cuh ([k/8][row][8]).  A k-tile of either
// operand is therefore ONE contiguous bulk copy (TMA engine) signalled on an mbarrier: no tensor
// maps, no swizzle bookkeeping, no LSU traffic.
//
// Persistent CTAs walk (m-tile, n-tile) pairs:
//   producer thread   3-deep ring of (A 16 KB + W BN*128 B) k-tiles, running ahead across tiles
//   2 warpgroups      64 rows each: wgmma m64nBNk16 x4 per k-tile into register accumulators, then the
//                     epilogue through a per-warpgroup shared-memory strip (64 columns at a time):
//                     bias / GELU / residual -> stores (row-major bf16, tile-image bf16 for the next
//                     GEMM, or fp32 residual stream)
// The row LayerNorm that writes the GEMMs' A images (ln_rows) is at the end of this file.
#include <algorithm>

#include "common.cuh"
#include "tc.cuh"

namespace svcb {

// 3: fp32 out = GELU(acc + bias) + res[m % res_mod] — the stem's second convolution as a GEMM over an
// im2col image, with the positional embedding (period n_ctx rows) as the addend (whisper/model.py:150-157)
// 4: bf16 out = acc + bias in the head-major QKV layout of the attention kernel (common.cuh qkv_heads_off;
//    N = 3 D, rows are items of res_mod positions each; pad rows are zeroed by the caller once)
// 5: the stem's conv1 (rows = items x res_mod frames): GELU(acc + bias) scattered straight into conv2's im2col tile
//    image A2[b * n2 + t2][j * N + co] = h1[b][co][2 t2 + j - 1] (frame t feeds (t/2, j=1) when even, ((t+1)/2, j=0)
//    and ((t-1)/2, j=2) when odd) — no h1 tensor, no im2col pass; the caller zeroes the image once (t = -1 taps, pad rows)
// 6: a stride-2 VALID convolution of the HuBERT stem feeding the next one (rows = items x res_mod frames, aux = taps of
//    the NEXT conv, 2 or 3): GELU(acc + bias) scattered into the next conv's im2col tile image
//    A[b * Tn + t2][j * N + co] = h[b][co][2 t2 + j], Tn = (res_mod - aux) / 2 + 1 (every entry of the image is written)
// 7: fp32 out[m * aux + col] = GELU(acc + bias) + res[m * aux + col] for the first res_mod columns only (aux = leading
//    dimension of out / res): one group of HuBERT's grouped positional convolution, N padded from 48 to 256
// 8: the IVF coarse search (csrc/retrieval_api.cu): f = acc + bias = |c|^2 - 2 x.c; each thread keeps the aux (= nprobe)
//    smallest (score, column) pairs of its 16 columns, ties to the lower column, and writes them as int2 {score bits,
//    column} to out[m][N / 16][aux] — the [M, N] score matrix is never stored

constexpr int GM_BM = 128, GM_BK = 64, GM_STAGES = 3;
constexpr int GM_EPI_LD = 72;   // floats per row of an epilogue strip (64 columns + 8: conflict-free fragment stores)
constexpr int GM_THREADS = 288;

// element offset of (m, k) inside a tile image with KT k-tiles per row-tile
__host__ __device__ inline size_t img_off(int m, int k, int KT) {
  return ((size_t)(m >> 7) * KT + (k >> 6)) * (GM_BM * GM_BK) + (size_t)((k & 63) >> 3) * (GM_BM * 8) + (m & 127) * 8 + (k & 7);
}

template <int BN, int EPI>
__global__ void __launch_bounds__(GM_THREADS, 1)
gemm_tc_kernel(const __nv_bfloat16* __restrict__ Aimg, const __nv_bfloat16* __restrict__ Wimg,
               const float* __restrict__ bias, void* out, const float* res, int M, int N, int K, int res_mod, int aux) {
  constexpr uint32_t A_BYTES = GM_BM * GM_BK * 2, B_BYTES = BN * GM_BK * 2, ST_BYTES = A_BYTES + B_BYTES;
  extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t bar_full[GM_STAGES], bar_empty[GM_STAGES];
  const int tid = threadIdx.x, warp = tid >> 5;
  const int KT = K / GM_BK, NT = N / BN, MT = (M + GM_BM - 1) / GM_BM;
  const int ntiles = MT * NT;

  if (tid == 0) {
    for (int s = 0; s < GM_STAGES; ++s) { tc::mbar_init(&bar_full[s], 1); tc::mbar_init(&bar_empty[s], 2); }
    tc::fence_barrier_init();
  }
  __syncthreads();

  if (tid == 256) {
    // ------------------------------------------------------------------ producer
    int kc = 0;  // global k-tile counter (ring position)
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int mt = tile / NT, nt = tile - mt * NT;
      const __nv_bfloat16* a_src = Aimg + (size_t)mt * KT * (GM_BM * GM_BK);
      const __nv_bfloat16* w_src = Wimg + (size_t)nt * KT * (BN * GM_BK);
      for (int kt = 0; kt < KT; ++kt, ++kc) {
        const int st = kc % GM_STAGES;
        if (kc >= GM_STAGES) tc::mbar_wait(&bar_empty[st], (uint32_t)(((kc / GM_STAGES) - 1) & 1));
        uint8_t* As = smem + (size_t)st * ST_BYTES;
        tc::mbar_arrive_expect_tx(&bar_full[st], ST_BYTES);
        tc::bulk_g2s(As, a_src + (size_t)kt * (GM_BM * GM_BK), A_BYTES, &bar_full[st]);
        tc::bulk_g2s(As + A_BYTES, w_src + (size_t)kt * (BN * GM_BK), B_BYTES, &bar_full[st]);
      }
    }
  } else if (warp < 8) {
    // ------------------------------------------------------------------ MMA + epilogue (warpgroup wg: rows 64 wg ..)
    const int wg = warp >> 2, t = tid & 127;
    float* strip = reinterpret_cast<float*>(smem + (size_t)GM_STAGES * ST_BYTES) + wg * 64 * GM_EPI_LD;
    const uint32_t s0 = tc::smem_u32(smem);
    const uint32_t lbo_a = GM_BM * 16u, lbo_b = BN * 16u;
    const uint64_t ks_a = (2u * lbo_a) >> 4, ks_b = (2u * lbo_b) >> 4;
    int kc = 0;
    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
      const int mt = tile / NT, nt = tile - mt * NT;
      float acc[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
      for (int kt = 0; kt < KT; ++kt, ++kc) {
        const int st = kc % GM_STAGES;
        tc::mbar_wait(&bar_full[st], (uint32_t)((kc / GM_STAGES) & 1));
        const uint32_t a0 = s0 + (uint32_t)st * ST_BYTES;
        const uint64_t ad = tc::smem_desc(a0 + (uint32_t)wg * 64u * 16u, lbo_a), bd = tc::smem_desc(a0 + A_BYTES, lbo_b);
        tc::wg_fence();
#pragma unroll
        for (int kk = 0; kk < GM_BK / 16; ++kk) tc::Wg<BN, 0>::ss(acc, ad + kk * ks_a, bd + kk * ks_b, 1u);
        tc::wg_commit();
        tc::wg_wait<1>();                   // the previous k-tile's MMAs are done: release its stage
        if (kt > 0 && t == 0) tc::mbar_arrive(&bar_empty[(kc - 1) % GM_STAGES]);
      }
      tc::wg_wait<0>();
      tc::wg_hold(acc);
      if (t == 0) tc::mbar_arrive(&bar_empty[(kc - 1) % GM_STAGES]);

      // epilogue: 64-column chunks through the strip; thread = (row t % 64, 32-column half t / 64)
      const int m = mt * GM_BM + wg * 64 + (t & 63);
      const int n0 = nt * BN;
#pragma unroll 1
      for (int ch = 0; ch < BN / 64; ++ch) {
        tc::named_sync(1 + wg, 128);        // the previous chunk has been read
        tc::acc_to_smem<BN>(acc, strip, GM_EPI_LD, 8 * ch, 8 * ch + 8);
        tc::named_sync(1 + wg, 128);
#pragma unroll 1
        for (int sub = 0; sub < 2; ++sub) {
          const int cl = (t >> 6) * 32 + sub * 16;   // column inside the chunk
          const int c0 = ch * 64 + cl;              // column inside the tile
          float v[16];
#pragma unroll
          for (int j = 0; j < 16; j += 4) {
            const float4 q = *reinterpret_cast<const float4*>(strip + (t & 63) * GM_EPI_LD + cl + j);
            v[j] = q.x; v[j + 1] = q.y; v[j + 2] = q.z; v[j + 3] = q.w;
          }
          float r16[16];
#pragma unroll
          for (int j = 0; j < 16; ++j) r16[j] = 0.f;
          if ((EPI == EPI_RESID_F32 || EPI == EPI_GELU_ADD_F32) && m < M && res) {   // (EPI_RESID_F32 without res: plain fp32 output)
            const int mr = (EPI == EPI_GELU_ADD_F32 && res_mod > 0) ? m % res_mod : m;
            const float4* rr = reinterpret_cast<const float4*>(res + (size_t)mr * N + n0 + c0);
#pragma unroll
            for (int j = 0; j < 4; ++j) { const float4 q = rr[j]; r16[4 * j] = q.x; r16[4 * j + 1] = q.y; r16[4 * j + 2] = q.z; r16[4 * j + 3] = q.w; }
          }
          if (m < M) {
            float f[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) f[j] = v[j] + (bias ? __ldg(bias + n0 + c0 + j) : 0.f);
          if (EPI == EPI_GELU_ADD_F32 || EPI == EPI_GELU_CONV2_IMG || EPI == EPI_GELU_VALID_S2_IMG || EPI == EPI_GELU_ADD_F32_LD) {
#pragma unroll
            for (int j = 0; j < 16; ++j) f[j] = 0.5f * f[j] * (1.f + erff(f[j] * 0.70710678118654752440f));
          }
          if (EPI == EPI_IVF_TOPK) {
            int2* o = static_cast<int2*>(out) + ((size_t)m * (N / 16) + (n0 + c0) / 16) * aux;
            // aux passes of an arg-min over the columns not yet written, each re-reading the strip (f[] and v[] stay
            // dead: the accumulators already hold most of the register file)
            const float* sr = strip + (t & 63) * GM_EPI_LD + cl;
            uint32_t taken = 0;
#pragma unroll 1
            for (int p = 0; p < aux; ++p) {
              float bs = 0.f;
              int bc = 16;
#pragma unroll
              for (int j = 0; j < 16; ++j) {
                const float fj = sr[j] + __ldg(bias + n0 + c0 + j);
                if (!((taken >> j) & 1u) && (bc == 16 || fj < bs)) { bs = fj; bc = j; }
              }
              taken |= 1u << bc;
              o[p] = make_int2(__float_as_int(bs), n0 + c0 + bc);
            }
          } else if (EPI == EPI_GELU_ADD_F32_LD) {
            float* o = static_cast<float*>(out) + (size_t)m * aux;
            const float* rr = res + (size_t)m * aux;
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              const int col = n0 + c0 + j;
              if (col < res_mod) o[col] = f[j] + rr[col];
            }
          } else if (EPI == EPI_RESID_F32 || EPI == EPI_GELU_ADD_F32) {
            float* o = static_cast<float*>(out) + (size_t)m * N + n0 + c0;
#pragma unroll
            for (int j = 0; j < 16; j += 4)
              *reinterpret_cast<float4*>(o + j) = make_float4(f[j] + r16[j], f[j + 1] + r16[j + 1], f[j + 2] + r16[j + 2], f[j + 3] + r16[j + 3]);
          } else {
            __align__(16) __nv_bfloat16 h[16];
#pragma unroll
            for (int j = 0; j < 16; ++j) {
              float x = f[j];
              if (EPI == EPI_GELU_BF16_IMAGE) x = 0.5f * x * (1.f + erff(x * 0.70710678118654752440f));
              h[j] = __float2bfloat16_rn(x);
            }
            if (EPI == EPI_GELU_VALID_S2_IMG) {
              __nv_bfloat16* ob = static_cast<__nv_bfloat16*>(out);
              const int nfr = res_mod, Tn = (nfr - aux) / 2 + 1, KT2 = aux * N / GM_BK;
              const int bi = m / nfr, t = m - bi * nfr;
              const uint4 q0 = *reinterpret_cast<const uint4*>(h), q1 = *reinterpret_cast<const uint4*>(h + 8);
              auto put = [&](int t2, int j) {   // frame t is tap j of output frame t2: t = 2 t2 + j
                if (t2 >= 0 && t2 < Tn) {
                  *reinterpret_cast<uint4*>(ob + img_off(bi * Tn + t2, j * N + n0 + c0, KT2)) = q0;
                  *reinterpret_cast<uint4*>(ob + img_off(bi * Tn + t2, j * N + n0 + c0 + 8, KT2)) = q1;
                }
              };
              if (t & 1) put((t - 1) >> 1, 1);
              else { put(t >> 1, 0); if (aux == 3) put((t >> 1) - 1, 2); }
            } else if (EPI == EPI_GELU_CONV2_IMG) {
              __nv_bfloat16* ob = static_cast<__nv_bfloat16*>(out);
              const int nfr = res_mod, n2 = (nfr - 1) / 2 + 1, KT2 = 3 * N / GM_BK;
              const int bi = m / nfr, t = m - bi * nfr;
              const uint4 q0 = *reinterpret_cast<const uint4*>(h), q1 = *reinterpret_cast<const uint4*>(h + 8);
              if (t & 1) {
                const int ta = (t + 1) >> 1, tb = (t - 1) >> 1;
                if (ta < n2) {
                  *reinterpret_cast<uint4*>(ob + img_off(bi * n2 + ta, n0 + c0, KT2)) = q0;
                  *reinterpret_cast<uint4*>(ob + img_off(bi * n2 + ta, n0 + c0 + 8, KT2)) = q1;
                }
                *reinterpret_cast<uint4*>(ob + img_off(bi * n2 + tb, 2 * N + n0 + c0, KT2)) = q0;
                *reinterpret_cast<uint4*>(ob + img_off(bi * n2 + tb, 2 * N + n0 + c0 + 8, KT2)) = q1;
              } else {
                *reinterpret_cast<uint4*>(ob + img_off(bi * n2 + (t >> 1), N + n0 + c0, KT2)) = q0;
                *reinterpret_cast<uint4*>(ob + img_off(bi * n2 + (t >> 1), N + n0 + c0 + 8, KT2)) = q1;
              }
            } else if (EPI == EPI_QKV_HEADS) {   // res_mod = positions per item; 16 columns = two octets of one head
              __nv_bfloat16* ob = static_cast<__nv_bfloat16*>(out);
              const int Dm = N / 3, n = n0 + c0;
              const int w = n / Dm, hd = (n - w * Dm) >> 6, d = n & 63;
              const int bi = m / res_mod, t = m - bi * res_mod;
              const size_t o = qkv_heads_off(bi, w, hd, t, d, Dm >> 6, qkv_heads_tp(res_mod));
              *reinterpret_cast<uint4*>(ob + o) = *reinterpret_cast<const uint4*>(h);
              *reinterpret_cast<uint4*>(ob + o + (w == 0 ? 1024 : 512)) = *reinterpret_cast<const uint4*>(h + 8);
            } else if (EPI == EPI_GELU_BF16_IMAGE) {  // A operand of the next GEMM
              __nv_bfloat16* ob = static_cast<__nv_bfloat16*>(out);
              *reinterpret_cast<uint4*>(ob + img_off(m, n0 + c0, N / GM_BK)) = *reinterpret_cast<const uint4*>(h);
              *reinterpret_cast<uint4*>(ob + img_off(m, n0 + c0 + 8, N / GM_BK)) = *reinterpret_cast<const uint4*>(h + 8);
            } else {
              __nv_bfloat16* o = static_cast<__nv_bfloat16*>(out) + (size_t)m * N + n0 + c0;
              *reinterpret_cast<uint4*>(o) = *reinterpret_cast<const uint4*>(h);
              *reinterpret_cast<uint4*>(o + 8) = *reinterpret_cast<const uint4*>(h + 8);
            }
          }
        }
      }
      }
    }
  }
}

template <int BN, int EPI>
static int launch_gemm_t(const __nv_bfloat16* A, const __nv_bfloat16* W, const float* bias, void* out,
                         const float* res, int M, int N, int K, int res_mod, cudaStream_t s, int aux = 0) {
  constexpr size_t smem = (size_t)GM_STAGES * (GM_BM * GM_BK * 2 + BN * GM_BK * 2) + 2 * 64 * GM_EPI_LD * 4;
  static DevSmemCache attr_cache;
  SVCB_CUDA_CHECK(ensure_dyn_smem(gemm_tc_kernel<BN, EPI>, smem, attr_cache));
  const int n_sm = device_sm_count();
  if (n_sm <= 0) { set_error("gemm_tc: cannot query the SM count"); return SVCB_E_CUDA; }
  const int ntiles = ((M + GM_BM - 1) / GM_BM) * (N / BN);
  const int grid = std::min(ntiles, n_sm);
  KernelScope ks("whisper_gemm_tc", s, 2.0 * M * (double)N * K,
                 2.0 * ((double)M * K + (double)N * K) + (EPI == EPI_RESID_F32 ? 8.0 : EPI == EPI_GELU_ADD_F32 ? 4.0 : 2.0) * M * (double)N);
  gemm_tc_kernel<BN, EPI><<<grid, GM_THREADS, smem, s>>>(A, W, bias, out, res, M, N, K, res_mod, aux);
  SVCB_LAUNCH_CHECK("gemm_tc");
  return SVCB_OK;
}

// A_img: tile image [ceil(M/128)][K/64][8][128][8]; W_img: tile image [N/256][K/64][8][256][8]
int launch_gemm_tc(const void* A_img, const void* W_img, const float* bias, void* out, const float* res,
                   int M, int N, int K, GemmEpi epi, cudaStream_t s, int res_mod, int aux) {
  if (M <= 0) return SVCB_OK;
  if (K % 64 || N % 256) { set_error("gemm_tc: need K % 64 == 0 and N % 256 == 0"); return SVCB_E_BAD_SHAPE; }
  const __nv_bfloat16* A = static_cast<const __nv_bfloat16*>(A_img);
  const __nv_bfloat16* W = static_cast<const __nv_bfloat16*>(W_img);
  switch (epi) {
    case EPI_BF16_ROWMAJOR: return launch_gemm_t<256, EPI_BF16_ROWMAJOR>(A, W, bias, out, res, M, N, K, 0, s);
    case EPI_GELU_BF16_IMAGE: return launch_gemm_t<256, EPI_GELU_BF16_IMAGE>(A, W, bias, out, res, M, N, K, 0, s);
    case EPI_RESID_F32: return launch_gemm_t<256, EPI_RESID_F32>(A, W, bias, out, res, M, N, K, 0, s);
    case EPI_GELU_CONV2_IMG:
      if (res_mod <= 0 || M % res_mod || N % GM_BK) { set_error("gemm_tc: epilogue 5 needs rows = items x res_mod frames"); return SVCB_E_BAD_SHAPE; }
      return launch_gemm_t<256, EPI_GELU_CONV2_IMG>(A, W, bias, out, res, M, N, K, res_mod, s);
    case EPI_GELU_ADD_F32_LD:
      if (!res || res_mod <= 0 || res_mod > N || aux < res_mod) { set_error("gemm_tc: epilogue 7 needs res, valid columns (res_mod) and a leading dimension (aux)"); return SVCB_E_BAD_SHAPE; }
      return launch_gemm_t<256, EPI_GELU_ADD_F32_LD>(A, W, bias, out, res, M, N, K, res_mod, s, aux);
    case EPI_GELU_VALID_S2_IMG:
      if (res_mod <= 0 || M % res_mod || N % GM_BK || (aux != 2 && aux != 3) || res_mod < aux) {
        set_error("gemm_tc: epilogue 6 needs rows = items x res_mod frames and aux = 2 or 3 taps");
        return SVCB_E_BAD_SHAPE;
      }
      return launch_gemm_t<256, EPI_GELU_VALID_S2_IMG>(A, W, bias, out, res, M, N, K, res_mod, s, aux);
    case EPI_QKV_HEADS:
      if (res_mod <= 0 || M % res_mod || N % 192) { set_error("gemm_tc: epilogue 4 needs rows = items x res_mod, N = 3 x heads x 64"); return SVCB_E_BAD_SHAPE; }
      return launch_gemm_t<256, EPI_QKV_HEADS>(A, W, bias, out, res, M, N, K, res_mod, s);
    case EPI_GELU_ADD_F32:
      return launch_gemm_t<256, EPI_GELU_ADD_F32>(A, W, bias, out, res, M, N, K, res_mod, s);
    default:   // (EPI_IVF_TOPK has its own launcher, launch_ivf_coarse_tc)
      set_error("gemm_tc: unknown epilogue");
      return SVCB_E_BAD_SHAPE;
  }
}

// IVF coarse search (epilogue 8): cand[M][N/16][nprobe] int2 {score bits, column}, score = cnorm[col] - 2 x.c
int launch_ivf_coarse_tc(const void* A_img, const void* W_img, const float* cnorm, void* cand, int M, int N, int K, int nprobe,
                         cudaStream_t s) {
  if (M <= 0) return SVCB_OK;
  if (K % 64 || N % 256 || nprobe < 1 || nprobe > 8) { set_error("ivf_coarse_tc: need K % 64 == 0, N % 256 == 0, 1 <= nprobe <= 8"); return SVCB_E_BAD_SHAPE; }
  constexpr size_t smem = (size_t)GM_STAGES * (GM_BM * GM_BK * 2 + 256 * GM_BK * 2) + 2 * 64 * GM_EPI_LD * 4;
  static DevSmemCache attr_cache;
  SVCB_CUDA_CHECK(ensure_dyn_smem(gemm_tc_kernel<256, EPI_IVF_TOPK>, smem, attr_cache));
  const int n_sm = device_sm_count();
  if (n_sm <= 0) { set_error("ivf_coarse_tc: cannot query the SM count"); return SVCB_E_CUDA; }
  const int ntiles = ((M + GM_BM - 1) / GM_BM) * (N / 256);
  // algorithmic FLOPs of the fp32 search (K = 3 d holds the three bf16 split products)
  KernelScope ks("ivf_coarse_tc", s, 2.0 * M * (double)N * (K / 3),
                 2.0 * ((double)M * K + (double)N * K) + 4.0 * N + 8.0 * M * (double)(N / 16) * nprobe);
  gemm_tc_kernel<256, EPI_IVF_TOPK><<<std::min(ntiles, n_sm), GM_THREADS, smem, s>>>(
      static_cast<const __nv_bfloat16*>(A_img), static_cast<const __nv_bfloat16*>(W_img), cnorm, cand, nullptr, M, N, K, 0, nprobe);
  SVCB_LAUNCH_CHECK("ivf_coarse_tc");
  return SVCB_OK;
}

// The coarse search's A operand: query rows x [M, d] fp32 -> bf16 tile image [ceil(M/128) * 128][3 d] holding
// [x_hi | x_lo | x_hi] (x_hi = bf16(x), x_lo = bf16(x - x_hi)), rows past M zero.  With the centroid image
// [-2 c_hi | -2 c_hi | -2 c_lo] one bf16 GEMM over K = 3 d gives -2 (x_hi c_hi + x_lo c_hi + x_hi c_lo): bf16x3.
// Thread = one (row, octet of x), consecutive threads on consecutive rows: the image holds the octets of 128 rows
// contiguously, so a warp's stores are 512 contiguous bytes (row-major threads spread them 2 KB apart).
__global__ void __launch_bounds__(256)
ivf_pack_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ img, int M, int Mp, int d) {
  const int no = d / 8;
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)Mp * no) return;
  const int o = (int)(idx / Mp), m = (int)(idx - (size_t)o * Mp), k = o * 8;
  __align__(16) __nv_bfloat16 hi[8], lo[8];
  if (m < M) {
    const float4* s4 = reinterpret_cast<const float4*>(x + (size_t)m * d + k);
    const float4 u0 = __ldg(s4), u1 = __ldg(s4 + 1);
    const float v[8] = {u0.x, u0.y, u0.z, u0.w, u1.x, u1.y, u1.z, u1.w};
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      hi[e] = __float2bfloat16_rn(v[e]);
      lo[e] = __float2bfloat16_rn(v[e] - __bfloat162float(hi[e]));
    }
  } else {
#pragma unroll
    for (int e = 0; e < 8; ++e) { hi[e] = __float2bfloat16_rn(0.f); lo[e] = hi[e]; }
  }
  const int KT = 3 * d / GM_BK;
  const uint4 qh = *reinterpret_cast<const uint4*>(hi), ql = *reinterpret_cast<const uint4*>(lo);
  *reinterpret_cast<uint4*>(img + img_off(m, k, KT)) = qh;
  *reinterpret_cast<uint4*>(img + img_off(m, d + k, KT)) = ql;
  *reinterpret_cast<uint4*>(img + img_off(m, 2 * d + k, KT)) = qh;
}

int launch_ivf_pack(const float* x, void* img, int M, int d, cudaStream_t s) {
  if (M <= 0) return SVCB_OK;
  if (d % 64) { set_error("ivf_pack: d must be a multiple of 64"); return SVCB_E_BAD_SHAPE; }
  const int Mp = (M + GM_BM - 1) / GM_BM * GM_BM;
  const size_t n = (size_t)Mp * (d / 8);
  KernelScope ks("ivf_pack", s, 0.0, 4.0 * M * (double)d + 6.0 * Mp * (double)d);
  ivf_pack_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(x, static_cast<__nv_bfloat16*>(img), M, Mp, d);
  SVCB_LAUNCH_CHECK("ivf_pack");
  return SVCB_OK;
}

// Stem conv2 (Conv1d(D, D, k=3, stride 2, pad 1), whisper/model.py:150) as a GEMM: this kernel builds
// the A tile image of its im2col matrix, A[m = b*n2 + t2][k = j*D + ci] = h1[b][ci][2*t2 + j - 1]
// (zero outside the sequence and in the rows that pad M to whole 128-row tiles), bf16.
// One CTA = one (row tile, k tile): a k tile of 64 lies inside one tap j because D % 64 == 0.
__global__ void __launch_bounds__(256)
im2col_s2_image_kernel(const float* __restrict__ h1, __nv_bfloat16* __restrict__ img, int D, int n, int n2, int M, int taps,
                       int pad) {
  __shared__ float tile[64][129];
  const int mt = blockIdx.x, kt = blockIdx.y, tid = threadIdx.x;
  const int j = (kt * 64) / D, ci0 = (kt * 64) % D;
  for (int idx = tid; idx < 64 * 128; idx += 256) {
    const int cc = idx >> 7, r = idx & 127;
    const int m = mt * 128 + r;
    float v = 0.f;
    if (m < M) {
      const int b = m / n2, t2 = m - b * n2;
      const int t = 2 * t2 + j - pad;
      if (t >= 0 && t < n) v = __ldg(h1 + ((size_t)b * D + ci0 + cc) * n + t);
    }
    tile[cc][r] = v;
  }
  __syncthreads();
  const int KT = taps * D / 64;
  __nv_bfloat16* dst = img + ((size_t)mt * KT + kt) * (GM_BM * GM_BK);
  for (int idx = tid; idx < 8 * 128; idx += 256) {
    const int kc = idx >> 7, r = idx & 127;
    __align__(16) __nv_bfloat16 h[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = __float2bfloat16_rn(tile[kc * 8 + e][r]);
    *reinterpret_cast<uint4*>(dst + (size_t)(kc * 128 + r) * 8) = *reinterpret_cast<const uint4*>(h);
  }
}

// Stem conv1 (Conv1d(n_mels, D, k=3, pad 1), whisper/model.py:149) as a GEMM: the A tile image of ITS im2col matrix,
// A[m = b*n + t][k = j*n_mels + ci] = mel[b][ci][t + j - 1], zero outside the sequence, for k >= 3 n_mels (K padded
// to 64) and in the rows that pad M to whole tiles.  One CTA = one (row tile, k tile).
__global__ void __launch_bounds__(256)
im2col_s1_image_kernel(const float* __restrict__ mel, __nv_bfloat16* __restrict__ img, int nm, int n, int M, int KT) {
  __shared__ float tile[64][129];
  const int mt = blockIdx.x, kt = blockIdx.y, tid = threadIdx.x;
  for (int idx = tid; idx < 64 * 128; idx += 256) {
    const int cc = idx >> 7, r = idx & 127;
    const int m = mt * 128 + r, k = kt * 64 + cc;
    float v = 0.f;
    if (m < M && k < 3 * nm) {
      const int b = m / n, t1 = m - b * n;
      const int j = k / nm, ci = k - j * nm;
      const int t = t1 + j - 1;
      if (t >= 0 && t < n) v = __ldg(mel + ((size_t)b * nm + ci) * n + t);
    }
    tile[cc][r] = v;
  }
  __syncthreads();
  __nv_bfloat16* dst = img + ((size_t)mt * KT + kt) * (GM_BM * GM_BK);
  for (int idx = tid; idx < 8 * 128; idx += 256) {
    const int kc = idx >> 7, r = idx & 127;
    __align__(16) __nv_bfloat16 h[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = __float2bfloat16_rn(tile[kc * 8 + e][r]);
    *reinterpret_cast<uint4*>(dst + (size_t)(kc * 128 + r) * 8) = *reinterpret_cast<const uint4*>(h);
  }
}

int launch_im2col_s1_image(const float* mel, void* img, int B, int n_mels, int n, cudaStream_t s) {
  const int M = B * n, KT = (3 * n_mels + 63) / 64;
  dim3 grid((M + 127) / 128, KT);
  KernelScope ks("im2col_s1_image", s, 0.0, (double)M * KT * 64 * 2 + 4.0 * B * n_mels * (double)n * 3);
  im2col_s1_image_kernel<<<grid, 256, 0, s>>>(mel, static_cast<__nv_bfloat16*>(img), n_mels, n, M, KT);
  SVCB_LAUNCH_CHECK("im2col_s1_image");
  return SVCB_OK;
}

// HuBERT's positional convolution (Conv1d(768, 768, 128, padding 64, groups 16), hubert_model.py:115-121), one group:
// A[m = b*T + t][k = j*cg + ci] = x[b*T + t + j - pad][c0 + ci] from the fp32 time-major rows x [B*T, ld] (zero outside
// the item), cg = 48 channels per group = 6 octets per tap, K = taps * cg.  One CTA = one (row tile, k tile).
__global__ void __launch_bounds__(256)
im2col_rows_image_kernel(const float* __restrict__ x, __nv_bfloat16* __restrict__ img, int T, int M, int ld, int c0, int cg,
                         int pad, int KT) {
  const int mt = blockIdx.x, kt = blockIdx.y, opt = cg / 8;   // octets per tap
  __nv_bfloat16* dst = img + ((size_t)mt * KT + kt) * (GM_BM * GM_BK);
  for (int idx = threadIdx.x; idx < 8 * 128; idx += 256) {
    const int kc = idx >> 7, r = idx & 127;
    const int m = mt * 128 + r, o = kt * 8 + kc;   // global octet index along K
    const int j = o / opt, ci = (o - j * opt) * 8;
    __align__(16) __nv_bfloat16 h[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) h[e] = __float2bfloat16_rn(0.f);
    if (m < M) {
      const int b = m / T, t = m - b * T + j - pad;
      if (t >= 0 && t < T) {
        const float4* s4 = reinterpret_cast<const float4*>(x + ((size_t)b * T + t) * ld + c0 + ci);
        const float4 u0 = __ldg(s4), u1 = __ldg(s4 + 1);
        h[0] = __float2bfloat16_rn(u0.x); h[1] = __float2bfloat16_rn(u0.y); h[2] = __float2bfloat16_rn(u0.z); h[3] = __float2bfloat16_rn(u0.w);
        h[4] = __float2bfloat16_rn(u1.x); h[5] = __float2bfloat16_rn(u1.y); h[6] = __float2bfloat16_rn(u1.z); h[7] = __float2bfloat16_rn(u1.w);
      }
    }
    *reinterpret_cast<uint4*>(dst + (size_t)(kc * 128 + r) * 8) = *reinterpret_cast<const uint4*>(h);
  }
}

int launch_im2col_rows_image(const float* x, void* img, int B, int T, int ld, int c0, int cg, int taps, int pad, cudaStream_t s) {
  if (cg % 8 || (taps * cg) % 64 || (c0 % 4) || (ld % 4)) { set_error("im2col_rows_image: channel group must be octets, K a multiple of 64"); return SVCB_E_BAD_SHAPE; }
  const int M = B * T, KT = taps * cg / 64;
  dim3 grid((M + 127) / 128, KT);
  KernelScope ks("im2col_rows_image", s, 0.0, (double)M * taps * cg * 2 + 4.0 * M * cg);
  im2col_rows_image_kernel<<<grid, 256, 0, s>>>(x, static_cast<__nv_bfloat16*>(img), T, M, ld, c0, cg, pad, KT);
  SVCB_LAUNCH_CHECK("im2col_rows_image");
  return SVCB_OK;
}

// taps / pad: 3 / 1 for Whisper's conv2; 3 / 0 for the first stride-2 conv of the HuBERT stem (valid convolution)
int launch_im2col_s2_image(const float* h1, void* img, int B, int D, int n, int n2, cudaStream_t s, int taps, int pad) {
  if (D % 64) { set_error("im2col_s2_image: D must be a multiple of 64"); return SVCB_E_BAD_SHAPE; }
  const int M = B * n2;
  dim3 grid((M + 127) / 128, taps * D / 64);
  KernelScope ks("im2col_s2_image", s, 0.0, (double)M * taps * D * 2 + 4.0 * B * D * (double)n);
  im2col_s2_image_kernel<<<grid, 256, 0, s>>>(h1, static_cast<__nv_bfloat16*>(img), D, n, n2, M, taps, pad);
  SVCB_LAUNCH_CHECK("im2col_s2_image");
  return SVCB_OK;
}

// row-major bf16 [R,K] -> tile image with `rows` rows per tile (128 for A, 256 for W); used by the
// unit-test entry point — the encoder's kernels write A images directly and the host packs W.
__global__ void rowmajor_to_image_kernel(const __nv_bfloat16* __restrict__ src, __nv_bfloat16* __restrict__ dst,
                                         int R, int K, int rows) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // one 16-byte chunk each
  const int kc_per_row = K / 8;
  if (idx >= (size_t)R * kc_per_row) return;
  const int m = (int)(idx / kc_per_row), k = (int)(idx % kc_per_row) * 8;
  const size_t off = ((size_t)(m / rows) * (K / GM_BK) + (k >> 6)) * ((size_t)rows * GM_BK) +
                     (size_t)((k & 63) >> 3) * (rows * 8) + (size_t)(m % rows) * 8;
  *reinterpret_cast<uint4*>(dst + off) = *reinterpret_cast<const uint4*>(src + (size_t)m * K + k);
}

int launch_rowmajor_to_image(const void* src, void* dst, int R, int K, int rows, cudaStream_t s) {
  const size_t n = (size_t)R * (K / 8);
  rowmajor_to_image_kernel<<<(unsigned)((n + 255) / 256), 256, 0, s>>>(static_cast<const __nv_bfloat16*>(src),
                                                                       static_cast<__nv_bfloat16*>(dst), R, K, rows);
  SVCB_LAUNCH_CHECK("rowmajor_to_image");
  return SVCB_OK;
}

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}

// Row LayerNorm over the last dim of fp32 [M, D] (nn.LayerNorm, eps 1e-5; whisper/model.py:28-31):
// one warp per row, values held in registers, output bf16 (GEMM operand) or fp32 (ln_post).
template <bool OUT_BF16>
__global__ void __launch_bounds__(256)
ln_rows_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
               void* __restrict__ y, float* __restrict__ y32, int M, int D, float eps) {
  // bf16 output: the 8 rows of the block are staged in shared memory and leave as whole 128-byte lines of the tile
  // image (8 rows x one 16-byte octet are contiguous there); lane-wise 8-byte stores into the image touched 16
  // half-filled sectors per instruction and held the kernel at 2.2 TB/s
  extern __shared__ __align__(16) uint8_t ln_stage[];
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const bool live = row < M;
  if (!OUT_BF16 && !live) return;
  const float* xr = x + (size_t)(live ? row : M - 1) * D;
  const int srow = (D + 8) * 2;   // bytes per staged row (+16: conflict-free 16-byte reads down a column of rows)
  constexpr int MAXV = 16;  // D <= 32*4*16 = 2048
  float4 v[MAXV];
  const int nv = D / 128;  // float4 per lane
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (i < nv) {
      v[i] = *reinterpret_cast<const float4*>(xr + (size_t)(i * 32 + lane) * 4);
      s += v[i].x + v[i].y + v[i].z + v[i].w;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  const float mean = s / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (i < nv) {
      const float a = v[i].x - mean, b2 = v[i].y - mean, c = v[i].z - mean, d = v[i].w - mean;
      q += a * a + b2 * b2 + c * c + d * d;
    }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) q += __shfl_xor_sync(0xffffffffu, q, off);
  const float rstd = 1.f / sqrtf(q / (float)D + eps);
#pragma unroll
  for (int i = 0; i < MAXV; ++i) {
    if (i < nv) {
      const int c0 = (i * 32 + lane) * 4;
      const float4 gm = *reinterpret_cast<const float4*>(gamma + c0);
      const float4 bt = *reinterpret_cast<const float4*>(beta + c0);
      const float o0 = (v[i].x - mean) * rstd * gm.x + bt.x, o1 = (v[i].y - mean) * rstd * gm.y + bt.y;
      const float o2 = (v[i].z - mean) * rstd * gm.z + bt.z, o3 = (v[i].w - mean) * rstd * gm.w + bt.w;
      if (OUT_BF16) {  // GEMM tile image (A operand of the following linear layer), through the staging rows
        // (+ the fp32 rows when the normalised values are also the residual stream: post-LN layers, HuBERT)
        if (y32 && live) *reinterpret_cast<float4*>(y32 + (size_t)row * D + c0) = make_float4(o0, o1, o2, o3);
        uint2 pk = make_uint2(pack_bf16(o0, o1), pack_bf16(o2, o3));
        *reinterpret_cast<uint2*>(ln_stage + (size_t)(threadIdx.x >> 5) * srow + (size_t)c0 * 2) = pk;
      } else {
        *reinterpret_cast<float4*>(static_cast<float*>(y) + (size_t)row * D + c0) = make_float4(o0, o1, o2, o3);
      }
    }
  }
  if (OUT_BF16) {
    __syncthreads();
    const int row0 = blockIdx.x * 8, noct = D / 8;
    for (int idx = threadIdx.x; idx < noct * 8; idx += 256) {
      const int o = idx >> 3, r = idx & 7;
      if (row0 + r < M)
        *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(y) + img_off(row0 + r, o * 8, D / 64)) =
            *reinterpret_cast<const uint4*>(ln_stage + (size_t)r * srow + (size_t)o * 16);
    }
  }
}

// y32 (bf16 mode only, a buffer other than x): the same normalised rows in fp32 [M, D]
int launch_ln_rows(const float* x, const float* gamma, const float* beta, void* y, int M, int D, bool out_bf16,
                   cudaStream_t s, float* y32) {
  if (D % 128 || D > 2048) { set_error("ln_rows: D must be a multiple of 128 and <= 2048"); return SVCB_E_UNSUPPORTED; }
  KernelScope ks("ln_rows", s, 8.0 * M * (double)D, (out_bf16 ? (y32 ? 10.0 : 6.0) : 8.0) * M * (double)D);
  if (out_bf16) ln_rows_kernel<true><<<(M + 7) / 8, 256, (size_t)8 * (D + 8) * 2, s>>>(x, gamma, beta, y, y32, M, D, 1e-5f);
  else ln_rows_kernel<false><<<(M + 7) / 8, 256, 0, s>>>(x, gamma, beta, y, nullptr, M, D, 1e-5f);
  SVCB_LAUNCH_CHECK("ln_rows");
  return SVCB_OK;
}

}  // namespace svcb

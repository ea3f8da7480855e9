// Whisper encoder: flash-style multi-head self-attention (head dim 64, no mask) and the row
// LayerNorm that feeds the GEMMs.
//
// Replaces MultiHeadAttention.qkv_attention (whisper/model.py:88-101): q,k scaled by d^-1/4 each
// (= scores * d^-1/2), softmax in fp32, w @ v — without materialising the [B,20,T,T] score tensor.
// bf16 mma.sync (m16n8k16) tiles, fp32 online softmax; one CTA = 64 queries of one head, 4 warps x
// 16 rows; K/V tiles of 64 keys double-buffered with cp.async in an XOR-swizzled layout that keeps
// ldmatrix conflict-free.  Round 1's encoder ran this kernel (247 TFLOP/s); since round 2 the encoder and HuBERT use the
// wgmma kernel of whisper_attn_tc.cu and this one only backs the unit-test entry point `svcb_op_attention_bf16`
// (an independent implementation the wgmma kernel is also compared with).
#include "common.cuh"
#include "tc.cuh"

namespace svcb {

constexpr int FA_BQ = 64, FA_BK = 64, FA_D = 64;

__device__ __forceinline__ uint32_t swz(int row, int chunk) {  // byte offset inside a [rows][128 B] tile
  return (uint32_t)row * 128u + (uint32_t)((chunk ^ (row & 7)) << 4);
}
__device__ __forceinline__ void ldsm_x4(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x4_t(uint32_t addr, uint32_t& r0, uint32_t& r1, uint32_t& r2, uint32_t& r3) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r0), "=r"(r1), "=r"(r2), "=r"(r3) : "r"(addr));
}
__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint32_t b0, uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.bf16.bf16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&v);
}
__device__ __forceinline__ void cp16(uint32_t dst, const void* src, bool valid) {
  const int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(dst), "l"(src), "r"(sz) : "memory");
}

__device__ __forceinline__ size_t gemm_img_off(int m, int k, int KT) {  // = whisper_gemm.cu:img_off
  return ((size_t)(m >> 7) * KT + (k >> 6)) * 8192 + (size_t)((k & 63) >> 3) * 1024 + (m & 127) * 8 + (k & 7);
}

// qkv: bf16 [B*T, 3*D] rows = (q | k | v); out: bf16 [B*T, D] row-major, or (img != 0) the GEMM tile
// image of the same matrix (A operand of the out-projection)
__global__ void __launch_bounds__(128)
whisper_attention_kernel(const __nv_bfloat16* __restrict__ qkv, __nv_bfloat16* __restrict__ out, int T, int D,
                         int img) {
  __shared__ __align__(128) uint8_t sQ[FA_BQ * 128];
  __shared__ __align__(128) uint8_t sKV[2][2][FA_BK * 128];  // [stage][k|v]
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int q0 = blockIdx.x * FA_BQ, h = blockIdx.y, b = blockIdx.z;
  const size_t row_stride = (size_t)3 * D;
  const __nv_bfloat16* base = qkv + (size_t)b * T * row_stride + (size_t)h * FA_D;
  const uint32_t sq = tc::smem_u32(sQ);
  const uint32_t skv[2][2] = {{tc::smem_u32(sKV[0][0]), tc::smem_u32(sKV[0][1])},
                              {tc::smem_u32(sKV[1][0]), tc::smem_u32(sKV[1][1])}};

  auto load_tile = [&](uint32_t dst, int row0, int col_off) {  // 64 rows x 8 chunks, 4 per thread
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = tid + 128 * i, r = c >> 3, ch = c & 7;
      const int gr = row0 + r;
      const bool ok = gr < T;
      cp16(dst + swz(r, ch), base + (size_t)(ok ? gr : 0) * row_stride + col_off + ch * 8, ok);
    }
  };
  load_tile(sq, q0, 0);
  load_tile(skv[0][0], 0, D);
  load_tile(skv[0][1], 0, 2 * D);
  asm volatile("cp.async.commit_group;" ::: "memory");

  const int nt = (T + FA_BK - 1) / FA_BK;
  const int g = lane >> 2, t4 = lane & 3;
  uint32_t qf[4][4];
  float o[8][4];
#pragma unroll
  for (int j = 0; j < 8; ++j) { o[j][0] = o[j][1] = o[j][2] = o[j][3] = 0.f; }
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};
  const float sl2 = 0.125f * 1.4426950408889634f;  // d^-1/2 * log2(e)

  for (int it = 0; it < nt; ++it) {
    const int st = it & 1;
    if (it + 1 < nt) {
      load_tile(skv[st ^ 1][0], (it + 1) * FA_BK, D);
      load_tile(skv[st ^ 1][1], (it + 1) * FA_BK, 2 * D);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 1;" ::: "memory");
    __syncthreads();
    if (it == 0) {
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int r = warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1), ch = 2 * ks + (lane >> 4);
        ldsm_x4(sq + swz(r, ch), qf[ks][0], qf[ks][1], qf[ks][2], qf[ks][3]);
      }
    }
    // ---- S = Q K^T  (16 x 64 per warp)
    float s[8][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) { s[j][0] = s[j][1] = s[j][2] = s[j][3] = 0.f; }
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
      for (int np = 0; np < 4; ++np) {  // pairs of 8-key blocks
        uint32_t b0, b1, b2, b3;
        const int r = np * 16 + (lane & 7) + 8 * (lane >> 4), ch = 2 * ks + ((lane >> 3) & 1);
        ldsm_x4(skv[st][0] + swz(r, ch), b0, b1, b2, b3);
        mma16816(s[2 * np], qf[ks], b0, b1);
        mma16816(s[2 * np + 1], qf[ks], b2, b3);
      }
    }
    // ---- mask keys beyond T, online softmax (rows g and g+8 of this warp's 16)
    const int kbase = it * FA_BK;
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int j = 0; j < 8; ++j) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kbase + 8 * j + 2 * t4 + (e & 1);
        if (key >= T) s[j][e] = -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[j][e]);
      }
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 1));
      mx[r] = fmaxf(mx[r], __shfl_xor_sync(0xffffffffu, mx[r], 2));
    }
    float alpha[2], msc[2], rs[2] = {0.f, 0.f};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      const float m_new = fmaxf(m_run[r], mx[r]);
      alpha[r] = exp2f((m_run[r] - m_new) * sl2);
      m_run[r] = m_new;
      msc[r] = m_new * sl2;
    }
    uint32_t pf[4][4];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float p0 = exp2f(fmaf(s[j][0], sl2, -msc[0])), p1 = exp2f(fmaf(s[j][1], sl2, -msc[0]));
      const float p2 = exp2f(fmaf(s[j][2], sl2, -msc[1])), p3 = exp2f(fmaf(s[j][3], sl2, -msc[1]));
      rs[0] += p0 + p1; rs[1] += p2 + p3;
      pf[j >> 1][(j & 1) * 2 + 0] = pack_bf16(p0, p1);
      pf[j >> 1][(j & 1) * 2 + 1] = pack_bf16(p2, p3);
    }
#pragma unroll
    for (int r = 0; r < 2; ++r) {
      rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 1);
      rs[r] += __shfl_xor_sync(0xffffffffu, rs[r], 2);
      l_run[r] = l_run[r] * alpha[r] + rs[r];
    }
#pragma unroll
    for (int j = 0; j < 8; ++j) { o[j][0] *= alpha[0]; o[j][1] *= alpha[0]; o[j][2] *= alpha[1]; o[j][3] *= alpha[1]; }
    // ---- O += P V
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {    // 16 keys per step
#pragma unroll
      for (int dp = 0; dp < 4; ++dp) {  // pairs of 8-wide d blocks
        uint32_t b0, b1, b2, b3;
        const int r = ks * 16 + (lane & 7) + 8 * ((lane >> 3) & 1), ch = 2 * dp + (lane >> 4);
        ldsm_x4_t(skv[st][1] + swz(r, ch), b0, b1, b2, b3);
        mma16816(o[2 * dp], pf[ks], b0, b1);
        mma16816(o[2 * dp + 1], pf[ks], b2, b3);
      }
    }
    __syncthreads();
  }
  // ---- normalise and store
  const float inv0 = 1.f / l_run[0], inv1 = 1.f / l_run[1];
  const int r0 = q0 + warp * 16 + g, r1 = r0 + 8;
  if (img) {
    const int KT = D / 64;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = h * FA_D + 8 * j + 2 * t4;
      if (r0 < T) *reinterpret_cast<uint32_t*>(out + gemm_img_off(b * T + r0, col, KT)) = pack_bf16(o[j][0] * inv0, o[j][1] * inv0);
      if (r1 < T) *reinterpret_cast<uint32_t*>(out + gemm_img_off(b * T + r1, col, KT)) = pack_bf16(o[j][2] * inv1, o[j][3] * inv1);
    }
  } else {
    __nv_bfloat16* ob = out + (size_t)b * T * D + (size_t)h * FA_D;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int col = 8 * j + 2 * t4;
      if (r0 < T) *reinterpret_cast<uint32_t*>(ob + (size_t)r0 * D + col) = pack_bf16(o[j][0] * inv0, o[j][1] * inv0);
      if (r1 < T) *reinterpret_cast<uint32_t*>(ob + (size_t)r1 * D + col) = pack_bf16(o[j][2] * inv1, o[j][3] * inv1);
    }
  }
}

int launch_whisper_attention(const void* qkv_bf16, void* out_bf16, int B, int T, int D, int heads, int img,
                             cudaStream_t s) {
  if (D % heads || D / heads != FA_D) { set_error("whisper_attention: head dim must be 64"); return SVCB_E_UNSUPPORTED; }
  dim3 grid((T + FA_BQ - 1) / FA_BQ, heads, B);
  KernelScope ks("whisper_attention", s, 4.0 * B * heads * (double)T * T * FA_D, 2.0 * 4.0 * B * (double)T * D);
  whisper_attention_kernel<<<grid, 128, 0, s>>>(static_cast<const __nv_bfloat16*>(qkv_bf16),
                                                static_cast<__nv_bfloat16*>(out_bf16), T, D, img);
  SVCB_LAUNCH_CHECK("whisper_attention");
  return SVCB_OK;
}

// ---------------------------------------------------------------------------------------------
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
        *reinterpret_cast<uint4*>(static_cast<__nv_bfloat16*>(y) + gemm_img_off(row0 + r, o * 8, D / 64)) =
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

// Self-test of the wgmma plumbing in tc.cuh: one 128 x N x K bf16 GEMM tile with a row-shifted A
// descriptor (the convolution-tap trick), exposed as svcb_op_tc_gemm_selftest for the GPU tests.
#include "common.cuh"
#include "tc.cuh"

namespace svcb {

// one warpgroup; the two 64-row halves of the tile one after the other
template <int N>
__global__ void __launch_bounds__(128)
tc_gemm_selftest_kernel(const __nv_bfloat16* __restrict__ A, const __nv_bfloat16* __restrict__ Bm,
                        float* __restrict__ D, int R, int K, int shift) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int KC = K / 8;
  uint8_t* As = smem;                         // [KC][R][16 B]
  uint8_t* Bs = smem + (size_t)KC * R * 16;   // [KC][N][16 B]
  const int tid = threadIdx.x, w = tid >> 5, l = tid & 31;
  for (int idx = tid; idx < KC * R; idx += 128) {
    const int r = idx % R, kc = idx / R;
    *reinterpret_cast<uint4*>(As + ((size_t)kc * R + r) * 16) =
        *reinterpret_cast<const uint4*>(A + (size_t)r * K + kc * 8);
  }
  for (int idx = tid; idx < KC * N; idx += 128) {
    const int n = idx % N, kc = idx / N;
    *reinterpret_cast<uint4*>(Bs + ((size_t)kc * N + n) * 16) =
        *reinterpret_cast<const uint4*>(Bm + (size_t)n * K + kc * 8);
  }
  tc::fence_proxy_async_smem();
  __syncthreads();
  const uint32_t a0 = tc::smem_u32(As), b0 = tc::smem_u32(Bs);
  for (int half = 0; half < 2; ++half) {
    float d[N / 2];
#pragma unroll
    for (int i = 0; i < N / 2; ++i) d[i] = 0.f;
    tc::wg_fence();
    tc::wg_mma_k<N>(d, a0 + (uint32_t)(half * 64 + shift) * 16u, (uint32_t)R * 16u, b0, (uint32_t)N * 16u, K / 16, 0u);
    tc::wg_commit();
    tc::wg_wait<0>();
    tc::wg_hold(d);
    const int r = half * 64 + 16 * w + (l >> 2);
#pragma unroll
    for (int i = 0; i < N / 8; ++i) {
      const int c = 8 * i + 2 * (l & 3);
      *reinterpret_cast<float2*>(D + (size_t)r * N + c) = make_float2(d[4 * i], d[4 * i + 1]);
      *reinterpret_cast<float2*>(D + (size_t)(r + 8) * N + c) = make_float2(d[4 * i + 2], d[4 * i + 3]);
    }
  }
}

template <int N>
static int launch_selftest_n(const __nv_bfloat16* A, const __nv_bfloat16* Bm, float* D, int R, int K, int shift, size_t smem,
                             cudaStream_t s) {
  SVCB_CUDA_CHECK(cudaFuncSetAttribute(tc_gemm_selftest_kernel<N>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
  tc_gemm_selftest_kernel<N><<<1, 128, smem, s>>>(A, Bm, D, R, K, shift);
  SVCB_LAUNCH_CHECK("tc_gemm_selftest");
  return SVCB_OK;
}

}  // namespace svcb

extern "C" int svcb_op_tc_gemm_selftest(const void* A_bf16, const void* B_bf16, float* D, int32_t R,
                                        int32_t N, int32_t K, int32_t shift, svcb_stream stream) {
  using namespace svcb;
  if (N % 16 || N < 16 || N > 256 || K % 16 || R < 128 + shift || shift < 0) {
    set_error("tc_gemm_selftest: need N%16==0, 16<=N<=256, K%16==0, R>=128+shift");
    return SVCB_E_BAD_SHAPE;
  }
  const size_t smem = (size_t)(K / 8) * (R + N) * 16;
  if (smem > 200 * 1024) { set_error("tc_gemm_selftest: tile too large"); return SVCB_E_BAD_SHAPE; }
  const auto* A = static_cast<const __nv_bfloat16*>(A_bf16);
  const auto* Bm = static_cast<const __nv_bfloat16*>(B_bf16);
  const cudaStream_t s = static_cast<cudaStream_t>(stream);
  switch (N / 16) {
#define SVCB_SELFTEST_N(nb) case nb: return launch_selftest_n<16 * nb>(A, Bm, D, R, K, shift, smem, s);
    SVCB_SELFTEST_N(1) SVCB_SELFTEST_N(2) SVCB_SELFTEST_N(3) SVCB_SELFTEST_N(4) SVCB_SELFTEST_N(5) SVCB_SELFTEST_N(6)
    SVCB_SELFTEST_N(7) SVCB_SELFTEST_N(8) SVCB_SELFTEST_N(9) SVCB_SELFTEST_N(10) SVCB_SELFTEST_N(11) SVCB_SELFTEST_N(12)
    SVCB_SELFTEST_N(13) SVCB_SELFTEST_N(14) SVCB_SELFTEST_N(15) SVCB_SELFTEST_N(16)
#undef SVCB_SELFTEST_N
  }
  return SVCB_E_BAD_SHAPE;
}

// Lloyd k-means for building IVF-Flat indexes: replaces faiss's Clustering::train and IndexIVF::add (faiss 1.7.4
// Clustering.cpp, IndexIVF.cpp) as driven by feature_retrieval/index.py:122-154 (`train`, `add`), and the
// MiniBatchKMeans compression of feature_retrieval/transform.py:29-53.
//
//   km_pack        centroids [k, d] -> the coarse search's W image [-2 c_hi | -2 c_hi | -2 c_lo] and |c|^2 (pack_ivf's
//                  layout; the norms are summed in fp64 and rounded once, as pack_ivf does)
//   assignment     per chunk of rows: ivf_pack, ivf_coarse_tc (gemm_tc epilogue 8, nprobe 1), then km_argmin: one warp
//                  per row merges the per-16-column winners, ties to the lower centroid, and forms faiss's distance
//                  max(|x|^2 + |c|^2 - 2 x.c, 0) with x.c recomputed in fp32 for the chosen centroid.  The same instructions as svcb_ivf_retrieve's coarse search, so a
//                  row's centroid is the list that search probes first, whatever n, the chunk or the row's position.
//   update         a stable counting sort of the rows by centroid (per-tile counts, a per-centroid scan over the tiles,
//                  the bucket offsets, a warp-per-tile scatter ranked with __match_any_sync), then each centroid as
//                  the fp32 sum of its rows in ascending row order times 1 / count, as faiss's compute_centroids
//   km_split       faiss's split_clusters perturbation for (empty, split) pairs chosen on the host
// Every result is bitwise reproducible: no floating-point value depends on the order atomics land in.
#include <cuda_bf16.h>

#include <algorithm>
#include <cstdint>

#include "common.cuh"

namespace svcb {

constexpr int KM_MAX_D = 2048, KM_DEFAULT_CHUNK = 16384;
constexpr int KM_CENTROID_THREADS = 128, KM_CENTROID_COLS = KM_MAX_D / KM_CENTROID_THREADS;
constexpr int64_t KM_TILE_COUNTS = 1 << 22;   // bound on the per-tile count table (ints)

__device__ __forceinline__ bool km_less(float s, int c, float bs, int bc) { return s < bs || (s == bs && c < bc); }

// centroids [k, d] -> wimg: bf16 tile image [Np/256][3d/64][8][256][8] of [-2 c_hi | -2 c_hi | -2 c_lo], rows past k
// zero.  Thread = (row, octet), consecutive threads on consecutive rows (contiguous 16-byte stores).
__global__ void __launch_bounds__(256)
km_pack_kernel(const float* __restrict__ c, __nv_bfloat16* __restrict__ img, int k, int Np, int d) {
  const size_t idx = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (size_t)Np * (d / 8)) return;
  const int o = (int)(idx / Np), n = (int)(idx - (size_t)o * Np), kk = o * 8;
  __align__(16) __nv_bfloat16 hi[8], lo[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const float m2 = -2.f * (n < k ? __ldg(c + (size_t)n * d + kk + e) : 0.f);   // exact; -0 on padding, as pack_ivf
    hi[e] = __float2bfloat16_rn(m2);
    lo[e] = __float2bfloat16_rn(m2 - __bfloat162float(hi[e]));
  }
  const int KT = 3 * d / 64;
  auto at = [&](int col) {
    return img + ((size_t)(n >> 8) * KT + (col >> 6)) * (256 * 64) + (size_t)((col & 63) >> 3) * (256 * 8) + (n & 255) * 8;
  };
  const uint4 qh = *reinterpret_cast<const uint4*>(hi), ql = *reinterpret_cast<const uint4*>(lo);
  *reinterpret_cast<uint4*>(at(kk)) = qh;
  *reinterpret_cast<uint4*>(at(d + kk)) = qh;
  *reinterpret_cast<uint4*>(at(2 * d + kk)) = ql;
}

// cnorm[n] = |c_n|^2 summed in fp64 and rounded once (pack_ivf), +inf past k.  One warp per row.
__global__ void __launch_bounds__(256)
km_cnorm_kernel(const float* __restrict__ c, float* __restrict__ cnorm, int k, int Np, int d) {
  const int n = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (n >= Np) return;
  if (n >= k) { if (lane == 0) cnorm[n] = __int_as_float(0x7f800000); return; }
  double s = 0.0;
  for (int j = lane; j < d; j += 32) { const double v = __ldg(c + (size_t)n * d + j); s = fma(v, v, s); }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_xor_sync(0xffffffffu, s, off);
  if (lane == 0) cnorm[n] = __double2float_rn(s);
}

// cand [M][nc] {score bits, column} (nprobe 1) -> assign[m] = arg-min over the k real centroids (ties to the lower one,
// as ivf_select), dist[m] = max(|x|^2 + |c|^2 - 2 x.c, 0) with x.c in fp32; -1 / +inf when no score is a number.
// One warp per row.
__global__ void __launch_bounds__(256)
km_argmin_kernel(const int2* __restrict__ cand, const float* __restrict__ x, const float* __restrict__ c,
                 const float* __restrict__ cnorm, int* __restrict__ assign, float* __restrict__ dist, int M, int nc, int k,
                 int d) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  float bs = __int_as_float(0x7f800000);
  int bc = 0x7fffffff;
  const int2* cr = cand + (size_t)row * nc;
  for (int j = lane; j < nc; j += 32) {
    const int2 e = __ldg(cr + j);
    const float s = __int_as_float(e.x);
    if (e.y < k && km_less(s, e.y, bs, bc)) { bs = s; bc = e.y; }
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const float os = __shfl_xor_sync(0xffffffffu, bs, off);
    const int oc = __shfl_xor_sync(0xffffffffu, bc, off);
    if (km_less(os, oc, bs, bc)) { bs = os; bc = oc; }
  }
  const bool ok = bc < k;
  // the reported distance in fp32 as faiss forms it, with x.c exact in fp32 rather than the bf16x3 score
  const float4* xr = reinterpret_cast<const float4*>(x + (size_t)row * d);
  const float4* cr4 = reinterpret_cast<const float4*>(c + (size_t)(ok ? bc : 0) * d);
  float xn = 0.f, ip = 0.f;
  for (int i = lane; i < d / 4; i += 32) {
    const float4 q = __ldg(xr + i), v = __ldg(cr4 + i);
    xn = __fmaf_rn(q.x, q.x, xn); xn = __fmaf_rn(q.y, q.y, xn);
    xn = __fmaf_rn(q.z, q.z, xn); xn = __fmaf_rn(q.w, q.w, xn);
    ip = __fmaf_rn(q.x, v.x, ip); ip = __fmaf_rn(q.y, v.y, ip);
    ip = __fmaf_rn(q.z, v.z, ip); ip = __fmaf_rn(q.w, v.w, ip);
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    xn += __shfl_xor_sync(0xffffffffu, xn, off);
    ip += __shfl_xor_sync(0xffffffffu, ip, off);
  }
  if (lane == 0) {
    assign[row] = ok ? bc : -1;
    dist[row] = ok ? fmaxf(__fsub_rn(__fadd_rn(xn, __ldg(cnorm + bc)), __fmul_rn(2.f, ip)), 0.f) : __int_as_float(0x7f800000);
  }
}

// tcount[row / TR][assign[row]] += 1
__global__ void __launch_bounds__(256)
km_tile_count_kernel(const int* __restrict__ assign, int* __restrict__ tcount, int n, int k, int TR) {
  const int row = blockIdx.x * 256 + threadIdx.x;
  if (row >= n) return;
  const int a = __ldg(assign + row);
  if (a >= 0 && a < k) atomicAdd(tcount + (size_t)(row / TR) * k + a, 1);
}

// per centroid: tcount[t][c] <- rows of c in tiles before t (exclusive scan over the tiles); counts[c] = ext[c] = total
__global__ void __launch_bounds__(256)
km_tile_scan_kernel(int* __restrict__ tcount, int* __restrict__ counts, int* __restrict__ ext, int ntiles, int k) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= k) return;
  int run = 0;
  for (int t = 0; t < ntiles; ++t) {
    const int v = tcount[(size_t)t * k + c];
    tcount[(size_t)t * k + c] = run;
    run += v;
  }
  if (counts) counts[c] = run;
  ext[c] = run;
}

// one warp per tile, 32 rows at a time in ascending order: a row's place is its centroid's offset + the rows of that
// centroid in earlier tiles + those already placed from this tile + its rank among equal lanes
__global__ void __launch_bounds__(256)
km_scatter_kernel(const int* __restrict__ assign, int* __restrict__ cursor, const int* __restrict__ offsets,
                  int* __restrict__ order, int n, int k, int TR, int ntiles) {
  const int t = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (t >= ntiles) return;
  const int r0 = t * TR, r1 = min(n, r0 + TR);
  int* cur = cursor + (size_t)t * k;
  for (int base = r0; base < r1; base += 32) {
    const int row = base + lane;
    int a = row < r1 ? __ldg(assign + row) : -1;
    if (a >= k) a = -1;
    const unsigned grp = __match_any_sync(0xffffffffu, a);
    const int rank = __popc(grp & ((1u << lane) - 1u));
    int c0 = 0;
    if (a >= 0) {
      c0 = cur[a];
      order[__ldg(offsets + a) + c0 + rank] = row;
    }
    __syncwarp();
    if (a >= 0 && rank == 0) cur[a] = c0 + __popc(grp);
    __syncwarp();
  }
}

// centroid c = (0 + x_r0 + x_r1 + ...) * (1 / count) in fp32, rows ascending (faiss compute_centroids); empty: untouched
__global__ void __launch_bounds__(KM_CENTROID_THREADS)
km_centroid_kernel(const float* __restrict__ x, const int* __restrict__ order, const int* __restrict__ offsets,
                   float* __restrict__ centroids, int d) {
  const int c = blockIdx.x, tid = threadIdx.x;
  const int o0 = __ldg(offsets + c), o1 = __ldg(offsets + c + 1);
  if (o0 == o1) return;
  float acc[KM_CENTROID_COLS];
#pragma unroll
  for (int i = 0; i < KM_CENTROID_COLS; ++i) acc[i] = 0.f;
  for (int o = o0; o < o1; ++o) {
    const float* xr = x + (size_t)__ldg(order + o) * d;
#pragma unroll
    for (int i = 0; i < KM_CENTROID_COLS; ++i) {
      const int j = tid + i * KM_CENTROID_THREADS;
      if (j < d) acc[i] = __fadd_rn(acc[i], __ldg(xr + j));
    }
  }
  const float norm = __fdiv_rn(1.f, (float)(o1 - o0));
#pragma unroll
  for (int i = 0; i < KM_CENTROID_COLS; ++i) {
    const int j = tid + i * KM_CENTROID_THREADS;
    if (j < d) centroids[(size_t)c * d + j] = __fmul_rn(acc[i], norm);
  }
}

// faiss split_clusters for each (ci, cj) in order: c_ci = c_cj, then even coordinates of c_ci scaled by 1 + 1/1024 and
// of c_cj by 1 - 1/1024, odd coordinates the other way round.  Coordinates are independent, so one thread each.
__global__ void __launch_bounds__(256)
km_split_kernel(float* __restrict__ centroids, const int* __restrict__ pairs, int npairs, int d) {
  const int j = blockIdx.x * 256 + threadIdx.x;
  if (j >= d) return;
  const float up = 1.f + 1.f / 1024.f, down = 1.f - 1.f / 1024.f;   // both exact in fp32
  for (int p = 0; p < npairs; ++p) {
    const int ci = __ldg(pairs + 2 * p), cj = __ldg(pairs + 2 * p + 1);
    const float v = centroids[(size_t)cj * d + j];
    centroids[(size_t)ci * d + j] = __fmul_rn(v, (j & 1) ? down : up);
    centroids[(size_t)cj * d + j] = __fmul_rn(v, (j & 1) ? up : down);
  }
}

static int km_np(int k) { return (k + 255) / 256 * 256; }
static int km_chunk(int chunk) { return chunk <= 0 ? KM_DEFAULT_CHUNK : (chunk + 127) / 128 * 128; }

// rows per tile of the counting sort: at least 1024, more when n / 1024 tiles of k counts would exceed KM_TILE_COUNTS
static int km_tile_rows(int n, int k) {
  const int64_t max_tiles = std::max<int64_t>(1, KM_TILE_COUNTS / k);
  const int64_t tr = std::max<int64_t>(1024, ((int64_t)n + max_tiles - 1) / max_tiles);
  return (int)((tr + 31) / 32 * 32);
}

struct KmAssignLayout {
  size_t img, cand, total;
};
static KmAssignLayout km_assign_layout(int d, int k, int chunk) {
  KmAssignLayout L;
  WsPlan P;
  L.img = P.take((size_t)chunk * 3 * d * 2);
  L.cand = P.take((size_t)chunk * (km_np(k) / 16) * sizeof(int2));
  L.total = P.off;
  return L;
}

struct KmUpdateLayout {
  int TR, ntiles;
  size_t tcount, ext, total;
};
static KmUpdateLayout km_update_layout(int n, int k) {
  KmUpdateLayout L;
  L.TR = km_tile_rows(n, k);
  L.ntiles = std::max(1, (n + L.TR - 1) / L.TR);
  WsPlan P;
  L.tcount = P.take((size_t)L.ntiles * k * 4);
  L.ext = P.take((size_t)(k + 1) * 4);
  L.total = P.off;
  return L;
}

static bool km_shape_ok(int n, int d, int k) {
  return n >= 0 && k >= 1 && d >= 64 && d <= KM_MAX_D && d % 64 == 0;
}

}  // namespace svcb

using namespace svcb;

extern "C" {

size_t svcb_kmeans_workspace_bytes(int32_t n, int32_t d, int32_t k, int32_t chunk) {
  if (!km_shape_ok(n, d, k)) return 0;
  const int ch = std::min(km_chunk(chunk), std::max(128, (n + 127) / 128 * 128));
  return std::max(km_assign_layout(d, k, ch).total, km_update_layout(n, k).total);
}

int svcb_kmeans_pack(const float* centroids, float* wimg, float* cnorm, int32_t k, int32_t d, svcb_stream stream) {
  if (!centroids || !wimg || !cnorm || !km_shape_ok(0, d, k)) {
    set_error("svcb_kmeans_pack: need centroids, wimg, cnorm, k >= 1 and d % 64 == 0 with 64 <= d <= 2048");
    return SVCB_E_BAD_SHAPE;
  }
  if (((uintptr_t)wimg & 15)) { set_error("svcb_kmeans_pack: wimg must be 16-byte aligned"); return SVCB_E_BAD_ALIGN; }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const int Np = km_np(k);
  const size_t nt = (size_t)Np * (d / 8);
  {
    KernelScope ks("km_pack", s, 0.0, 4.0 * k * (double)d + 6.0 * Np * (double)d);
    km_pack_kernel<<<(unsigned)((nt + 255) / 256), 256, 0, s>>>(centroids, reinterpret_cast<__nv_bfloat16*>(wimg), k, Np, d);
    SVCB_LAUNCH_CHECK("km_pack");
  }
  {
    KernelScope ks("km_cnorm", s, 2.0 * k * (double)d, 4.0 * k * (double)d + 4.0 * Np);
    km_cnorm_kernel<<<(Np + 7) / 8, 256, 0, s>>>(centroids, cnorm, k, Np, d);
    SVCB_LAUNCH_CHECK("km_cnorm");
  }
  return SVCB_OK;
}

int svcb_kmeans_assign(const float* x, const float* centroids, const float* wimg, const float* cnorm, int32_t* assign,
                       float* dist, int32_t n, int32_t d, int32_t k, int32_t chunk, void* ws, size_t ws_bytes,
                       svcb_stream stream) {
  if (!x || !centroids || !wimg || !cnorm || !assign || !dist || !km_shape_ok(n, d, k)) {
    set_error("svcb_kmeans_assign: need x, centroids, wimg, cnorm, assign, dist, n >= 0, k >= 1 and d % 64 == 0 with "
              "64 <= d <= 2048");
    return SVCB_E_BAD_SHAPE;
  }
  if (((uintptr_t)x & 15) || ((uintptr_t)centroids & 15) || ((uintptr_t)wimg & 15)) {
    set_error("svcb_kmeans_assign: x, centroids and wimg must be 16-byte aligned");
    return SVCB_E_BAD_ALIGN;
  }
  if (n == 0) return SVCB_OK;
  const int ch = std::min(km_chunk(chunk), (n + 127) / 128 * 128);
  const KmAssignLayout L = km_assign_layout(d, k, ch);
  SVCB_TRY(check_workspace(ws, ws_bytes, L.total, "kmeans assign"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(ws);
  const int Np = km_np(k);
  for (int r0 = 0; r0 < n; r0 += ch) {
    const int m = std::min(ch, n - r0);
    const float* xc = x + (size_t)r0 * d;
    SVCB_TRY(launch_ivf_pack(xc, base + L.img, m, d, s));
    SVCB_TRY(launch_ivf_coarse_tc(base + L.img, wimg, cnorm, base + L.cand, m, Np, 3 * d, 1, s));
    KernelScope ks("km_argmin", s, 4.0 * m * (double)d, 8.0 * m * (double)(Np / 16) + 8.0 * m * (double)d + 12.0 * m);
    km_argmin_kernel<<<(m + 7) / 8, 256, 0, s>>>(reinterpret_cast<const int2*>(base + L.cand), xc, centroids, cnorm,
                                                 assign + r0, dist + r0, m, Np / 16, k, d);
    SVCB_LAUNCH_CHECK("km_argmin");
  }
  return SVCB_OK;
}

int svcb_kmeans_update(const float* x, const int32_t* assign, float* centroids, int32_t* counts, int32_t* offsets,
                       int32_t* order, int32_t n, int32_t d, int32_t k, void* ws, size_t ws_bytes, svcb_stream stream) {
  if (!assign || !offsets || !order || (centroids && !x) || !km_shape_ok(n, d, k)) {
    set_error("svcb_kmeans_update: need assign, offsets, order (x with centroids), n >= 0, k >= 1 and d % 64 == 0 with "
              "64 <= d <= 2048");
    return SVCB_E_BAD_SHAPE;
  }
  const KmUpdateLayout L = km_update_layout(n, k);
  SVCB_TRY(check_workspace(ws, ws_bytes, L.total, "kmeans update"));
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(ws);
  int* tcount = reinterpret_cast<int*>(base + L.tcount);
  int* ext = reinterpret_cast<int*>(base + L.ext);
  SVCB_CUDA_CHECK(cudaMemsetAsync(tcount, 0, (size_t)L.ntiles * k * 4, s));
  SVCB_CUDA_CHECK(cudaMemsetAsync(ext + k, 0, 4, s));
  if (n > 0) {
    KernelScope ks("km_tile_count", s, 0.0, 8.0 * n);
    km_tile_count_kernel<<<(n + 255) / 256, 256, 0, s>>>(assign, tcount, n, k, L.TR);
    SVCB_LAUNCH_CHECK("km_tile_count");
  }
  {
    KernelScope ks("km_tile_scan", s, 0.0, 8.0 * L.ntiles * (double)k + 8.0 * k);
    km_tile_scan_kernel<<<(k + 255) / 256, 256, 0, s>>>(tcount, counts, ext, L.ntiles, k);
    SVCB_LAUNCH_CHECK("km_tile_scan");
  }
  SVCB_TRY(launch_bucket_offsets(ext, offsets, k + 1, s));
  if (n > 0) {
    KernelScope ks("km_scatter", s, 0.0, 12.0 * n);
    km_scatter_kernel<<<(L.ntiles + 7) / 8, 256, 0, s>>>(assign, tcount, offsets, order, n, k, L.TR, L.ntiles);
    SVCB_LAUNCH_CHECK("km_scatter");
  }
  if (centroids) {
    KernelScope ks("km_centroid", s, (double)n * d + (double)k * d, 4.0 * n * (double)d + 4.0 * n + 4.0 * k * (double)d);
    km_centroid_kernel<<<k, KM_CENTROID_THREADS, 0, s>>>(x, order, offsets, centroids, d);
    SVCB_LAUNCH_CHECK("km_centroid");
  }
  return SVCB_OK;
}

int svcb_kmeans_split(float* centroids, const int32_t* pairs, int32_t npairs, int32_t d, svcb_stream stream) {
  if (!centroids || npairs < 0 || (npairs && !pairs) || d < 1) { set_error("svcb_kmeans_split: bad argument"); return SVCB_E_BAD_SHAPE; }
  if (npairs == 0) return SVCB_OK;
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  KernelScope ks("km_split", s, 2.0 * npairs * (double)d, 12.0 * npairs * (double)d);
  km_split_kernel<<<(d + 255) / 256, 256, 0, s>>>(centroids, pairs, npairs, d);
  SVCB_LAUNCH_CHECK("km_split");
  return SVCB_OK;
}

}  // extern "C"

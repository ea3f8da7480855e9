// Feature retrieval on an IVF-Flat L2 index: replaces FaissRVCRetrievableFeatureIndex.retriv
// (feature_retrieval/index.py:57-62,75-94) on an `IVF{nlist},Flat` index read by faiss (index.py:147-154).
//
//   ivf_pack        query rows -> the A tile image [x_hi | x_lo | x_hi] of the coarse GEMM (whisper_gemm.cu)
//   ivf_coarse_tc   gemm_tc epilogue 8: |c|^2 - 2 x.c over every centroid (bf16x3 as one bf16 GEMM, K = 3 d), each
//                   epilogue thread keeps the nprobe best of its 16 columns -> cand [M][Np/16][nprobe]
//   ivf_select      one warp per row: merge the candidates to the row's nprobe lists (ascending, ties to the lower
//                   list as faiss's heap keeps the first seen); count rows per first list
//   ivf_order       exclusive scan of those counts (one CTA)
//   ivf_scatter     rows sorted by first list: the warps of one CTA mostly scan the same list, out of L2
//   ivf_scan_blend  one warp per row: exact fp32 sum (x - v)^2 over the probed lists in stored order into a k-best
//                   list held one entry per lane (ties to the vector scanned first), then the RVC weights and blend
// Every row is computed by the same instructions whatever M or its position, so results are bitwise reproducible;
// the order the rows are visited in (ivf_scatter's atomics) changes only which warp computes a row.
#include <cuda_bf16.h>

#include <cstdint>
#include <memory>

#include "common.cuh"

namespace svcb {

constexpr int IVF_MAX_K = 32, IVF_MAX_NPROBE = 8, IVF_MAX_D = 2048;

__device__ __forceinline__ bool key_less(float s, int c, float bs, int bc) { return s < bs || (s == bs && c < bc); }

// cand [M][nc][np] {score bits, column} -> probe [M][np] (list ids ascending by score, -1 past the nlist real lists);
// count[first list] += 1 (bucket nlist: no list)
__global__ void __launch_bounds__(256)
ivf_select_kernel(const int2* __restrict__ cand, int* __restrict__ probe, int* __restrict__ count, int M, int nc, int np,
                  int nlist) {
  const int row = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (row >= M) return;
  float bs[IVF_MAX_NPROBE];
  int bc[IVF_MAX_NPROBE];
#pragma unroll
  for (int i = 0; i < IVF_MAX_NPROBE; ++i) { bs[i] = __int_as_float(0x7f800000); bc[i] = 0x7fffffff; }
  const int2* cr = cand + (size_t)row * nc * np;
  for (int j = lane; j < nc * np; j += 32) {
    const int2 e = __ldg(cr + j);
    float s = __int_as_float(e.x);
    int c = e.y;
    if (c >= nlist) continue;   // padding centroids (score +inf) and unfilled slots
#pragma unroll
    for (int i = 0; i < IVF_MAX_NPROBE; ++i) {
      if (key_less(s, c, bs[i], bc[i])) {
        const float ts = bs[i]; const int tc = bc[i];
        bs[i] = s; bc[i] = c; s = ts; c = tc;
      }
    }
  }
  int first = nlist;
  for (int p = 0; p < np; ++p) {   // np rounds of a warp arg-min over the lanes' heads
    float s = bs[0];
    int c = bc[0];
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float os = __shfl_xor_sync(0xffffffffu, s, off);
      const int oc = __shfl_xor_sync(0xffffffffu, c, off);
      if (key_less(os, oc, s, c)) { s = os; c = oc; }
    }
    const int lst = c < nlist ? c : -1;
    if (lane == 0) probe[(size_t)row * np + p] = lst;
    if (p == 0 && lst >= 0) first = lst;
    if (lst >= 0 && bc[0] == c) {   // the owner pops its head
#pragma unroll
      for (int i = 0; i + 1 < IVF_MAX_NPROBE; ++i) { bs[i] = bs[i + 1]; bc[i] = bc[i + 1]; }
      bs[IVF_MAX_NPROBE - 1] = __int_as_float(0x7f800000); bc[IVF_MAX_NPROBE - 1] = 0x7fffffff;
    }
  }
  if (lane == 0) atomicAdd(count + first, 1);
}

// cursor[b] = sum_{b' < b} count[b'] over n buckets, one CTA of 1024 threads
__global__ void __launch_bounds__(1024)
ivf_order_kernel(const int* __restrict__ count, int* __restrict__ cursor, int n) {
  __shared__ int wsum[32];
  __shared__ int carry;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (tid == 0) carry = 0;
  __syncthreads();
  for (int base = 0; base < n; base += 1024) {
    const int v = base + tid < n ? count[base + tid] : 0;
    int incl = v;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += u;
    }
    if (lane == 31) wsum[warp] = incl;
    __syncthreads();
    if (warp == 0) {
      int w = wsum[lane], wi = w;
#pragma unroll
      for (int off = 1; off < 32; off <<= 1) {
        const int u = __shfl_up_sync(0xffffffffu, wi, off);
        if (lane >= off) wi += u;
      }
      wsum[lane] = wi - w;   // exclusive prefix of the warp totals
    }
    __syncthreads();
    if (base + tid < n) cursor[base + tid] = carry + wsum[warp] + incl - v;
    __syncthreads();
    if (tid == 1023) carry += wsum[warp] + incl;
    __syncthreads();
  }
}

__global__ void __launch_bounds__(256)
ivf_scatter_kernel(const int* __restrict__ probe, int* __restrict__ cursor, int* __restrict__ order, int M, int np, int nlist) {
  const int row = blockIdx.x * 256 + threadIdx.x;
  if (row >= M) return;
  const int l = probe[(size_t)row * np];
  order[atomicAdd(cursor + (l >= 0 ? l : nlist), 1)] = row;
}

// One warp per row (rows in `order`).  x is held as float2 pairs (i * 32 + lane) of the row: d / 64 per lane.
__global__ void __launch_bounds__(256)
ivf_scan_blend_kernel(const float* __restrict__ x, const int* __restrict__ order, const int* __restrict__ probe,
                      const int32_t* __restrict__ offs, const float* __restrict__ vecs, const int64_t* __restrict__ vids,
                      float* __restrict__ out, float* __restrict__ dist, int64_t* __restrict__ ids, int M, int d, int np,
                      int k, float ratio) {
  constexpr int MAXV = IVF_MAX_D / 64;
  const int w = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (w >= M) return;
  const int row = order[w], nv = d / 64;
  const float2* xr = reinterpret_cast<const float2*>(x + (size_t)row * d);
  float2 xv[MAXV];
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv) xv[i] = __ldg(xr + i * 32 + lane);
  float bd = __int_as_float(0x7f800000);   // this lane's entry of the k-best list (lane < k), ascending
  int bi = -1;                             // its row in vecs, -1 = none
  for (int p = 0; p < np; ++p) {
    const int l = __ldg(probe + (size_t)row * np + p);
    if (l < 0) break;
    const int v0 = __ldg(offs + l), v1 = __ldg(offs + l + 1);
    for (int v = v0; v < v1; ++v) {
      const float2* vr = reinterpret_cast<const float2*>(vecs + (size_t)v * d);
      float acc = 0.f;
#pragma unroll
      for (int i = 0; i < MAXV; ++i) {
        if (i < nv) {
          const float2 u = __ldg(vr + i * 32 + lane);
          const float a = __fsub_rn(xv[i].x, u.x), b = __fsub_rn(xv[i].y, u.y);
          acc = __fmaf_rn(a, a, acc);
          acc = __fmaf_rn(b, b, acc);
        }
      }
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
      // insert after every entry <= acc (those were scanned first); a NaN distance is never kept
      const int pos = __popc(__ballot_sync(0xffffffffu, lane < k && bd <= acc));
      if (pos < k && acc == acc) {
        const float ud = __shfl_up_sync(0xffffffffu, bd, 1);
        const int ui = __shfl_up_sync(0xffffffffu, bi, 1);
        if (lane == pos) { bd = acc; bi = v; }
        else if (lane > pos && lane < k) { bd = ud; bi = ui; }
      }
    }
  }
  const bool have = lane < k && bi >= 0;
  const int found = __popc(__ballot_sync(0xffffffffu, have));
  const int nzero = __popc(__ballot_sync(0xffffffffu, have && bd == 0.f));
  if (dist && lane < k) dist[(size_t)row * k + lane] = bd;
  if (ids && lane < k) ids[(size_t)row * k + lane] = have ? __ldg(vids + bi) : -1;
  if (!out) return;
  float* orow = out + (size_t)row * d;
  if (found == 0) {   // nothing to blend with: the row passes through
#pragma unroll
    for (int i = 0; i < MAXV; ++i)
      if (i < nv) reinterpret_cast<float2*>(orow)[i * 32 + lane] = xv[i];
    return;
  }
  // weight = square(1 / score), weight /= weight.sum() in float32 (index.py:85-86); zero distances share the weight
  float wt = 0.f;
  if (have) {
    if (nzero) wt = bd == 0.f ? 1.f : 0.f;
    else { const float r = __frcp_rn(bd); wt = __fmul_rn(r, r); }
  }
  float wsum = 0.f;
  for (int i = 0; i < k; ++i) wsum = __fadd_rn(wsum, __shfl_sync(0xffffffffu, wt, i));
  wt = __fdiv_rn(wt, wsum);
  float2 bl[MAXV];
#pragma unroll
  for (int i = 0; i < MAXV; ++i) bl[i] = make_float2(0.f, 0.f);
  for (int j = 0; j < k; ++j) {   // sum over the neighbours in rank order (index.py:88)
    const float wj = __shfl_sync(0xffffffffu, wt, j);
    const int vj = __shfl_sync(0xffffffffu, bi, j);
    if (vj < 0 || wj == 0.f) continue;
    const float2* vr = reinterpret_cast<const float2*>(vecs + (size_t)vj * d);
#pragma unroll
    for (int i = 0; i < MAXV; ++i) {
      if (i < nv) {
        const float2 u = __ldg(vr + i * 32 + lane);
        bl[i].x = __fadd_rn(bl[i].x, __fmul_rn(wj, u.x));
        bl[i].y = __fadd_rn(bl[i].y, __fmul_rn(wj, u.y));
      }
    }
  }
  const float omr = __fsub_rn(1.f, ratio);   // (1 - ratio) * features + ratio * blend (index.py:61)
#pragma unroll
  for (int i = 0; i < MAXV; ++i)
    if (i < nv)
      reinterpret_cast<float2*>(orow)[i * 32 + lane] =
          make_float2(__fadd_rn(__fmul_rn(omr, xv[i].x), __fmul_rn(ratio, bl[i].x)),
                      __fadd_rn(__fmul_rn(omr, xv[i].y), __fmul_rn(ratio, bl[i].y)));
}

static size_t align256r(size_t x) { return (x + 255) & ~(size_t)255; }

struct IvfLayout {
  size_t img, cand, probe, count, cursor, order, total;
};
static IvfLayout ivf_layout(int d, int Np, int nlist, int np, int M) {
  IvfLayout L;
  const size_t Mp = ((size_t)M + 127) / 128 * 128;
  size_t off = 0;
  L.img = off; off = align256r(off + Mp * 3 * d * 2);
  L.cand = off; off = align256r(off + (size_t)M * (Np / 16) * np * sizeof(int2));
  L.probe = off; off = align256r(off + (size_t)M * np * 4);
  L.count = off; off = align256r(off + (size_t)(nlist + 1) * 4);
  L.cursor = off; off = align256r(off + (size_t)(nlist + 1) * 4);
  L.order = off; off = align256r(off + (size_t)M * 4);
  L.total = off;
  return L;
}

}  // namespace svcb

using namespace svcb;

struct svcb_ivf {
  svcb_ivf_config cfg;
  int Np = 0;   // nlist rounded up to whole 256-column GEMM tiles
  const float* wimg = nullptr;
  const float* cnorm = nullptr;
  const float* vecs = nullptr;
  const int32_t* offs = nullptr;
  const int64_t* ids = nullptr;
};

extern "C" {

int svcb_ivf_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                    const svcb_ivf_config* cfg_host, svcb_ivf** out) {
  if (!dev_blob || !table_host || !cfg_host || !out) { set_error("svcb_ivf_create: bad argument"); return SVCB_E_BAD_SHAPE; }
  const svcb_ivf_config c = *cfg_host;
  if (c.d < 64 || c.d > IVF_MAX_D || c.d % 64 || c.nlist < 1 || c.nprobe < 1 || c.nprobe > IVF_MAX_NPROBE || c.ntotal < 0 ||
      c.ntotal > INT32_MAX) {
    set_error("svcb_ivf_create: need d % 64 == 0 with 64 <= d <= 2048, nlist >= 1, 1 <= nprobe <= 8, 0 <= ntotal < 2^31");
    return SVCB_E_BAD_SHAPE;
  }
  SVCB_TRY(check_blob_device(dev_blob));
  BlobTensors t;
  SVCB_TRY(t.read(dev_blob, blob_bytes, table_host, n_entries));
  auto ix = std::make_unique<svcb_ivf>();
  ix->cfg = c;
  ix->Np = (c.nlist + 255) / 256 * 256;
  const uint64_t d = c.d, Np = ix->Np, n = c.ntotal;
  ix->wimg = t.get("ivf.wimg", Np * 3 * d / 2);
  ix->cnorm = t.get("ivf.cnorm", Np);
  ix->vecs = t.get("ivf.vectors", n * d);
  ix->offs = reinterpret_cast<const int32_t*>(t.get("ivf.offsets", (uint64_t)c.nlist + 1));
  ix->ids = reinterpret_cast<const int64_t*>(t.get("ivf.ids", 2 * n));
  SVCB_TRY(t.status("ivf blob"));
  *out = ix.release();
  return SVCB_OK;
}

void svcb_ivf_destroy(svcb_ivf* ix) { delete ix; }

size_t svcb_ivf_workspace_bytes(const svcb_ivf* ix, int32_t M, int32_t k) {
  if (!ix || M <= 0 || k < 1 || k > IVF_MAX_K) return 0;
  return ivf_layout(ix->cfg.d, ix->Np, ix->cfg.nlist, ix->cfg.nprobe, M).total;
}

int svcb_ivf_retrieve(const svcb_ivf* ix, const float* x, float* out, float* dist, int64_t* ids, int32_t M, int32_t k,
                      float ratio, void* ws, size_t ws_bytes, svcb_stream stream) {
  if (!ix || !x || M < 0) { set_error("svcb_ivf_retrieve: bad argument"); return SVCB_E_BAD_SHAPE; }
  if (k < 1 || k > IVF_MAX_K) { set_error("svcb_ivf_retrieve: need 1 <= k <= 32"); return SVCB_E_BAD_SHAPE; }
  if (((uintptr_t)x & 15) || ((uintptr_t)out & 15)) { set_error("svcb_ivf_retrieve: x and out must be 16-byte aligned"); return SVCB_E_BAD_ALIGN; }
  if (M == 0) return SVCB_OK;
  const svcb_ivf_config& c = ix->cfg;
  const int np = c.nprobe;
  const IvfLayout L = ivf_layout(c.d, ix->Np, c.nlist, np, M);
  if (!ws || ((uintptr_t)ws & 255) || ws_bytes < L.total) { set_error("ivf workspace too small or misaligned"); return SVCB_E_WORKSPACE; }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(ws);
  int* probe = reinterpret_cast<int*>(base + L.probe);
  int* count = reinterpret_cast<int*>(base + L.count);
  int* cursor = reinterpret_cast<int*>(base + L.cursor);
  int* order = reinterpret_cast<int*>(base + L.order);
  SVCB_TRY(launch_ivf_pack(x, base + L.img, M, c.d, s));
  SVCB_TRY(launch_ivf_coarse_tc(base + L.img, ix->wimg, ix->cnorm, base + L.cand, M, ix->Np, 3 * c.d, np, s));
  SVCB_CUDA_CHECK(cudaMemsetAsync(count, 0, (size_t)(c.nlist + 1) * 4, s));
  {
    KernelScope ks("ivf_select", s, 0.0, 8.0 * M * (double)(ix->Np / 16) * np + 4.0 * M * np);
    ivf_select_kernel<<<(M + 7) / 8, 256, 0, s>>>(reinterpret_cast<const int2*>(base + L.cand), probe, count, M, ix->Np / 16,
                                                  np, c.nlist);
    SVCB_LAUNCH_CHECK("ivf_select");
  }
  {
    KernelScope ks("ivf_order", s, 0.0, 8.0 * (c.nlist + 1) + 12.0 * M);
    ivf_order_kernel<<<1, 1024, 0, s>>>(count, cursor, c.nlist + 1);
    SVCB_LAUNCH_CHECK("ivf_order");
    ivf_scatter_kernel<<<(M + 255) / 256, 256, 0, s>>>(probe, cursor, order, M, np, c.nlist);
    SVCB_LAUNCH_CHECK("ivf_scatter");
  }
  {
    // bytes: the rows in and out plus each probed list once per row at the average list size (the lists a row
    // probes are known on the device only); FLOPs: subtract + square-accumulate per scanned element
    const double scanned = (double)M * std::min(np, c.nlist) * ((double)c.ntotal / c.nlist) * c.d * 4.0;
    KernelScope ks("ivf_scan_blend", s, 3.0 * scanned / 4.0, scanned + (out ? 8.0 : 4.0) * M * (double)c.d + 12.0 * M * k);
    ivf_scan_blend_kernel<<<(M + 7) / 8, 256, 0, s>>>(x, order, probe, ix->offs, ix->vecs, ix->ids, out, dist, ids, M, c.d, np,
                                                      k, ratio);
    SVCB_LAUNCH_CHECK("ivf_scan_blend");
  }
  return SVCB_OK;
}

}  // extern "C"

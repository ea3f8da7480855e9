// C ABI for the PPG extractor: truncated Whisper AudioEncoder (whisper/model.py:132-163 after the
// loader's surgery, whisper/inference.py:11-29).  Stage pipeline:
//   conv1+GELU (GEMM over an im2col image of the log-mel; its epilogue scatters into conv2's im2col image) ->
//   conv2(stride 2)+GELU+pos-emb (GEMM) -> n_layer x { LN -> QKV GEMM (head-major panels) -> wgmma attention
//   (whisper_attn_tc.cu) -> out-proj GEMM (+residual) -> LN -> MLP GEMM+GELU -> MLP GEMM (+residual) } -> ln_post
#include <memory>
#include <string>
#include <vector>

#include "common.cuh"

namespace svcb {
struct WBlock {
  const float *ln1g, *ln1b, *ln2g, *ln2b, *bqkv, *bo, *b1, *b2;
  const void *wqkv, *wo, *w1, *w2;
};
}  // namespace svcb

struct svcb_whisper {
  svcb_whisper_config cfg;
  const float *conv1_wimg, *conv1_b, *conv2_wimg, *conv2_b, *pos, *lnp_g, *lnp_b;
  std::vector<svcb::WBlock> blocks;
};

using namespace svcb;

static size_t align256(size_t x) { return (x + 255) & ~(size_t)255; }

struct WLayout {
  size_t h1, x, a, qkv, att, mid, total;
  int n2, M;
};
static WLayout whisper_layout(const svcb_whisper_config& c, int B, int n) {
  WLayout L;
  L.n2 = (n - 1) / 2 + 1;
  L.M = B * L.n2;
  const size_t D = c.n_state;
  size_t off = 0;
  // im2col tile image of the log-mel for conv1: [ceil(B n / 128)][K1p / 64][8][128][8] bf16, K1p = 3 n_mels padded to 64
  L.h1 = off; off = align256(off + ((size_t)B * n + 127) / 128 * 128 * ((3 * (size_t)c.n_mels + 63) / 64 * 64) * 2);
  L.x = off; off = align256(off + (size_t)L.M * D * 4);
  const size_t Mp = (size_t)(L.M + 127) / 128 * 128;  // tile images are padded to whole 128-row tiles
  L.a = off; off = align256(off + Mp * D * 2);
  // QKV in the attention kernel's head-major layout (common.cuh qkv_heads_off): items padded to 128 positions
  L.qkv = off; off = align256(off + (size_t)B * qkv_heads_tp(L.n2) * 3 * D * 2);
  L.att = off; off = align256(off + Mp * D * 2);
  L.mid = off; off = align256(off + Mp * 4 * D * 2);
  L.total = off + 4096;
  return L;
}

extern "C" {

int svcb_whisper_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host,
                        int32_t n_entries, const svcb_whisper_config* cfg_host, svcb_whisper** out) {
  if (!dev_blob || !table_host || !cfg_host || !out) { set_error("null argument"); return SVCB_E_BAD_SHAPE; }
  SVCB_TRY(check_blob_device(dev_blob));
  const svcb_whisper_config& c = *cfg_host;
  if (c.n_state % 256 || c.n_state / c.n_head != 64 || c.n_layer < 1 || c.n_state > 2048) {
    set_error("whisper config: n_state must be a multiple of 256 (<= 2048) with 64-wide heads");
    return SVCB_E_UNSUPPORTED;
  }
  BlobTensors t;
  SVCB_TRY(t.read(dev_blob, blob_bytes, table_host, n_entries));
  auto w = std::make_unique<svcb_whisper>();
  w->cfg = c;
  const uint64_t D = c.n_state;
  w->conv1_wimg = t.get("conv1.wimg", D * ((3 * (uint64_t)c.n_mels + 63) / 64 * 64) / 2); w->conv1_b = t.get("conv1.b", D);
  w->conv2_wimg = t.get("conv2.wimg", D * 3 * D / 2); w->conv2_b = t.get("conv2.b", D);
  w->pos = t.get("pos", (uint64_t)c.n_ctx * D);
  w->lnp_g = t.get("ln_post.g", D); w->lnp_b = t.get("ln_post.b", D);
  w->blocks.resize(c.n_layer);
  for (int i = 0; i < c.n_layer; ++i) {
    const std::string p = "blk." + std::to_string(i);
    WBlock& b = w->blocks[i];
    b.ln1g = t.get(p + ".ln1.g", D); b.ln1b = t.get(p + ".ln1.b", D);
    b.ln2g = t.get(p + ".ln2.g", D); b.ln2b = t.get(p + ".ln2.b", D);
    b.wqkv = t.get(p + ".wqkv", 3 * D * D / 2); b.bqkv = t.get(p + ".bqkv", 3 * D);
    b.wo = t.get(p + ".wo", D * D / 2); b.bo = t.get(p + ".bo", D);
    b.w1 = t.get(p + ".w1", 4 * D * D / 2); b.b1 = t.get(p + ".b1", 4 * D);
    b.w2 = t.get(p + ".w2", 4 * D * D / 2); b.b2 = t.get(p + ".b2", D);
  }
  SVCB_TRY(t.status("whisper blob"));
  *out = w.release();
  return SVCB_OK;
}

void svcb_whisper_destroy(svcb_whisper* w) { delete w; }

size_t svcb_whisper_workspace_bytes(const svcb_whisper* w, int32_t B, int32_t n_frames) {
  if (!w || B <= 0 || n_frames <= 0) return 0;
  return whisper_layout(w->cfg, B, n_frames).total;
}

int svcb_whisper_encode(const svcb_whisper* w, const float* mel, float* out, int32_t B, int32_t n_frames,
                        void* ws, size_t ws_bytes, svcb_stream stream) {
  if (!w || !mel || !out || B <= 0 || n_frames <= 0) { set_error("svcb_whisper_encode: bad argument"); return SVCB_E_BAD_SHAPE; }
  const svcb_whisper_config& c = w->cfg;
  const WLayout L = whisper_layout(c, B, n_frames);
  if (L.n2 > c.n_ctx) { set_error("incorrect audio shape: more than n_audio_ctx positions"); return SVCB_E_BAD_SHAPE; }
  if (!ws || ((uintptr_t)ws & 255) || ws_bytes < L.total) { set_error("whisper workspace too small or misaligned"); return SVCB_E_WORKSPACE; }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* base = static_cast<char*>(ws);
  void* a1 = base + L.h1;
  float* x = reinterpret_cast<float*>(base + L.x);
  void* a = base + L.a; void* qkv = base + L.qkv; void* att = base + L.att; void* mid = base + L.mid;
  const int D = c.n_state, n = n_frames, n2 = L.n2, M = L.M;
  // conv1 + GELU (whisper/model.py:149) as a tensor-core GEMM over the im2col image of the log-mel; its epilogue
  // scatters GELU(h1) straight into conv2's im2col tile image (parked in the MLP hidden buffer, free until the first
  // block), which is zeroed first: the t = -1 taps and the rows that pad M to whole tiles are never written.  (The fp32
  // CUDA-core conv1 + the separate im2col pass were 2.0 of the encoder's 33.6 ms.)
  SVCB_CUDA_CHECK(cudaMemsetAsync(mid, 0, (size_t)(M + 127) / 128 * 128 * 3 * D * 2, s));
  SVCB_TRY(launch_im2col_s1_image(mel, a1, B, c.n_mels, n, s));
  SVCB_TRY(launch_gemm_tc(a1, w->conv1_wimg, w->conv1_b, mid, nullptr, B * n, D, (3 * c.n_mels + 63) / 64 * 64, EPI_GELU_CONV2_IMG, s, n));
  // conv2 (k=3, stride 2) + GELU + positional embedding, time-major (:150-157): im2col image x the [D, 3D] weight image
  SVCB_TRY(launch_gemm_tc(mid, w->conv2_wimg, w->conv2_b, x, w->pos, M, D, 3 * D, EPI_GELU_ADD_F32, s, n2));
  // pad positions of the head-major QKV buffer are read (times P = 0) but never written: keep them finite
  if (qkv_heads_tp(n2) != n2) SVCB_CUDA_CHECK(cudaMemsetAsync(qkv, 0, (size_t)B * qkv_heads_tp(n2) * 3 * D * 2, s));
  for (int i = 0; i < c.n_layer; ++i) {
    const WBlock& b = w->blocks[i];
    SVCB_TRY(launch_ln_rows(x, b.ln1g, b.ln1b, a, M, D, true, s));
    SVCB_TRY(launch_gemm_tc(a, b.wqkv, b.bqkv, qkv, nullptr, M, 3 * D, D, EPI_QKV_HEADS, s, n2));
    SVCB_TRY(launch_whisper_attention_tc(qkv, att, B, n2, D, c.n_head, 0, s));
    SVCB_TRY(launch_gemm_tc(att, b.wo, b.bo, x, x, M, D, D, EPI_RESID_F32, s));
    SVCB_TRY(launch_ln_rows(x, b.ln2g, b.ln2b, a, M, D, true, s));
    SVCB_TRY(launch_gemm_tc(a, b.w1, b.b1, mid, nullptr, M, 4 * D, D, EPI_GELU_BF16_IMAGE, s));
    SVCB_TRY(launch_gemm_tc(mid, b.w2, b.b2, x, x, M, D, 4 * D, EPI_RESID_F32, s));
  }
  return launch_ln_rows(x, w->lnp_g, w->lnp_b, out, M, D, false, s);
}


int svcb_whisper_log_mel(const float* audio, const float* mel_filters, const float* noise, float noise_gain,
                         float* mel, void* scratch, int32_t B, int32_t n_samples, int32_t n_mels,
                         svcb_stream stream) {
  if (!audio || !mel_filters || !mel || !scratch) { set_error("log_mel: null pointer"); return SVCB_E_BAD_SHAPE; }
  if (B < 0 || n_samples < 0 || n_mels <= 0) { set_error("log_mel: bad shape"); return SVCB_E_BAD_SHAPE; }
  return launch_log_mel(audio, mel_filters, noise, noise_gain, mel, static_cast<unsigned*>(scratch), B, n_samples,
                        n_mels, static_cast<cudaStream_t>(stream));
}

size_t svcb_op_gemm_bf16_scratch_bytes(int32_t M, int32_t N, int32_t K) {
  return ((size_t)(M + 127) / 128 * 128 * K + (size_t)N * K) * 2 + 1024;
}

int svcb_op_gemm_bf16(const void* A_bf16, const void* W_bf16, const float* bias, void* out, const float* res,
                      int32_t M, int32_t N, int32_t K, int32_t epilogue, void* scratch, size_t scratch_bytes,
                      svcb_stream stream) {
  // row-major operands in, converted to tile images in `scratch`; epilogue 1 writes the tile image of out
  if (!scratch || scratch_bytes < svcb_op_gemm_bf16_scratch_bytes(M, N, K)) { set_error("gemm scratch too small"); return SVCB_E_WORKSPACE; }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  char* a_img = static_cast<char*>(scratch);
  char* w_img = a_img + (((size_t)(M + 127) / 128 * 128 * K * 2 + 255) & ~(size_t)255);
  SVCB_TRY(launch_rowmajor_to_image(A_bf16, a_img, M, K, 128, s));
  SVCB_TRY(launch_rowmajor_to_image(W_bf16, w_img, N, K, 256, s));
  return launch_gemm_tc(a_img, w_img, bias, out, res, M, N, K, static_cast<GemmEpi>(epilogue), s);
}

size_t svcb_op_attention_tc_bf16_scratch_bytes(int32_t B, int32_t T, int32_t D) {
  if (B <= 0 || T <= 0 || D <= 0) return 0;
  const size_t Mp = ((size_t)B * T + 127) / 128 * 128;
  return align256((size_t)B * qkv_heads_tp(T) * 3 * D * 2) + align256(Mp * D * 2) + 512;
}

int svcb_op_attention_tc_bf16(const void* qkv_bf16, void* out_bf16, int32_t B, int32_t T, int32_t D, int32_t heads,
                              int32_t v_layout, void* scratch, size_t scratch_bytes, svcb_stream stream) {
  // row-major q|k|v in, converted to the GEMM tile image the encoder produces; result converted back
  if (!scratch || ((uintptr_t)scratch & 255) || scratch_bytes < svcb_op_attention_tc_bf16_scratch_bytes(B, T, D)) {
    set_error("attention_tc scratch too small or misaligned");
    return SVCB_E_WORKSPACE;
  }
  cudaStream_t s = static_cast<cudaStream_t>(stream);
  const size_t M = (size_t)B * T;
  char* qimg = static_cast<char*>(scratch);
  const size_t qbytes = (size_t)B * qkv_heads_tp(T) * 3 * D * 2;
  char* oimg = qimg + align256(qbytes);
  SVCB_CUDA_CHECK(cudaMemsetAsync(qimg, 0, qbytes, s));
  SVCB_TRY(launch_qkv_rowmajor_to_heads(qkv_bf16, qimg, B, T, D, s));
  SVCB_TRY(launch_whisper_attention_tc(qimg, oimg, B, T, D, heads, v_layout, s));
  return launch_image_to_rowmajor(oimg, out_bf16, (int)M, D, s);
}

}  // extern "C"

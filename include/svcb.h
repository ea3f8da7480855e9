/* svcb.h — C ABI of libsvc_b200.so: the sm_90a SVC inference hot path.
 *
 * The reference (PlayVoice/whisper-vits-svc) has no FFI / plugin layer: its hot path sits
 * behind nn.Module methods (SURVEY.md §8b).  This header is the boundary a maintainer binds
 * instead (ctypes stub in INTEGRATION.md); each entry point names the reference code it
 * replaces (paths relative to the reference root).
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - activations are fp32, contiguous, [B, C, T] with T innermost unless stated;
 *   - no allocation, no ownership transfer, no host synchronisation inside a call: the
 *     caller owns inputs, outputs and the workspace; work is enqueued on `stream`;
 *   - return 0 on success, <0 = svcb_status; svcb_last_error() gives a thread-local message;
 *   - a model handle is immutable after creation: concurrent calls on different streams
 *     are fine when their workspaces differ;
 *   - sm_90a only, no fallback: svcb_model_create, svcb_whisper_create, svcb_hubert_create,
 *     svcb_ivf_create and svcb_speaker_create fail with SVCB_E_UNSUPPORTED elsewhere.
 */
#ifndef SVCB_H_
#define SVCB_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum {
  SVCB_OK = 0,
  SVCB_E_BAD_SHAPE = -1,
  SVCB_E_BAD_ALIGN = -2,
  SVCB_E_UNSUPPORTED = -3,
  SVCB_E_CUDA = -4,
  SVCB_E_MISSING_TENSOR = -5,
  SVCB_E_WORKSPACE = -6
} svcb_status;

typedef void* svcb_stream; /* cudaStream_t */

#define SVCB_MAX_UPS 8
#define SVCB_MAX_RES 4

/* hp.vits.*, hp.gen.*, hp.data.* of configs/base.yaml plus the constants hard-coded at
 * vits/models.py:220-238 (2 heads, 6 layers, FFN k3, window 4; flow k5, 4 WN layers, 4 flows). */
typedef struct {
  int32_t ppg_dim, vec_dim, spk_dim, inter_channels, hidden_channels, filter_channels;
  int32_t enc_layers, enc_heads, enc_kernel, enc_window;
  int32_t n_flows, wn_layers, wn_kernel;
  int32_t gen_input, gen_initial_channel;
  int32_t n_ups;
  int32_t up_rates[SVCB_MAX_UPS];
  int32_t up_kernels[SVCB_MAX_UPS];
  int32_t n_res;
  int32_t res_kernels[SVCB_MAX_RES];
  int32_t res_dilations[SVCB_MAX_RES][3];
  int32_t sampling_rate;
  int32_t n_harmonics;   /* 11 = fundamental + 10 overtones (vits_decoder/nsf.py:368) */
  int32_t precision;     /* convs and prior attention: 0 = fp32 CUDA cores, 3 = bf16x3 split wgmma MMA (parity
                          * grade), 1 = plain bf16 wgmma MMA; other values: SVCB_E_UNSUPPORTED at create */
} svcb_config;

/* One named tensor inside the packed weight blob (host-side table, read at create time). */
typedef struct {
  char name[96];
  uint64_t offset_bytes; /* from the start of the blob, 256-byte aligned */
  uint64_t numel;        /* fp32 elements */
} svcb_tensor_entry;

typedef struct svcb_model svcb_model;

/* Optional debugging taps: device pointers (or NULL) that receive a copy of an intermediate.
 * Index meaning in svcb_tap_id. */
typedef enum {
  SVCB_TAP_ENC_FRONT = 0,   /* [B,H,T] after pre+hub+pitch embedding (vits/models.py:47) */
  SVCB_TAP_ENC_LAYER0 = 1,  /* ..+5: output of encoder layer i (attentions.py:68-70) */
  SVCB_TAP_ZP = 7,          /* [B,C,T] (models.py:51) */
  SVCB_TAP_FLOW0 = 8,       /* ..+3: output of coupling layer i (index = flows[2*i]) */
  SVCB_TAP_GEN_PRE = 12,    /* [B,ch0,T] after conv_pre+Mish (generator.py:178-179) */
  SVCB_TAP_GEN_UP0 = 13,    /* ..+4: ups[i](x)+noise_convs[i](source) (generator.py:183-186) */
  SVCB_TAP_GEN_STAGE0 = 18, /* ..+4: mean of the 3 AMP blocks (generator.py:188-194) */
  SVCB_TAP_COUNT = 24
} svcb_tap_id;

typedef struct {
  float* ptr[SVCB_TAP_COUNT];
} svcb_taps;

const char* svcb_last_error(void);
int svcb_version(void);
/* sizeof() of the ABI structs as compiled: 0 svcb_config, 1 svcb_tensor_entry, 2 svcb_taps, 3 svcb_ivf_config
 * (lets a foreign-language binding verify its struct layout at load time). */
size_t svcb_sizeof(int32_t which);

/* Replaces: SynthesizerInfer.__init__ + load_svc_model (svc_inference.py:61-74,163-170).
 * `dev_blob` holds fp32 tensors already folded/re-laid-out by the host packer
 * (whisper-vits-svc_b200/pack.py documents every name and layout). The blob must outlive
 * the handle. */
int svcb_model_create(const void* dev_blob, size_t blob_bytes,
                      const svcb_tensor_entry* table_host, int32_t n_entries,
                      const svcb_config* cfg_host, svcb_model** out);
void svcb_model_destroy(svcb_model* m);

/* Bytes of caller-owned scratch needed by any of the calls below at (B, T frames). */
size_t svcb_workspace_bytes(const svcb_model* m, int32_t B, int32_t T);

/* Bytes of scratch svcb_source needs at (B, T): only the per-frame phase scan (3*B*n_harm*T doubles),
 * not the whole pipeline's peak — pitch2source runs on the WHOLE utterance before the 2500-frame
 * chunk loop (svc_inference.py:89-91), so its scratch must stay O(T) small for hour-long inputs. */
size_t svcb_source_workspace_bytes(const svcb_model* m, int32_t B, int32_t T);

/* Replaces: Generator.pitch2source (vits_decoder/generator.py:160-165) ->
 * SourceModuleHnNSF.forward (nsf.py:383-394) -> SineGen (nsf.py:217-316).
 * f0 [B,T] Hz (0 = unvoiced); rand_ini [B,n_harm] replaces torch.rand (nsf.py:232-235; column 0
 * is ignored); noise [B, T*hop, n_harm] replaces torch.randn_like (nsf.py:311);
 * source out [B,1,T*hop]. */
int svcb_source(const svcb_model* m, const float* f0, const float* rand_ini, const float* noise,
                float* source, int32_t B, int32_t T, void* ws, size_t ws_bytes, svcb_stream stream);

/* Replaces: Generator.source2wav (generator.py:167-173): x*32768, clamp, int16. */
int svcb_source2wav(const float* source, int16_t* out, size_t n, svcb_stream stream);

/* Replaces: f0_to_coarse (vits/utils.py:20-33) + TextEncoder.forward (vits/models.py:39-52).
 * ppg [B,T,ppg_dim] and vec [B,T,vec_dim] are TIME-MAJOR as the reference receives them;
 * pit [B,T]; lengths [B] int64 (ppg_l); eps [B,C,T] replaces torch.randn_like (models.py:51);
 * z_p out [B,C,T]. */
int svcb_prior(const svcb_model* m, const float* ppg, const float* vec, const float* pit,
               const int64_t* lengths, const float* eps, float* z_p, int32_t B, int32_t T,
               void* ws, size_t ws_bytes, const svcb_taps* taps, svcb_stream stream);

/* Replaces: ResidualCouplingBlock.forward(reverse=True) (vits/models.py:89-94) incl. Flip and
 * ResidualCouplingLayer/WN (vits/modules.py:178-203,288-321).  spk [B,spk_dim]; z out [B,C,T]. */
int svcb_flow(const svcb_model* m, const float* z_p, const int64_t* lengths, const float* spk,
              float* z, int32_t B, int32_t T, void* ws, size_t ws_bytes, const svcb_taps* taps,
              svcb_stream stream);

/* Replaces: Generator.inference (vits_decoder/generator.py:175-200).
 * z [B,gen_input,T] (already multiplied by the mask, as models.py:255 passes it);
 * source [B,1,T*hop]; wave out [B,1,T*hop]. */
int svcb_generator(const svcb_model* m, const float* spk, const float* z, const float* source,
                   float* wave, int32_t B, int32_t T, void* ws, size_t ws_bytes,
                   const svcb_taps* taps, svcb_stream stream);

/* Replaces: SynthesizerInfer.inference (vits/models.py:251-256) = prior -> flow -> generator. */
int svcb_infer(const svcb_model* m, const float* ppg, const float* vec, const float* pit,
               const float* spk, const int64_t* lengths, const float* source, const float* eps,
               float* wave, int32_t B, int32_t T, void* ws, size_t ws_bytes,
               const svcb_taps* taps, svcb_stream stream);

/* Number of kernels enqueued by the most recent call on this thread (bench.py's gpu_launches). */
int64_t svcb_last_launch_count(void);

/* ------------------------------------------------------------------ PPG extractor (Whisper) */
/* ModelDimensions of the checkpoint (whisper/model.py:14-25) after the loader's truncation
 * (whisper/inference.py:16-19): n_layer = kept blocks = n_audio_layer - n_audio_layer/4. */
typedef struct {
  int32_t n_mels, n_ctx, n_state, n_head, n_layer;
} svcb_whisper_config;
typedef struct svcb_whisper svcb_whisper;

/* Replaces whisper.inference.load_model (whisper/inference.py:11-29).  Blob names/layouts:
 * whisper-vits-svc_b200/whisper_infer.py:pack_whisper (linear weights bf16, the rest fp32). */
int svcb_whisper_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host,
                        int32_t n_entries, const svcb_whisper_config* cfg_host, svcb_whisper** out);
void svcb_whisper_destroy(svcb_whisper* w);
size_t svcb_whisper_workspace_bytes(const svcb_whisper* w, int32_t B, int32_t n_frames);
/* Replaces AudioEncoder.forward (whisper/model.py:144-163): mel [B, n_mels, n_frames] fp32 ->
 * out [B, (n_frames-1)/2+1, n_state] fp32.  bf16 tensor-core GEMMs/attention, fp32 accumulate,
 * fp32 residual stream (the reference itself runs fp16 on GPU, whisper/inference.py:22-23). */
int svcb_whisper_encode(const svcb_whisper* w, const float* mel, float* out, int32_t B, int32_t n_frames,
                        void* ws, size_t ws_bytes, svcb_stream stream);

/* ------------------------------------------------------------------ content encoder (HuBERT-Soft, SURVEY 8f-2) */
typedef struct svcb_hubert svcb_hubert;
/* Replaces hubert.inference.load_model / hubert_model.hubert_soft (hubert/inference.py:17-23, hubert_model.py:212-222).
 * Blob names/layouts: whisper-vits-svc_b200/hubert_infer.py:pack_hubert (linear weights as bf16 tile images, the
 * convolutional stem and the grouped positional conv fp32).  n_layer = transformer layers in the blob (12). */
int svcb_hubert_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                       int32_t n_layer, svcb_hubert** out);
void svcb_hubert_destroy(svcb_hubert* h);
/* frames produced for n_samples of 16 kHz audio (pad 40 + 40, k10 s5, then six stride-2 convs): ~ n_samples / 320 */
int32_t svcb_hubert_frames(int32_t n_samples);
size_t svcb_hubert_workspace_bytes(const svcb_hubert* h, int32_t B, int32_t n_samples);
/* Replaces HubertSoft.units (hubert/hubert_model.py:68-72): wav [B, n_samples] fp32 (16 kHz, equal-length chunks) ->
 * out [B, svcb_hubert_frames(n_samples), 256] fp32.  taps: null, or 5 device pointers (each may be null) that receive
 * the time-major intermediates [B*T, 512 | 768]: 0 features, 1 projected, 2 embedded, 3 after layer 0, 4 encoded.
 * flags: bit 0 = the six stride-2 convs of the stem in fp32 on the CUDA cores instead of bf16 wgmma GEMMs,
 * bit 1 = the grouped positional convolution likewise. */
int svcb_hubert_units(const svcb_hubert* h, const float* wav, float* out, int32_t B, int32_t n_samples, void* ws,
                      size_t ws_bytes, float* const* taps, int32_t flags, svcb_stream stream);

/* Replaces whisper.audio.log_mel_spectrogram (whisper/audio.py:68-100) plus the extractor's mel noise
 * (whisper/inference.py:46,58) for B equal-length chunks of 16 kHz audio already on the device:
 * audio [B, n_samples] fp32 -> mel [B, n_mels, n_samples/160] fp32 (Hann STFT 400/160, reflect-centred,
 * last frame dropped, |.|^2, mel_filters [n_mels, 201] fp32, log10 clamp 1e-10, per-chunk max-8 floor,
 * (x+4)/4, + noise_gain * noise when noise != NULL).  scratch: >= 4*B bytes of device memory. */
int svcb_whisper_log_mel(const float* audio, const float* mel_filters, const float* noise, float noise_gain,
                         float* mel, void* scratch, int32_t B, int32_t n_samples, int32_t n_mels,
                         svcb_stream stream);

/* ------------------------------------------------------------------ feature retrieval (IVF-Flat, L2) */
/* An IndexIVFFlat of the reference's feature_retrieval/ (svc_train_retrieval.py writes them with faiss).
 * d % 64 == 0 and 64 <= d <= 2048, nlist >= 1, 1 <= nprobe <= 8 (faiss's nprobe; nprobe > nlist probes every list). */
typedef struct {
  int32_t d, nlist, nprobe, pad_;
  int64_t ntotal;
} svcb_ivf_config;   /* svcb_sizeof(3) */
typedef struct svcb_ivf svcb_ivf;

/* Replaces faiss.read_index of an IVF-Flat file (feature_retrieval/index.py:147-154).  Blob names/layouts:
 * whisper-vits-svc_b200/retrieval.py:pack_ivf — "ivf.wimg" the centroids as a bf16 GEMM tile image
 * [Np][3 d] = [-2 c_hi | -2 c_hi | -2 c_lo], Np = nlist rounded up to 256; "ivf.cnorm" [Np] |c|^2 (+inf past nlist);
 * "ivf.vectors" [ntotal, d] fp32 in list order; "ivf.offsets" [nlist + 1] int32; "ivf.ids" [ntotal] int64. */
int svcb_ivf_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                    const svcb_ivf_config* cfg_host, svcb_ivf** out);
void svcb_ivf_destroy(svcb_ivf* ix);
size_t svcb_ivf_workspace_bytes(const svcb_ivf* ix, int32_t M, int32_t k);
/* Replaces FaissRVCRetrievableFeatureIndex.retriv (feature_retrieval/index.py:57-62,75-94).
 * x [M,d] fp32 row-major (16-byte aligned); out [M,d] (NULL = search only); dist [M,k] / ids [M,k] int64 optional
 * (ascending; +inf / -1 where the probed lists hold fewer than k vectors).  1 <= k <= 32.
 * out = (1 - ratio) x + ratio sum_i w_i v_i with w = (1/dist)^2 normalised, except: zero-distance neighbours share
 * the weight equally; fewer than k found -> the blend runs over those found; none found -> out = x.
 * Deterministic; a row's result does not depend on M or on its position. */
int svcb_ivf_retrieve(const svcb_ivf* ix, const float* x, float* out, float* dist, int64_t* ids, int32_t M, int32_t k,
                      float ratio, void* ws, size_t ws_bytes, svcb_stream stream);

/* ------------------------------------------------------------------ speaker encoder (LSTM with projection) */
typedef struct svcb_speaker svcb_speaker;
/* Replaces LSTMSpeakerEncoder(80, 256, 768, 3) + load_checkpoint (speaker/models/lstm.py:35-60,124-131) and the
 * AudioProcessor of speaker_pretrain/config.json.  Blob names/layouts: whisper-vits-svc_b200/speaker_infer.py:pack_speaker.
 * Fails with SVCB_E_UNSUPPORTED unless the device is sm_90 and can hold the recurrence's 128 CTAs co-resident
 * (cooperative launch, one CTA per SM). */
int svcb_speaker_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                        svcb_speaker** out);
void svcb_speaker_destroy(svcb_speaker* s);
/* mel frames of n_samples of 16 kHz audio: 1 + n_samples / 256 */
int32_t svcb_speaker_frames(int64_t n_samples);
/* scratch for svcb_speaker_embed on B items of total_samples samples (any split).  Items run in passes of up to 64,
 * and a pass holds every window step's gate inputs in fp32 and the h image of a whole layer: about 0.6 GB for one
 * utterance of 250 or more frames and about 3.1 GB for a pass of 64 (Lw x Mp rows of 19 KB, Lw = min(250, T),
 * Mp = 10 items rounded up to 128). */
size_t svcb_speaker_workspace_bytes(const svcb_speaker* s, int32_t B, int64_t total_samples);
/* Replaces AudioProcessor.melspectrogram (speaker/utils/audio.py:561-571) for a ragged batch: item b is
 * wav[sample_offsets_host[b] .. sample_offsets_host[b+1]) (more than 512 samples each) ->
 * mel_out [sum_b T_b, 80] fp32 time-major, item b's T_b = svcb_speaker_frames(n_b) rows following item b-1's.
 * Pre-emphasis, reflect-centred periodic-Hann STFT (1024 / 256), magnitude, Slaney mel, 20 log10 - ref_level_db,
 * symmetric clipped normalisation, all in fp32.  ws may be NULL. */
int svcb_speaker_mel(const svcb_speaker* s, const float* wav, const int64_t* sample_offsets_host, int32_t B, float* mel_out,
                     void* ws, size_t ws_bytes, svcb_stream stream);
/* Replaces LSTMSpeakerEncoder.compute_embedding (speaker/models/lstm.py:76-101) for a ragged batch: item b is
 * mel rows [frame_offsets_host[b], frame_offsets_host[b+1]) of mel [*, 80] (16-byte aligned) -> out [B, 256], the mean
 * of the 10 L2-normalised window embeddings; window_out [10 B, 256] receives those (may be NULL).  Products
 * bf16x3 on the tensor cores with fp32 accumulation, gate math fp32.  An item's result does not depend on the batch. */
int svcb_speaker_embed(const svcb_speaker* s, const float* mel, const int64_t* frame_offsets_host, int32_t B, float* out,
                       float* window_out, void* ws, size_t ws_bytes, svcb_stream stream);

/* Operator entry points of the encoder (unit tests):
 * out[M,N] = A[M,K] . W[N,K]^T + bias with epilogue 0: bf16 row-major out, 1: GELU(erf) then bf16
 * out as the GEMM tile image ([ceil(M/128)][N/64][8][128][8], the A operand of a following GEMM),
 * 2: + res (fp32 [M,N]) -> fp32 out.  A, W bf16 row-major (converted to tile images in `scratch`);
 * N % 256 == 0, K % 64 == 0. */
size_t svcb_op_gemm_bf16_scratch_bytes(int32_t M, int32_t N, int32_t K);
int svcb_op_gemm_bf16(const void* A_bf16, const void* W_bf16, const float* bias, void* out, const float* res,
                      int32_t M, int32_t N, int32_t K, int32_t epilogue, void* scratch, size_t scratch_bytes,
                      svcb_stream stream);
/* softmax(q k^T / sqrt(64)) v per head as the encoder runs it (csrc/whisper_attn_tc.cu): qkv bf16 [B*T, 3*D] rows
 * (q|k|v), out bf16 [B*T, D].  q k^T and p v as wgmma MMAs with S and O in registers, operands taken from the
 * head-major layout the QKV GEMM writes (built here from the row-major input).
 * v_layout: 0 = the V panel read as an MN-major operand with LBO = 128 B between 8-key groups (what the encoder
 * uses), 1 = LBO / SBO exchanged (kept for the descriptor unit test).  scratch: 256-byte aligned. */
size_t svcb_op_attention_tc_bf16_scratch_bytes(int32_t B, int32_t T, int32_t D);
int svcb_op_attention_tc_bf16(const void* qkv_bf16, void* out_bf16, int32_t B, int32_t T, int32_t D, int32_t heads,
                              int32_t v_layout, void* scratch, size_t scratch_bytes, svcb_stream stream);

/* Per-kernel timing for roofline reports: after svcb_timing_enable(1) every launch is bracketed
 * by CUDA events on its stream; after the caller synchronises, svcb_timing_report() returns
 * "name launches total_ms algorithmic_flops algorithmic_bytes" lines.  Not thread-safe; off by
 * default (zero overhead). */
void svcb_timing_enable(int32_t on);
const char* svcb_timing_report(void);

/* ---- single-operator entry points (unit-test surface; same kernels the pipeline uses) ---- */

/* y[B,Cout,Tout] = act(conv1d(x[B,Cin,Tin], w) + bias); w is the PACKED layout [Cin][K][CoutPad8]
 * (see pack.py:pack_conv).  Mirrors torch.nn.functional.conv1d as used at every call site
 * listed in SURVEY.md §8c.  act: 0 none, 1 relu, 2 mish, 3 gelu(erf), 4 tanh. */
int svcb_op_conv1d(const float* x, const float* w_packed, const float* bias, float* y,
                   int32_t B, int32_t Cin, int32_t Cout, int32_t Tin, int32_t K, int32_t stride,
                   int32_t dilation, int32_t pad, int32_t act, svcb_stream stream);

/* Replaces SnakeAlias.forward (vits_decoder/alias/act.py:124-128).  ea = exp(alpha) [C],
 * inv_b = 1/(exp(beta)+1e-9) [C], fu/fd = the 12 up/down taps. */
int svcb_op_snake_alias(const float* x, float* y, const float* ea, const float* inv_b,
                        const float* fu, const float* fd, int32_t B, int32_t C, int32_t L,
                        svcb_stream stream);

/* y = LayerNorm_C(x + r) * gamma + beta over the channel dim of [B,C,T] (vits/modules.py:19-22;
 * r may be NULL).  gamma/beta are [C] (gb_batch_stride 0) or [B,C] (stride C: SpeakerAdapter,
 * vits_decoder/generator.py:36-47). */
int svcb_op_layernorm_c(const float* x, const float* r, const float* gamma, const float* beta,
                        float* y, int32_t B, int32_t C, int32_t T, int32_t gb_batch_stride,
                        float eps, svcb_stream stream);

/* Windowed relative-position self-attention (vits/attentions.py:225-274): qkv [B,3*H,T]
 * (q | k | v), emb_rel_k / emb_rel_v [2w+1, H/heads], lengths [B] int64, out [B,H,T]. */
int svcb_op_rel_attention(const float* qkv, const float* emb_rel_k, const float* emb_rel_v,
                          const int64_t* lengths, float* out, int32_t B, int32_t H, int32_t heads,
                          int32_t window, int32_t T, svcb_stream stream);

/* The same attention on the tensor cores (csrc/rel_attn_tc.cu; what the pipeline runs in precision 1 / 3): q.k^T
 * and p.v as wgmma MMAs over bf16 hi/lo split operands, fp32 softmax; head dim 96 and window 4 only.
 * scratch >= svcb_op_rel_attention_tc_scratch_bytes(B, heads, T), 256-byte aligned. */
size_t svcb_op_rel_attention_tc_scratch_bytes(int32_t B, int32_t heads, int32_t T);
int svcb_op_rel_attention_tc(const float* qkv, const float* emb_rel_k, const float* emb_rel_v,
                             const int64_t* lengths, float* out, int32_t B, int32_t H, int32_t heads,
                             int32_t window, int32_t T, void* scratch, size_t scratch_bytes, svcb_stream stream);

/* General stride-1 "same" Conv1d on the tensor cores (csrc/conv_tc.cu): x [B,Cin,T] fp32,
 * w_tc = pack.py:pack_conv_tc_general image, y [B,Cout,T] ([B,Cout/2,T] with the gate flag).
 * flags: 1 input mask, 2 output mask (need lengths), 4 WaveNet gate on interleaved channel pairs,
 * 8 accumulate into y.  act as svcb_op_conv1d.  nsplit 1 = bf16, 3 = bf16x3. */
int svcb_op_conv_tc(const float* x, const void* w_tc, const float* bias, float* y, const float* res,
                    const int64_t* lengths, int32_t B, int32_t Cin, int32_t Cout, int32_t T, int32_t K,
                    int32_t dilation, int32_t nsplit, int32_t flags, int32_t act, svcb_stream stream);

/* One `SnakeAlias -> Conv1d(C->C, K, dilation, same padding) + bias (+ res)` link of
 * AMPBlock.forward (vits_decoder/bigv.py:50-58) on the tensor cores: snake_pack (bf16 hi/lo operand
 * image in `scratch`) followed by the wgmma convolution.  w_tc = pack.py:pack_conv_tc image;
 * nsplit 1 = bf16, 3 = bf16x3 (parity grade). */
size_t svcb_op_amp_conv_tc_scratch_bytes(int32_t B, int32_t C, int32_t L);
int svcb_op_amp_conv_tc(const float* x, float* y, const float* res, const float* ea, const float* inv_b,
                        const float* fu, const float* fd, const void* w_tc, const float* bias, int32_t B,
                        int32_t C, int32_t L, int32_t K, int32_t dilation, int32_t nsplit, void* scratch,
                        size_t scratch_bytes, svcb_stream stream);

/* One `SnakeAlias_in -> Conv1d(C->C, K, dilation) + bias (+ res) [-> SnakeAlias_out]` link of the narrow
 * generator stages (C = 20 or 10; vits_decoder/bigv.py:50-58) in space-to-depth form (csrc/amp_s2d.cu):
 * snake_pack_s2d, then the block-Toeplitz wgmma convolution whose epilogue writes y (fp32, may be NULL)
 * and — when y_act != NULL — SnakeAlias_out(result) as the next link's bf16 hi/lo operand image, returned
 * here decoded to fp32 [B,C,L].  w_s2d = pack.py:pack_conv_s2d image; L % (160/C) == 0. */
size_t svcb_op_amp_s2d_link_scratch_bytes(int32_t B, int32_t C, int32_t L);
int svcb_op_amp_s2d_link(const float* x, float* y, const float* res, float* y_act, const float* ea_in,
                         const float* ib_in, const float* ea_out, const float* ib_out, const float* fu,
                         const float* fd, const void* w_s2d, const float* bias, int32_t B, int32_t C, int32_t L,
                         int32_t K, int32_t dilation, void* scratch, size_t scratch_bytes, svcb_stream stream);

/* Self-test of the wgmma plumbing: D[128,N] = A[shift:shift+128, :K] . B[N,K]^T with
 * bf16 operands (row-major, device) and fp32 accumulation in registers. */
int svcb_op_tc_gemm_selftest(const void* A_bf16, const void* B_bf16, float* D, int32_t R, int32_t N,
                             int32_t K, int32_t shift, svcb_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* SVCB_H_ */

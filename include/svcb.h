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
 *     svcb_ivf_create, svcb_speaker_create, svcb_vad_create and svcb_crepe_create fail with SVCB_E_UNSUPPORTED
 *     elsewhere.
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

/* svcb_infer for a ragged batch of chunks: the layouts of svcb_infer, padded to T frames.  Item b is the first
 * n_b = n_frames_host[b] (1..T) frames of ppg, vec, pit and eps and the first n_b*hop samples of source; nothing past
 * them reaches its result.  The first n_b*hop samples of item b's wave are bitwise those of a lone svcb_infer of the
 * item (B = 1, T = n_b, lengths = {n_b}, same inputs); its later samples are zero.  (svcb_infer with lengths < T keeps
 * the reference's padded-batch semantics instead: the generator there runs unmasked over all T frames.)
 * The lengths are checked on the host before any launch.  SVCB_E_UNSUPPORTED, also before any launch, unless the model
 * is at precision 3 and every generator stage takes the same form with per-item ends at T and at every n_b: the tensor-core
 * upsamplers (comb, fused, or tensor-core phases with the tensor-core noise conv), AMP_TC or space-to-depth AMP
 * blocks, and the fused tail (a 16-byte aligned wave); configs/base.yaml's generator does at any length.
 * ws_bytes >= svcb_workspace_bytes(m, B, T), which includes a region for the lengths.  No taps. */
int svcb_infer_ragged(const svcb_model* m, const float* ppg, const float* vec, const float* pit, const float* spk,
                      const int32_t* n_frames_host, const float* source, const float* eps, float* wave,
                      int32_t B, int32_t T, void* ws, size_t ws_bytes, svcb_stream stream);

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
/* svcb_whisper_encode for a ragged batch: item b is the first n_frames_host[b] (1..n_frames) columns of its mel, and
 * its columns past them must be zero (svcb_whisper_log_mel_ragged writes them so).  Item b's first
 * (n_frames_host[b]-1)/2+1 output rows are bitwise those of a lone svcb_whisper_encode of its own frames; its later
 * rows are zero.  ws_bytes >= svcb_whisper_workspace_bytes(w, B, n_frames), which includes a region for the lengths. */
int svcb_whisper_encode_ragged(const svcb_whisper* w, const float* mel, const int32_t* n_frames_host, float* out, int32_t B,
                               int32_t n_frames, void* ws, size_t ws_bytes, svcb_stream stream);

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
/* svcb_hubert_units (tensor-core stem, no taps) for a ragged batch: item b is the first n_samples_host[b] samples of its
 * row of wav (1..n_samples, at least one frame each).  Item b's first svcb_hubert_frames(n_samples_host[b]) output rows
 * are bitwise those of a lone svcb_hubert_units of its own samples; its later rows are zero.
 * ws_bytes >= svcb_hubert_workspace_bytes(h, B, n_samples), which includes a region for the lengths. */
int svcb_hubert_units_ragged(const svcb_hubert* h, const float* wav, const int32_t* n_samples_host, float* out, int32_t B,
                             int32_t n_samples, void* ws, size_t ws_bytes, svcb_stream stream);

/* Replaces whisper.audio.log_mel_spectrogram (whisper/audio.py:68-100) plus the extractor's mel noise
 * (whisper/inference.py:46,58) for B equal-length chunks of 16 kHz audio already on the device:
 * audio [B, n_samples] fp32 -> mel [B, n_mels, n_samples/160] fp32 (Hann STFT 400/160, reflect-centred,
 * last frame dropped, |.|^2, mel_filters [n_mels, 201] fp32, log10 clamp 1e-10, per-chunk max-8 floor,
 * (x+4)/4, + noise_gain * noise when noise != NULL).  scratch: >= 4*B bytes of device memory. */
int svcb_whisper_log_mel(const float* audio, const float* mel_filters, const float* noise, float noise_gain,
                         float* mel, void* scratch, int32_t B, int32_t n_samples, int32_t n_mels,
                         svcb_stream stream);
/* svcb_whisper_log_mel without noise for a ragged batch: item b is the first n_samples_host[b] (201..n_samples) samples
 * of its row of audio, reflect-padded at its own end and floored at the max over its own n_samples_host[b]/160 frames,
 * which are bitwise those of a lone svcb_whisper_log_mel; its later frames are zero.  scratch: >= 8*B bytes. */
int svcb_whisper_log_mel_ragged(const float* audio, const int32_t* n_samples_host, const float* mel_filters, float* mel,
                                void* scratch, int32_t B, int32_t n_samples, int32_t n_mels, svcb_stream stream);

/* ------------------------------------------------------------------ linear spectrogram (training data, 32 kHz) */
/* Replaces vits/spectrogram.py:spectrogram_torch(y, 1024, sr, 320, 1024, center=False) as prepare/preprocess_spec.py
 * calls it, for a ragged batch: item b is audio[sample_offsets_host[b] .. sample_offsets_host[b+1]) (fp32, already
 * divided by max_wav_value), n_b = its length, which must exceed 352 (the reflect padding); B > 0.
 * out: fp32, item b's [513, n_b / 320] block bin-major, following item b-1's block.  Reflect pad 352 at both ends,
 * periodic-Hann frames of 1024 at hop 320, magnitude sqrt(re^2 + im^2 + 1e-6), all in fp32 by a direct DFT.  Each
 * item's block is bitwise that of a lone call.  scratch is not used at present and may be NULL. */
int svcb_linear_spec_ragged(const float* audio, const int64_t* sample_offsets_host, int32_t B, float* out, void* scratch,
                            size_t scratch_bytes, svcb_stream stream);

/* ------------------------------------------------------------------ log-mel of the validation pass (32 kHz) */
/* Replaces vits_extend/stft.py:TacotronSTFT.mel_spectrogram (n_fft 1024, hop 320, win 1024, center=False) as
 * vits_extend/validation.py calls it on a padded batch: audio [B, L] fp32 (1 <= B <= 65535, L > 352, the reflect
 * padding) -> mel [B, n_mels, L / 320] fp32.  Reflect pad 352 at both ends of every row, periodic-Hann frames of 1024 at
 * hop 320, magnitude sqrt(re^2 + im^2 + 1e-9) by a direct DFT, mel_basis [n_mels, 513] fp32 (1 <= n_mels <= 128)
 * accumulated in ascending bin order over each filter's non-zero span, ln(max(x, 1e-5)), all in fp32.  Each row's
 * result is bitwise that of a lone call.  Bad arguments fail before any launch. */
int svcb_tacotron_mel(const float* audio, int32_t B, int64_t L, const float* mel_basis, int32_t n_mels, float* mel,
                      svcb_stream stream);

/* ------------------------------------------------------------------ resampling of raw recordings (training data) */
/* Replaces librosa.load(path, sr=sample_rate)'s resampling in prepare/preprocess_a.py:11 (resample_wave), as
 * scipy.signal.resample_poly's polyphase FIR, for a ragged batch at one ratio up/down (sr_out / sr_in, reduced):
 * item b is x[in_offsets_host[b] .. in_offsets_host[b+1]) (fp32 mono), n_b >= 1; B >= 1; up, down >= 1.
 * taps: the fp64 filter firwin(2 half + 1, 1 / max(up, down), ('kaiser', 5.0)) * up, half = 10 max(up, down), with
 * down - half % down leading zeros (n_taps in all); pre_remove = (half + leading zeros) / down.  Output j of item b is
 * sum_k taps[k] xup[(j + pre_remove) down - k], xup[i] = x[i / up] where up divides i and 0 <= i / up < n_b, else 0,
 * accumulated in fp64 and rounded once to fp32.  y: item b's ceil(n_b up / down) samples, following item b-1's from
 * y[0].  Each item is bitwise that of a lone call.  The host does not call this for up == down == 1. */
int svcb_resample_ragged(const float* x, const int64_t* in_offsets_host, int32_t B, int32_t up, int32_t down,
                         const double* taps, int64_t n_taps, int64_t pre_remove, float* y, svcb_stream stream);
/* Replaces prepare/preprocess_a.py:12-14 per item: y[offsets_host[b] .. offsets_host[b+1]) (fp32, n_b >= 1, B >= 1)
 * -> out at the same offsets, int16: y / m1 * 0.6 / max(0.01, max|y / m1 * 0.6|) * 32767 * 0.6 in float32 steps,
 * truncated toward zero, with m1 = max|y| of the item.  peak[b] = m1 (fp32, B entries); 0 marks a silent item, whose
 * output is zeros (the reference divides by zero there). */
int svcb_pcm16_normalise_ragged(const float* y, const int64_t* offsets_host, int32_t B, int16_t* out, float* peak,
                                svcb_stream stream);

/* ------------------------------------------------------------------ cutting the lowest STFT bins (training data) */
/* Replaces prepare/preprocess_cdc.py:16-25 (cut_direct_content) for a ragged batch of mono clips: item b is
 * x[offsets_host[b] .. offsets_host[b+1]) (fp32, as torchaudio.load gives it, finite), n_b >= 513, B >= 1.  Its
 * 1024 / 256 periodic-Hann STFT (center, reflect padding of 512) with bins 0 and 1 set to zero, inverted by the
 * overlap-add over the window envelope and computed in fp64 without a transform, rounded to fp32, x 32768, clamped to
 * [-32768, 32767] and truncated toward zero.  out: int16, item b's 256*(n_b/256) samples following item b-1's from
 * out[0].  Each item is bitwise that of a lone call. */
int svcb_cdc_ragged(const float* x, const int64_t* offsets_host, int32_t B, int16_t* out, svcb_stream stream);

/* ------------------------------------------------------------------ trimming silence (training data) */
/* Replaces the silence decision of pydub's detect_silence in prepare/preprocess_trim.py:15-20 (split_on_silence with
 * min_silence_len = 200, silence_thresh = -45, seek_step = 1) for a ragged batch of 16-bit mono clips: item b is
 * x[offsets_host[b] .. offsets_host[b+1]) (n_b >= 0 frames) at rates_host[b] Hz (1..192000); B >= 1.  With
 * L_b = round(1000 n_b / rate) ms (ties to even) and ms m at frame fs(m) = (int)(m * (rate / 1000.0)), window i of
 * frames [fs(i), fs(i + 200)), zero past n_b, is silent iff (unsigned) sqrt(S / N) <= 10^(-45/20) * 32768, S its sum of
 * squares and N = fs(i + 200) - fs(i): audioop.rms's decision, exactly.  flags: one byte per window i = 0 .. L_b - 200
 * (1 = silent; none when L_b < 200), item b's following item b-1's from flags[0].  Each item is bitwise that of a lone
 * call. */
int svcb_trim_silence_ragged(const int16_t* x, const int64_t* offsets_host, const int32_t* rates_host, int32_t B,
                             uint8_t* flags, svcb_stream stream);

/* ------------------------------------------------------------------ WORLD DIO + StoneMask F0 (training data) */
/* Replaces prepare/preprocess_f0.py:28-30: f0, t = pyworld.dio(x, fs=16000, f0_ceil=900, frame_period=10) (f0_floor 71,
 * two channels per octave, speed 1, allowed_range 0.1) and pyworld.stonemask(x, f0, t, fs=16000), in fp64, for a
 * ragged batch: item b is x[offsets_host[b] .. offsets_host[b+1]) (n_b >= 1 samples at 16 kHz); B >= 1.  out: float64,
 * item b's n_b / 160 + 1 frames following item b-1's from out[0], before the reference's round(value, 1).  Items of at
 * most 3 frames get zeros: WORLD's contour fix returns without writing for them.  The filter bank is a direct FIR
 * (equal to WORLD's FFT filtering in exact arithmetic, DESIGN.md §5); each item is bitwise that of a lone call.  ws:
 * svcb_world_f0_workspace_bytes(sum of n_b, B) bytes, 256-byte aligned (about 340 bytes per sample). */
size_t svcb_world_f0_workspace_bytes(int64_t total_samples, int32_t B);
int svcb_world_f0_ragged(const double* x, const int64_t* offsets_host, int32_t B, double* out, void* ws, size_t ws_bytes,
                         svcb_stream stream);

/* ------------------------------------------------------------------ Praat autocorrelation F0 (training data) */
/* Replaces prepare/preprocess_f0_mouth.py:11-22: parselmouth.Sound(x, 16000).to_pitch_ac(time_step=0.01,
 * voicing_threshold=0.5, pitch_floor=30, pitch_ceiling=1000).selected_array['frequency'] (15 candidates, a Hanning
 * window of 3 periods, silence threshold 0.03, octave cost 0.01, octave-jump cost 0.35, voiced/unvoiced cost 0.14), in
 * fp64, for a ragged batch: item b is x[offsets_host[b] .. offsets_host[b+1]) (n_b >= 1600 samples at 16 kHz: at
 * least the 0.1 s window); B >= 1.  out: float64, item b's floor((n_b / 16000 - 0.1) / 0.01) + 1 frames (evaluated in
 * double precision, about n_b / 160 - 9) following item b-1's from out[0], unpadded (the reference pads 6 zeros on
 * each side); 0 marks an unvoiced frame.  The autocorrelation is a direct sum (equal to Praat's FFT form in exact
 * arithmetic, DESIGN.md §5); each item is bitwise that of a lone call.  ws: svcb_praat_f0_workspace_bytes(sum of n_b,
 * B) bytes, 256-byte aligned (about 1.6 bytes per sample). */
size_t svcb_praat_f0_workspace_bytes(int64_t total_samples, int32_t B);
int svcb_praat_f0_ragged(const double* x, const int64_t* offsets_host, int32_t B, double* out, void* ws, size_t ws_bytes,
                         svcb_stream stream);

/* ------------------------------------------------------------------ salience-based F0 (pitch/inference.py) */
/* Replaces pitch/inference.py:31-41 before its np.repeat and moving average: libf0's salience(x, Fs=16000, H=320, N=2048,
 * F_min=45, F_max=1760) with its defaults (10 cents per bin, 636 bins, 10 harmonics weighted 0.9^idx, smoothing over 11
 * bins, gamma 0, transitions within 5 bins at 1 and beyond at 0.01, no constraint region), in fp64, for a ragged batch:
 * item b is x[offsets_host[b] .. offsets_host[b+1]) (float32, n_b >= 320 samples at 16 kHz: two frames); B >= 1.
 * f0: float64, item b's n_b / 320 + 1 frames following item b-1's from f0[0].  Optional taps, each may be NULL, laid out
 * per item as [636][frames] blocks following each other from index 0 (item b's at 636 x its first frame): y_tap the
 * binned spectrogram before smoothing, z_tap the thresholded salience; path_tap (int32, one per frame) the bins of the
 * path.  Each item is bitwise that of a lone call.  ws: svcb_salience_f0_workspace_bytes(sum of n_b, B) bytes,
 * 256-byte aligned (about 30 bytes per sample). */
size_t svcb_salience_f0_workspace_bytes(int64_t total_samples, int32_t B);
int svcb_salience_f0_ragged(const float* x, const int64_t* offsets_host, int32_t B, double* f0, double* y_tap,
                            double* z_tap, int32_t* path_tap, void* ws, size_t ws_bytes, svcb_stream stream);
/* The DP and trace back alone, on a given salience: item b is z[636 x frame_offsets_host[b] ..) as [636][F_b]
 * (F_b = frame_offsets_host[b+1] - frame_offsets_host[b] >= 1, frame_offsets_host[0] >= 0); path: int32, the path's
 * bins, F_b per item following each other from path[0], whatever frame_offsets_host[0] is.  ws: svcb_salience_dp_workspace_bytes(sum of F_b) bytes, 256-byte aligned. */
size_t svcb_salience_dp_workspace_bytes(int64_t total_frames);
int svcb_salience_dp_ragged(const double* z, const int64_t* frame_offsets_host, int32_t B, int32_t* path, void* ws,
                            size_t ws_bytes, svcb_stream stream);

/* ------------------------------------------------------------------ pYIN F0 (pyin_f0.py) */
/* libf0's pyin(x, Fs=16000, N=2048, H=160, F_min=50, F_max=1000) with its defaults (518 bins of 10 cents, 1036 HMM
 * states, 99 thresholds with Beta(1, 18) weights, transitions within 5 bins), in fp64, for a ragged batch: item b is
 * x[offsets_host[b] .. offsets_host[b+1]) (float32 at 16 kHz, n_b >= 1 sample); B >= 1.  The wrapper and its parameters
 * are this project's choice (pyin_f0.compute_f0_pyin); no reference command calls pyin.
 * tab: the device table of SVCB_PYIN_TAB_DOUBLES doubles computed by the host as the reference computes it (pyin_f0.py
 * tables()): the thresholds, the Beta weights, F_axis, then per HMM column its predecessors with A > 0 (ascending, as
 * exact doubles, -1 past the end) and their log(A + tiny).
 * f0, conf: float64, n_b // 160 + 1 per item, following each other from f0[0] / conf[0]; f0 is 0 where unvoiced.
 * Optional taps (null to skip), per item following each other: cmndf_tap [321][F_b], obs_tap the observations
 * [1036][F_b], path_tap (int32, one per frame) the Viterbi states.  Each item is bitwise that of a lone call.
 * ws: svcb_pyin_f0_workspace_bytes(sum of n_b, B) bytes, 256-byte aligned (about 90 bytes per sample). */
#define SVCB_PYIN_TAB_THR 0
#define SVCB_PYIN_TAB_BETA 99
#define SVCB_PYIN_TAB_FAXIS 198
#define SVCB_PYIN_TAB_BIDX 716
#define SVCB_PYIN_TAB_BLOG 13148
#define SVCB_PYIN_TAB_DOUBLES 25580
size_t svcb_pyin_f0_workspace_bytes(int64_t total_samples, int32_t B);
int svcb_pyin_f0_ragged(const float* x, const int64_t* offsets_host, int32_t B, const double* tab, double* f0,
                        double* conf, double* cmndf_tap, double* obs_tap, int32_t* path_tap, void* ws, size_t ws_bytes,
                        svcb_stream stream);
/* The Viterbi and trace back alone, on given observations: item b is obs[1036 x frame_offsets_host[b] ..) as
 * [1036][F_b] (F_b >= 1, frame_offsets_host[0] >= 0); path: int32, F_b per item following each other from path[0].
 * ws: svcb_pyin_dp_workspace_bytes(sum of F_b) bytes, 256-byte aligned. */
size_t svcb_pyin_dp_workspace_bytes(int64_t total_frames);
int svcb_pyin_dp_ragged(const double* obs, const int64_t* frame_offsets_host, int32_t B, const double* tab,
                        int32_t* path, void* ws, size_t ws_bytes, svcb_stream stream);

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

/* ------------------------------------------------------------------ k-means (building IVF-Flat indexes) */
/* Lloyd k-means as faiss 1.7.4's Clustering::train and IndexIVF::add run it for the reference's svc_train_retrieval.py
 * (feature_retrieval/index.py:122-154), and in place of its MiniBatchKMeans compression (transform.py:29-53).
 * Rows x [n, d] fp32 row-major (16-byte aligned), d % 64 == 0 and 64 <= d <= 2048, k >= 1 centroids.  The centroids
 * enter the assignment as pack_ivf's "ivf.wimg" / "ivf.cnorm" (svcb_ivf_create), Np = k rounded up to 256. */

/* Scratch for svcb_kmeans_assign (rows in chunks of `chunk`, 0 = 16384, rounded up to 128) and svcb_kmeans_update
 * at (n, d, k).  About chunk x (6 d + Np / 2) bytes: 210 MB at d = 1280, k = 10,000 and the default chunk. */
size_t svcb_kmeans_workspace_bytes(int32_t n, int32_t d, int32_t k, int32_t chunk);
/* centroids [k, d] -> wimg [Np][3 d] bf16 tile image (Np x 3 d / 2 floats, 16-byte aligned) and cnorm [Np] (|c|^2 summed
 * in fp64 and rounded once, +inf past k): the layout of retrieval.py:pack_ivf, built on the device between iterations. */
int svcb_kmeans_pack(const float* centroids, float* wimg, float* cnorm, int32_t k, int32_t d, svcb_stream stream);
/* Replaces the assignment step of Clustering::train and IndexIVF::add (quantizer->assign): assign [n] int32 the nearest
 * centroid, chosen by bf16x3 on the tensor cores (ivf_coarse_tc) with ties to the lower centroid; dist [n] =
 * max(|x|^2 + |c|^2 - 2 x.c, 0) as faiss reports it, in fp32 from centroids [k, d] (the fp32 rows wimg was packed from)
 * and cnorm.  A row's result does not depend on n, the chunk or its position, and its centroid is the list
 * svcb_ivf_retrieve probes first for that row over the same wimg / cnorm. */
int svcb_kmeans_assign(const float* x, const float* centroids, const float* wimg, const float* cnorm, int32_t* assign,
                       float* dist, int32_t n, int32_t d, int32_t k, int32_t chunk, void* ws, size_t ws_bytes,
                       svcb_stream stream);
/* Replaces compute_centroids (Clustering.cpp) and the list fill of IndexIVF::add: a stable counting sort of the rows by
 * assign -> counts [k] (may be NULL), offsets [k + 1], order [n] (each centroid's rows ascending), then, when centroids
 * is not NULL, centroid c = (fp32 sum of its rows in that order) x (1 / count); empty centroids are left untouched.
 * Bitwise reproducible. */
int svcb_kmeans_update(const float* x, const int32_t* assign, float* centroids, int32_t* counts, int32_t* offsets,
                       int32_t* order, int32_t n, int32_t d, int32_t k, void* ws, size_t ws_bytes, svcb_stream stream);
/* The perturbation of faiss's split_clusters for pairs [npairs][2] = (empty ci, split cj), applied in order:
 * c_ci = c_cj, then even coordinates of c_ci x (1 + 1/1024) and of c_cj x (1 - 1/1024), odd ones the other way round.
 * The choice of cj (a random walk over the counts) is the caller's. */
int svcb_kmeans_split(float* centroids, const int32_t* pairs, int32_t npairs, int32_t d, svcb_stream stream);

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

/* ------------------------------------------------------------------ voice-activity detector (Silero VAD, 16 kHz) */
typedef struct svcb_vad svcb_vad;
/* Replaces the 16 kHz branch of vad/assets/silero_vad.jit.  Blob names/layouts: whisper-vits-svc_b200/vad_infer.py:pack_vad.
 * Fails with SVCB_E_UNSUPPORTED unless the device is sm_90. */
int svcb_vad_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                    svcb_vad** out);
void svcb_vad_destroy(svcb_vad* v);
/* 512-sample windows of n_samples of 16 kHz audio: ceil(n_samples / 512), 0 for an empty item */
int64_t svcb_vad_windows(int64_t n_samples);
/* scratch for svcb_vad_probs on B items of total_windows windows in all: 1 KB per window (layer 0's gate inputs) */
size_t svcb_vad_workspace_bytes(const svcb_vad* v, int32_t B, int64_t total_windows);
/* Replaces get_speech_timestamps' probability loop (vad/utils.py:262-268) for a ragged batch: item b is
 * wav[sample_offsets_host[b] .. sample_offsets_host[b+1]) (offsets non-decreasing, checked before any launch) ->
 * probs_out [sum_b W_b] fp32, item b's W_b = svcb_vad_windows(n_b) probabilities following item b-1's; the last window
 * of an item is zero-padded to 512 samples and the LSTM state starts at zero for each item.  feat_out [sum_b W_b, 64]
 * receives the encoder output of each window (may be NULL).  All fp32.  An item's result does not depend on the batch. */
int svcb_vad_probs(const svcb_vad* v, const float* wav, const int64_t* sample_offsets_host, int32_t B, float* probs_out,
                   float* feat_out, void* ws, size_t ws_bytes, svcb_stream stream);

/* ------------------------------------------------------------------ pitch extractor (CREPE, 16 kHz) */
typedef struct svcb_crepe svcb_crepe;
/* Replaces crepe.load.model + Crepe(model) (crepe/load.py, crepe/model.py:14-92).  capacity 0 = 'full' (bf16 wgmma
 * convolutions, fp32 accumulation), 1 = 'tiny' (fp32 CUDA cores).  Blob names/layouts:
 * whisper-vits-svc_b200/crepe_infer.py:pack_crepe.  Fails with SVCB_E_UNSUPPORTED unless the device is sm_90. */
int svcb_crepe_create(const void* dev_blob, size_t blob_bytes, const svcb_tensor_entry* table_host, int32_t n_entries,
                      int32_t capacity, svcb_crepe** out);
void svcb_crepe_destroy(svcb_crepe* c);
/* frames of n_samples of 16 kHz audio at `hop`: 1 + n_samples / hop (crepe/core.py:663) */
int64_t svcb_crepe_frames(int64_t n_samples, int32_t hop);
/* scratch for svcb_crepe_probs on total_frames frames in all: frames run through the network in chunks of up to 4096,
 * about 0.5 MB per frame of a chunk at full capacity (conv1's output is 384 KB of it) */
size_t svcb_crepe_workspace_bytes(const svcb_crepe* c, int64_t total_frames);
/* Replaces crepe.preprocess (crepe/core.py:626-702, pad = True) and the noise line of pitch/inference.py:78 for a ragged
 * batch: item b is wav[sample_offsets_host[b] .. sample_offsets_host[b+1]) (offsets non-decreasing, checked before any
 * launch; an empty item has one frame) + 0.001 * noise (same layout, may be NULL), zero-padded by 512 on both sides ->
 * frames_out [sum_b F_b, 1024] fp32, F_b = svcb_crepe_frames(n_b, hop): each frame less its mean, over
 * max(1e-10, its unbiased standard deviation). */
int svcb_crepe_frame(const float* wav, const int64_t* sample_offsets_host, int32_t B, int32_t hop, const float* noise,
                     float* frames_out, svcb_stream stream);
/* Replaces crepe.infer (crepe/core.py:539-564; crepe/model.py:94-134: pad, conv, ReLU, BatchNorm (eval), max-pool 2, six
 * times, the classifier over (position, channel) features, sigmoid) and the range mask of crepe.postprocess
 * (crepe/core.py:597-603, fmin 50, fmax 1000) on the frames of svcb_crepe_frame: probs_out [sum_b F_b, 360] fp32,
 * bins outside [39, 299) = -inf.  A frame's row does not depend on the batch. */
int svcb_crepe_probs(const svcb_crepe* c, const float* wav, const int64_t* sample_offsets_host, int32_t B, int32_t hop,
                     const float* noise, float* probs_out, void* ws, size_t ws_bytes, svcb_stream stream);
/* scratch for svcb_crepe_decode: the back-pointers, 720 bytes per frame */
size_t svcb_crepe_decode_workspace_bytes(int64_t total_frames);
/* Replaces crepe.decode.viterbi + bins_to_frequency + crepe.periodicity (crepe/decode.py:55-80, crepe/convert.py:12-33,
 * crepe/core.py:710-722) as crepe.predict applies them (crepe/core.py:117-149): item b is rows
 * frame_offsets_host[b] .. frame_offsets_host[b+1] of probs [.., 360] (each item at least one frame) and is decoded in
 * independent segments of `segment` (1..512) frames: softmax over the bins, then the Viterbi path of
 * librosa.sequence.viterbi under transition[i][j] ~ max(12 - |i - j|, 0) with a uniform start, in fp64, the first maximum
 * on ties.  bins_out int32, pitch_out = 10 * 2^((20 bin + 1997.3794 + dither) / 1200) Hz (dither: cents per frame, may
 * be NULL), periodicity_out = probs[t][bin] (may be NULL); all indexed like the rows of probs. */
int svcb_crepe_decode(const float* probs, const int64_t* frame_offsets_host, int32_t B, int32_t segment, const float* dither,
                      int32_t* bins_out, float* pitch_out, float* periodicity_out, void* ws, size_t ws_bytes,
                      svcb_stream stream);

/* Operator entry points of the encoder (unit tests):
 * acc[M,N] = A[M,K] . W[N,K]^T + bias through epilogue 1..7 of csrc/whisper_gemm.cu, with its res_mod and aux
 * arguments as the encoders pass them: 1 GELU(erf) -> bf16 tile image of out ([ceil(M/128)][N/64][8][128][8]),
 * 2 + res -> fp32 [M,N], 3 GELU + res[m % res_mod], 4 bf16 head-major QKV (common.cuh qkv_heads_off), 5 GELU
 * scattered into the next stride-2 conv's im2col image, 6 the stride-2 valid scatter, 7 GELU + res over the first
 * res_mod columns of rows aux apart.  A, W bf16 row-major (converted to tile images in `scratch`); N % 256 == 0,
 * K % 64 == 0.  lens_host (may be NULL, epilogue 5 only): the frame count of each of the M / res_mod items, staged
 * into `scratch`.  `out` is only written where the epilogue stores: the caller sets its initial contents. */
size_t svcb_op_gemm_bf16_scratch_bytes(int32_t M, int32_t N, int32_t K);
int svcb_op_gemm_bf16(const void* A_bf16, const void* W_bf16, const float* bias, void* out, const float* res,
                      int32_t M, int32_t N, int32_t K, int32_t epilogue, int32_t res_mod, int32_t aux, const int32_t* lens_host,
                      void* scratch, size_t scratch_bytes, svcb_stream stream);
/* softmax(q k^T / sqrt(64)) v per head as the encoder runs it (csrc/whisper_attn_tc.cu): qkv bf16 [B*T, 3*D] rows
 * (q|k|v), out bf16 [B*T, D].  q k^T and p v as wgmma MMAs with S and O in registers, operands taken from the
 * head-major layout the QKV GEMM writes (built here from the row-major input).
 * v_layout: 0 = the V panel read as an MN-major operand with LBO = 128 B between 8-key groups (what the encoder
 * uses), 1 = LBO / SBO exchanged (kept for the descriptor unit test).  lens_host (may be NULL): item b attends over
 * its first lens_host[b] keys (1..T), its query rows past that are zeros or finite.  scratch: 256-byte aligned. */
size_t svcb_op_attention_tc_bf16_scratch_bytes(int32_t B, int32_t T, int32_t D);
int svcb_op_attention_tc_bf16(const void* qkv_bf16, void* out_bf16, int32_t B, int32_t T, int32_t D, int32_t heads,
                              int32_t v_layout, const int32_t* lens_host, void* scratch, size_t scratch_bytes, svcb_stream stream);
/* Row LayerNorm (eps 1e-5) of fp32 x [M, D] as the encoders run it: out_bf16 = 1 writes y as the bf16 GEMM tile image
 * of [M, D] (rows of the last tile past M are not written) and, when y32 is not NULL, the fp32 rows [M, D] too;
 * out_bf16 = 0 writes fp32 rows [M, D] to y.  D % 128 == 0, D <= 2048. */
int svcb_op_ln_rows(const float* x, const float* gamma, const float* beta, void* y, float* y32, int32_t M, int32_t D,
                    int32_t out_bf16, svcb_stream stream);
/* The im2col tile image of Whisper's conv1 (k = 3, pad 1) over mel [B, n_mels, n] fp32: img[b*n + t][j*n_mels + ci] =
 * bf16(mel[b][ci][t + j - 1]), K padded with zero columns to a multiple of 64, pad rows of the last tile zero. */
int svcb_op_im2col_s1_image(const float* mel, void* img, int32_t B, int32_t n_mels, int32_t n, svcb_stream stream);
/* The im2col tile image of one channel group of a 'same' convolution over time-major fp32 rows x [B*T, ld]:
 * img[b*T + t][j*cg + ci] = bf16(x[b*T + t + j - pad][c0 + ci]), zero outside [0, T) or, with lens_host (may be NULL),
 * outside [0, lens_host[b]); pad rows of the last tile zero.  scratch: 4 B bytes when lens_host is given. */
int svcb_op_im2col_rows_image(const float* x, void* img, const int32_t* lens_host, int32_t B, int32_t T, int32_t ld, int32_t c0,
                              int32_t cg, int32_t taps, int32_t pad, void* scratch, size_t scratch_bytes, svcb_stream stream);

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
 * nsplit 1 = bf16, 3 = bf16x3 (parity grade).  accum != 0: y = y_old + (conv + res), as the AMP blocks of a
 * stage add up their outputs; out_div != 0: then y / out_div (the stage mean). */
size_t svcb_op_amp_conv_tc_scratch_bytes(int32_t B, int32_t C, int32_t L);
int svcb_op_amp_conv_tc(const float* x, float* y, const float* res, const float* ea, const float* inv_b,
                        const float* fu, const float* fd, const void* w_tc, const float* bias, int32_t B,
                        int32_t C, int32_t L, int32_t K, int32_t dilation, int32_t nsplit, int32_t accum,
                        float out_div, void* scratch, size_t scratch_bytes, svcb_stream stream);

/* One `SnakeAlias_in -> Conv1d(C->C, K, dilation) + bias (+ res) [-> SnakeAlias_out]` link of the narrow
 * generator stages (C = 20 or 10; vits_decoder/bigv.py:50-58) in space-to-depth form (csrc/amp_s2d.cu):
 * snake_pack_s2d, then the block-Toeplitz wgmma convolution whose epilogue writes y (fp32, may be NULL)
 * and — when y_act != NULL — SnakeAlias_out(result) as the next link's bf16 hi/lo operand image, returned
 * here decoded to fp32 [B,C,L].  w_s2d = pack.py:pack_conv_s2d_link image (output columns in the kernel's
 * phase-slot order; the undilated conv's matrices when the link runs on a folded input, pack.py:s2d_fold);
 * L % (160/C) == 0 and L % 8 == 0 (the scratch size is 0 for other shapes).  out_dilation (1 .. 5, > 1 only with
 * y_act and a link whose input is not folded): the output image is written folded for a next link of that
 * dilation (1 = the standard image). */
size_t svcb_op_amp_s2d_link_scratch_bytes(int32_t B, int32_t C, int32_t L);
int svcb_op_amp_s2d_link(const float* x, float* y, const float* res, float* y_act, const float* ea_in,
                         const float* ib_in, const float* ea_out, const float* ib_out, const float* fu,
                         const float* fd, const void* w_s2d, const float* bias, int32_t B, int32_t C, int32_t L,
                         int32_t K, int32_t dilation, int32_t out_dilation, void* scratch, size_t scratch_bytes,
                         svcb_stream stream);
/* The same link over a ragged batch: item b ends at lens_host[b] samples (host, each a multiple of 8 and of 160/C in
 * [8, L]); y and y_act are written over each item's samples only.  The scratch (svcb_op_amp_s2d_link_scratch_bytes,
 * enough for B <= 128) holds the input image (hi, lo) and then the output image (hi, lo), each
 * (svcb_op_amp_s2d_link_scratch_bytes(B, C, L) - 512) / 4 bytes, followed by the lengths. */
int svcb_op_amp_s2d_link_ragged(const float* x, float* y, const float* res, float* y_act, const float* ea_in,
                                const float* ib_in, const float* ea_out, const float* ib_out, const float* fu,
                                const float* fd, const void* w_s2d, const float* bias, const int32_t* lens_host,
                                int32_t B, int32_t C, int32_t L, int32_t K, int32_t dilation, int32_t out_dilation,
                                void* scratch, size_t scratch_bytes, svcb_stream stream);

/* Self-test of the wgmma plumbing: D[128,N] = A[shift:shift+128, :K] . B[N,K]^T with
 * bf16 operands (row-major, device) and fp32 accumulation in registers. */
int svcb_op_tc_gemm_selftest(const void* A_bf16, const void* B_bf16, float* D, int32_t R, int32_t N,
                             int32_t K, int32_t shift, svcb_stream stream);

#ifdef __cplusplus
}
#endif
#endif /* SVCB_H_ */

/*
 * ovc.h -- C ABI of libovc_b200.so: the tone-colour-converter hot path of OpenVoice
 * (ToneColorConverter.convert -> SynthesizerTrn.voice_conversion) as hand-written
 * sm_90a (H100) CUDA kernels.
 *
 * The reference has no FFI / plugin interface (it is pure Python; SURVEY.md section 8b).  The
 * boundary this library replaces is the Python seam
 *
 *     model.voice_conversion(y, y_lengths, sid_src, sid_tgt, tau)
 *         -> (o_hat[B,1,256T], y_mask[B,1,T], (z, z_p, z_hat))      openvoice/models.py:492-499
 *
 * called from openvoice/api.py:154, plus checkpoint loading (openvoice/api.py:35-39) and model
 * construction from the JSON hparams (openvoice/api.py:21-28).  Entry points take plain
 * pointers and sizes only -- no torch types.  All functions return 0 on success and a negative
 * status otherwise; ovc_last_error() gives the message.  Nothing here ever falls back to a CPU
 * path: without a CUDA device every compute entry point fails.
 */
#ifndef OVC_B200_H
#define OVC_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVC_ABI_VERSION 18 /* 2: ovc_graph_replays, OVC_OPT_PDL .. OVC_OPT_PAIR; 3: option keys 1, 4 and 6 (kernel variant,
                               * activation TMA, tune bits) removed; 4: ovc_reference_encoder_ragged;
                               * 5: ovc_resample, ovc_resample_span; 6: ovc_item_params, the *_items entry points,
                               * ovc_philox_normals; 7: ovc_tts_encode_state, ovc_tts_decode_windows;
                               * 8: ovc_spectrogram_ring; 9: OVC_OPT_PAIR_OCC; 10: ovc_splice;
                               * 11: ovc_tts_encode_state_rows, ovc_tts_state_rows; 12: OVC_OPT_STAGED_EPI;
                               * 13: ovc_resample_plan, ovc_resample_rings;
                               * 14: ovc_voice_conversion_frames, ovc_convert_waveform_frames, ovc_tone_track_expand;
                               * 15: ovc_tts_encode_g, ovc_tts_encode_state_tokens, ovc_tts_decode_windows_tokens,
                               *     ovc_tts_encode_state_rows_tokens, ovc_tts_state_rows_tokens;
                               * 16: ovc_reference_encoder_stream, ovc_reference_encoder_stream_state_floats;
                               * 17: ovc_generate_frames, o_hat NULL on ovc_voice_conversion_frames (the latent half),
                               *     OVC_SPLICE_SRC_WRAP;
                               * 18: ovc_tts_fit, ovc_tts_encode_fit */

#if defined(__GNUC__)
#define OVC_API __attribute__((visibility("default")))
#else
#define OVC_API
#endif

enum {
  OVC_OK = 0,
  OVC_ERR_INVALID = -1,     /* bad argument / unsupported hyper-parameter               */
  OVC_ERR_CUDA = -2,        /* CUDA runtime error (message has cudaGetErrorString)      */
  OVC_ERR_STATE = -3,       /* call order violated (e.g. convert before finalize)       */
  OVC_ERR_MISSING = -4,     /* a checkpoint tensor needed by the hot path is missing    */
  OVC_ERR_NOMEM = -5
};

typedef struct ovc_ctx ovc_ctx;

/* Mirrors the `model` / `data` sections of the converter config.json that
 * OpenVoiceBaseClass.__init__ splats into SynthesizerTrn (openvoice/api.py:21-28,
 * openvoice/models.py:404-465).  The kernels are specialised for the released family
 * (SURVEY.md appendix A.1); anything else is refused by ovc_create with OVC_ERR_INVALID. */
typedef struct ovc_hparams {
  int32_t spec_channels;            /* filter_length/2+1 = 513          api.py:25            */
  int32_t inter_channels;           /* 192                              models.py:408        */
  int32_t hidden_channels;          /* 192                              models.py:409        */
  int32_t gin_channels;             /* 256 (at most 256: ovc_finalize_weights refuses more) models.py:422 */
  int32_t resblock;                 /* 1 (ResBlock1)                    models.py:242        */
  int32_t n_resblock_kernels;       /* 3                                                     */
  int32_t resblock_kernel_sizes[4]; /* 3,7,11                           models.py:261-264    */
  int32_t resblock_dilations[4][3]; /* {1,3,5} each                                          */
  int32_t n_upsamples;              /* 4                                                     */
  int32_t upsample_rates[4];        /* 8,8,2,2                          models.py:245-256    */
  int32_t upsample_kernel_sizes[4]; /* 16,16,4,4                                             */
  int32_t upsample_initial_channel; /* 512                                                   */
  int32_t zero_g;                   /* V2: g zeroed for enc_q and dec   models.py:423,495,498*/
  int32_t hop_length;               /* 256 (= product of upsample_rates)                     */
} ovc_hparams;

/* ABI version of the loaded library (== OVC_ABI_VERSION it was built with). */
OVC_API int ovc_abi_version(void);

/* Last error message of this thread ("" if none). Never NULL. */
OVC_API const char* ovc_last_error(void);

/* Build a converter context on CUDA device `device` (replaces SynthesizerTrn construction,
 * openvoice/api.py:23-30).  Fails with OVC_ERR_CUDA when no usable sm_90 device exists. */
OVC_API int ovc_create(const ovc_hparams* hp, int device, ovc_ctx** out);
OVC_API void ovc_destroy(ovc_ctx* ctx);

/* Feed one checkpoint tensor under its reference state-dict key, fp32, C-contiguous, host
 * memory (replaces load_state_dict(strict=False), openvoice/api.py:35-39; key schema in
 * SURVEY.md appendix A.2, weight-norm stored un-folded as weight_g / weight_v).  Keys that the
 * hot path does not use (ref_enc.*, enc_p.*, ...) are accepted and ignored (returns 1). */
OVC_API int ovc_load_tensor(ovc_ctx* ctx, const char* key, const float* data, const int64_t* shape, int ndim);

/* Fold weight-norm (g*v/||v||, per dim-0 slice), absorb the channel Flips of the flow into the
 * coupling weights, repack every conv for the kernels and upload.  Every tensor read is checked
 * against the shape the model's hyper-parameters give it: OVC_ERR_MISSING names the first missing
 * key, OVC_ERR_INVALID the first mis-shaped one (with its shape and the expected shape).  On
 * failure the loaded tensors are kept, so the caller can replace the offending one and retry. */
OVC_API int ovc_finalize_weights(ovc_ctx* ctx);

/* Number of floats of device workspace a call with (B, Tmax) needs (informational; the arena
 * grows on demand and is reused, so steady-state calls do not allocate). */
OVC_API size_t ovc_workspace_floats(const ovc_ctx* ctx, int B, int Tmax);

/* The hot path.  All pointers are DEVICE pointers on the context's device; the call only
 * enqueues work on `stream` (a cudaStream_t; NULL = default stream) and returns.
 *
 *   spec     [B, spec_channels, Tmax]  linear magnitude spectrogram            (api.py:150-152)
 *   lengths  [B] int64, valid frames per item (1 <= len <= Tmax)               (api.py:153)
 *   g_src    [B, gin] source tone-colour embedding (sid_src, [B,gin,1])        (models.py:493)
 *   g_tgt    [B, gin] target tone-colour embedding (sid_tgt)
 *   noise    [B, inter, Tmax] N(0,1) draws standing in for randn_like at models.py:220,
 *            or NULL: the kernel then draws Philox4x32-10 normals from `seed`.  Counter layout: item b, channel c,
 *            frame t draws philox(key = seed; stream = b, channel = c, frame = t), i.e. ovc_philox_normals(seed, b, 0,
 *            inter, 0, Tmax).  With ovc_voice_conversion_items the key, stream and frame offset can be given per item:
 *            philox(key = seed[b]; stream[b], c, (frame0[b] + t) mod 2^32)
 *   tau      scales the noise term only                                        (models.py:220)
 *   ragged   0: reference batch semantics -- the (unmasked) generator runs over all Tmax frames
 *               of every item exactly as SynthesizerTrn.voice_conversion does on a padded batch
 *            1: every item is converted at its own exact length, i.e. what
 *               ToneColorConverter.convert (batch 1, api.py:148-154) produces per utterance
 *   o_hat    [B, hop*Tmax] waveform out (zero past hop*len when ragged)        (models.py:498)
 *   z, z_p, z_hat  [B, inter, Tmax] latents, masked like the reference; each may be NULL
 */
OVC_API int ovc_voice_conversion(ovc_ctx* ctx, const float* spec, const int64_t* lengths,
                         const float* g_src, const float* g_tgt, const float* noise,
                         uint64_t seed, float tau, int B, int Tmax, int ragged,
                         float* o_hat, float* z, float* z_p, float* z_hat, void* stream);

/* Per-item sampling parameters: each pointer is a DEVICE array of B values, or NULL for "the call's scalar / the
 * default".  With a request's own seed, stream and frame offset, its noise no longer depends on where it sits in a
 * batch, which stream serves it or which window of a longer clip is being converted.  The arrays are read on the device
 * when the kernels run: a call that repeats the same pointers is replayed from its CUDA graph (OVC_OPT_GRAPH) and
 * follows the arrays' current contents.  Which entry point reads which field:
 *   seed           all four: the Philox key of item b (replaces `seed`; for ovc_tts_decode the decode key, which
 *                  SynthesizerTrn.infer-style callers set to the encode key + 1)
 *   stream         all four: counter word 0 of item b (default b)
 *   frame0         voice conversion / convert_waveform: frame counter offset, item b's frame t draws at
 *                  (frame0[b] + t) mod 2^32 (default 0) -- a window starting at frame lo of a longer clip passes lo
 *   tau            voice conversion / convert_waveform (replaces `tau`)
 *   noise_scale_w, length_scale, sdp_ratio   ovc_tts_encode (length_scale values must be positive)
 *   noise_scale    ovc_tts_decode
 * Fields an entry point does not list are ignored.  An explicit noise / noise_w tensor still wins over every key
 * field; the scale fields apply to it too.  NULL fields evaluate exactly the same expressions as the entry points
 * without _items: a struct of NULLs (or items == NULL) gives bit-identical results. */
typedef struct ovc_item_params {
  const uint64_t* seed;
  const int64_t* stream;
  const int64_t* frame0;
  const float* tau;
  const float* noise_scale;
  const float* noise_scale_w;
  const float* length_scale;
  const float* sdp_ratio;
} ovc_item_params;

/* ovc_voice_conversion with per-item parameters; `items` is a HOST pointer (NULL = none). */
OVC_API int ovc_voice_conversion_items(ovc_ctx* ctx, const float* spec, const int64_t* lengths,
                                       const float* g_src, const float* g_tgt, const float* noise,
                                       uint64_t seed, float tau, int B, int Tmax, int ragged,
                                       float* o_hat, float* z, float* z_p, float* z_hat, void* stream,
                                       const ovc_item_params* items);

/* out[c][t] = the Philox normal at (key = seed; stream, channel c0 + c, frame (frame0 + t) mod 2^32), c < C, t < T:
 * exactly the value the kernels draw in-kernel at that counter (see `noise` above; the TTS noise_w rows are channels
 * 0x7700 and 0x7701).  out [C, T] fp32 on the caller's current device; only enqueues on `cuda_stream`.  For tests and
 * for callers that must hand a kernel the noise a request would have drawn. */
OVC_API int ovc_philox_normals(uint64_t seed, int64_t stream, int64_t c0, int C, int64_t frame0, int T, float* out,
                               void* cuda_stream);

/* Copy many sample runs between device buffers in one launch: the join of the TTS decode's sentence rows, their
 * silences and the converter's input rows (an utterance buffer, or the audio rings of live streams).  No context; the
 * caller's current device; only enqueues on `stream` and takes stable pointers, so it can sit inside a captured graph.
 *   src   [src_rows, src_pitch] fp32 (device); may be NULL with src_rows = 0 (every segment a gap)
 *   dst   [dst_rows, dst_cap] fp32 (device)
 *   seg   [S][5] int64 (device): rows (src_row, src_off, count, dst_row, dst_off).  Segment s writes, for i < count,
 *           dst[dst_row * dst_cap + (dst_off + i) mod dst_cap] = src[src_row * src_pitch + src_off + i], or 0 when
 *           src_row < 0 (a silence gap).
 *         dst_cap is the ring wrap of a stream's audio ring; a buffer of whole utterances passes its row pitch and no
 *         write wraps.  Descriptor values are clamped on the device, so nothing is read or written outside src and dst
 *         whatever seg holds: dst_row into [0, dst_rows), dst_off mod dst_cap, count into [0, dst_cap], a source row
 *         into [0, src_rows), src_off into [0, src_pitch] and count to the samples left in the source row.  Segments
 *         whose destinations overlap leave an unspecified one of their values.
 *   flags OVC_SPLICE_PCM16: every copied value x becomes q / 32768.0f, q = rint_even(fl32(x * 32767.0f)) saturated to
 *         [-32768, 32767] (NaN: 0).  This is the project's specification of a float waveform written as a 16-bit PCM
 *         wav and read back as float: libsndfile's default float -> PCM_16 write (scale by 32767, round to nearest)
 *         and its PCM_16 -> float read (divide by 32768), which is what librosa.load returns for such a file. */
#define OVC_SPLICE_PCM16 1
/*   flags OVC_SPLICE_SRC_WRAP: the source rows are rings as well: element i reads
 *         src[src_row * src_pitch + (src_off + i) mod src_pitch] (src_off is reduced mod src_pitch on the device and the
 *         count is no longer cut at the end of the source row).  This gathers runs that wrap around a ring row, such as a
 *         live stream's latent frames, into a padded batch.  The flags combine. */
#define OVC_SPLICE_SRC_WRAP 2
OVC_API int ovc_splice(const float* src, int64_t src_rows, int64_t src_pitch, float* dst, int64_t dst_rows, int64_t dst_cap,
                       const int64_t* seg, int S, int flags, void* stream);

/* Front end of convert (row a2): linear magnitude spectrogram, replaces spectrogram_torch
 * (openvoice/mel_processing.py:40-75; call sites api.py:126-128,150-152) for n_fft = win = 1024,
 * hop 256: reflect-pad 384 at both ends of each item's own length, periodic hann, centre=False,
 * sqrt(re^2 + im^2 + 1e-6).
 *   wav          [B, Lmax] fp32 (device), rows zero padded past wav_lengths[b]
 *   wav_lengths  [B] int64 samples (device), each > 384 (reflect padding) and <= Lmax
 *   spec         [B, spec_channels, Tmax] out; frames >= wav_lengths[b]/hop are written as zeros
 *   frames       [B] int64 out (nullable): min(Tmax, wav_lengths[b] / hop)                          */
OVC_API int ovc_spectrogram(ovc_ctx* ctx, const float* wav, const int64_t* wav_lengths, int B, int Lmax,
                            int Tmax, float* spec, int64_t* frames, void* stream);

/* Magnitude-spectrogram frames of streams held in device audio rings (sample s of row r at
 * rings[r*ring_cap + s % ring_cap]), the front end of batched live streaming: many streams' window spectrograms in one launch, no gather in between.
 * Item b: frames [frame_lo[b], frame_lo[b] + frames[b]) of row[b] -> spec[b, :, 0:frames[b]], zeros up to Tmax.
 * stream_len[b]: samples of the whole stream, or INT64_MAX while it is open (reflect padding at the end only once closed).
 * Each frame is the ovc_spectrogram frame of the whole stream bit for bit, provided the ring row holds every sample the
 * frame reads (frame t: samples [t*hop - 384, t*hop + 640), reflected at the stream's ends).
 *   rings       [ring_rows, ring_cap] fp32 (device), ring_cap >= 1024
 *   row, frame_lo, frames, stream_len   [B] int64 (device); read on the device and clamped so that no read leaves rings
 *   spec        [B, spec_channels, Tmax] out: exactly the `spec` ovc_voice_conversion(_items) reads
 * Same STFT as ovc_spectrogram (n_fft = win = 1024, hop 256).  Only enqueues on `stream`. */
OVC_API int ovc_spectrogram_ring(ovc_ctx* ctx, const float* rings, int ring_rows, int64_t ring_cap, const int64_t* row,
                                 const int64_t* frame_lo, const int64_t* frames, const int64_t* stream_len,
                                 int B, int Tmax, float* spec, void* stream);

/* ToneColorConverter.convert's device work in one call (openvoice/api.py:148-155, batch of B):
 * spectrogram -> voice_conversion with per-item exact lengths (ragged).  Tmax = Lmax / hop.
 *   o_hat   [B, hop*Tmax] out; item b holds hop*frames[b] samples, zeros after
 *   frames  [B] int64 out (nullable)                                                               */
OVC_API int ovc_convert_waveform(ovc_ctx* ctx, const float* wav, const int64_t* wav_lengths, int B, int Lmax,
                                 const float* g_src, const float* g_tgt, const float* noise, uint64_t seed,
                                 float tau, float* o_hat, int64_t* frames, void* stream);
/* ovc_convert_waveform with per-item parameters (ovc_item_params; `items` a host pointer, NULL = none). */
OVC_API int ovc_convert_waveform_items(ovc_ctx* ctx, const float* wav, const int64_t* wav_lengths, int B, int Lmax,
                                       const float* g_src, const float* g_tgt, const float* noise, uint64_t seed,
                                       float tau, float* o_hat, int64_t* frames, void* stream,
                                       const ovc_item_params* items);

/* Time-varying tone colour (reference: SynthesizerTrn.voice_conversion with sid_src / sid_tgt of shape [B, gin, T]).
 * se_frames is a bit set naming the sides given per frame:
 *   OVC_SE_FRAMES_SRC  g_src is [B, gin, Tmax] (frame t of item b at g_src[(b*gin + c)*Tmax + t]); else [B, gin]
 *   OVC_SE_FRAMES_TGT  the same for g_tgt
 * The source side conditions enc_q and the flow forward, the target side the flow reverse and the generator's cond
 * (zero_g checkpoints keep enc_q and the generator unconditioned, as the per-item calls do).  A frame whose embedding
 * equals an item's per-item embedding gets bit-identical conditioning, so se_frames = 0 is exactly the _items entry
 * point and a constant per-frame embedding converts to the per-item result.  Per-frame calls grow the workspace by
 * B * Tmax * 4 bytes times 18944 (both sides) or 6656 (target only) conditioning columns; se_frames is part of the
 * CUDA graph key.  Everything else as ovc_voice_conversion_items / ovc_convert_waveform_items (for the latter Tmax =
 * Lmax / hop).  The conditioning kernel holds each lane's 8 weights of a row in registers and reads one side per block
 * of 32 output columns, so ovc_finalize_weights refuses gin_channels > 256 and conditioning sections whose sizes
 * (2 * hidden_channels per WN layer, upsample_initial_channel for the generator) are not multiples of 32, for every
 * call; every released checkpoint has gin 256, 2 * hidden 384 and 512. */
#define OVC_SE_FRAMES_SRC 1
#define OVC_SE_FRAMES_TGT 2
OVC_API int ovc_voice_conversion_frames(ovc_ctx* ctx, const float* spec, const int64_t* lengths, const float* g_src,
                                        const float* g_tgt, int se_frames, const float* noise, uint64_t seed, float tau,
                                        int B, int Tmax, int ragged, float* o_hat, float* z, float* z_p, float* z_hat,
                                        void* stream, const ovc_item_params* items);
OVC_API int ovc_convert_waveform_frames(ovc_ctx* ctx, const float* wav, const int64_t* wav_lengths, int B, int Lmax,
                                        const float* g_src, const float* g_tgt, int se_frames, const float* noise,
                                        uint64_t seed, float tau, float* o_hat, int64_t* frames, void* stream,
                                        const ovc_item_params* items);

/* The conversion in two halves, split at z_hat (the flow reverse's output, the generator's input).
 *
 * Latent half: ovc_voice_conversion_frames with o_hat == NULL runs the posterior encoder and both flow passes and
 * writes whichever of z, z_p, z_hat are given (at least one output must be); the generator does not run.  Everything
 * else (ragged, per-item parameters, se_frames, graph replay) is as with o_hat given, and the latents are the ones that
 * call writes, bit for bit.
 *
 * Generator half: the HiFi-GAN generator on a caller's z_hat, each item at its own length (ragged).
 *   z_hat    [B, inter, Tmax] fp32; frames past lengths[b] are not read
 *   lengths  [B] int64 (device), 1 <= len <= Tmax
 *   g_tgt    [B, gin] per item, or with se_frames = OVC_SE_FRAMES_TGT [B, gin, Tmax] per frame (the source side does not
 *            reach the generator, so OVC_SE_FRAMES_SRC is refused)
 *   o_hat    [B, hop*Tmax] out, zero past hop*len
 * Given the z_hat an ovc_voice_conversion_frames call (ragged = 1) writes, with the same lengths and target, o_hat equals
 * that call's o_hat bit for bit.  Same workspace as the voice conversion; replayed from a CUDA graph like it. */
OVC_API int ovc_generate_frames(ovc_ctx* ctx, const float* z_hat, const int64_t* lengths, const float* g_tgt, int se_frames,
                                int B, int Tmax, float* o_hat, void* stream);

/* Per-frame embeddings from keyframe tracks ("tone tracks").  Keys are n_keys pairs (key_frame[k], key_se[k, 0:gin]);
 * track b is keys [key0[b], key0[b] + nkeys[b]) with non-decreasing frames.  out[b, c, t] = g_b(frame0[b] + t) for
 * t < frames[b], 0 for frames[b] <= t < Tmax, where g(t) is the first key's embedding before the first key, the last
 * key's from the last key on, and se_k + ((t - f_k) / (f_{k+1} - f_k)) * (se_{k+1} - se_k) for f_k <= t < f_{k+1}, each
 * operation rounded to fp32 on its own; of keys sharing a frame the later one holds from that frame on (a hard switch).
 * Item b's frame t is evaluated at absolute frame frame0[b] + t, so a window of a longer clip gets the whole clip's values.
 *   key_frame [n_keys] int64, key_se [n_keys, gin] fp32, key0 / nkeys / frame0 / frames [B] int64 (all device); the
 *   per-item values are clamped on the device, so no read leaves the key arrays.
 *   out       [B, gin, Tmax] fp32: the per-frame layout ovc_*_frames read.
 * Only enqueues on `stream`; graph-capturable. */
OVC_API int ovc_tone_track_expand(ovc_ctx* ctx, const int64_t* key_frame, const float* key_se, int64_t n_keys,
                                  const int64_t* key0, const int64_t* nkeys, const int64_t* frame0, const int64_t* frames,
                                  int B, int Tmax, float* out, void* stream);

/* Tone-colour embedding of extract_se (row f2): ReferenceEncoder.forward (openvoice/models.py:339-359; call site
 * openvoice/api.py:130) on device -- LayerNorm over frequency, 6 x (Conv2d 3x3 s2 + ReLU), GRU(128) last state,
 * Linear.  Needs the checkpoint's ref_enc.* tensors (OVC_ERR_MISSING otherwise).
 *   spec  [N, spec_channels, T] magnitude spectrogram as written by ovc_spectrogram (all N items T frames)
 *   out   [N, gin]                                                                                          */
OVC_API int ovc_reference_encoder(ovc_ctx* ctx, const float* spec, int N, int T, float* out, void* stream);

/* ovc_reference_encoder on a ragged batch, as extract_se needs for reference clips of different lengths.
 *   spec     [N, spec_channels, Tmax]; item n's frames past lengths[n] are padding and are never read (NaN is fine)
 *   lengths  [N] int64 (device): frames per item, 1 <= len <= Tmax; every item is encoded at its own length,
 *            so row n equals ovc_reference_encoder on spec[n, :, :lengths[n]] alone, bit for bit.  A value outside
 *            [1, Tmax] is clamped into it on the device (never an out-of-bounds read); the ovc_spectrogram `frames`
 *            output can be passed as is.
 *   out      [N, gin]
 * Padding to a common length and calling ovc_reference_encoder is NOT equivalent: the reference's ReferenceEncoder
 * ignores its mask, so its stride-2 convs and GRU read the padded frames. */
OVC_API int ovc_reference_encoder_ragged(ovc_ctx* ctx, const float* spec, const int64_t* lengths,
                                         int N, int Tmax, float* out, void* stream);

/* The reference encoder advanced with live streams, so a stream's source embedding can be learned from its own audio
 * at constant cost per sample.  Each stream owns a state row of ovc_reference_encoder_stream_state_floats() floats
 * (0 before ovc_finalize_weights or without ref_enc.* tensors): the spectrogram frames consumed so far (c0), the GRU
 * hidden state and the <= 2 most recent rows of each conv input that later rows still read.  An all-zero row is a
 * fresh stream.  Frame t is final at n samples when t * hop + (n_fft - pad) <= n (streaming.ready_frames).
 *
 * desc [B][4] int64 (device) = (state_row, ring_row, n_adv, n_snap) per item.  With n_snap > 0 the row first advances
 * to the final frames of n_snap samples and out[b] ([B][gin]) gets the snapshot: bit for bit the embedding
 * ovc_reference_encoder_ragged gives for the stream's first n_snap samples alone (n_snap >= hop and > pad).  The row
 * then advances to the final frames of n_adv samples (never backwards).  The state is not otherwise changed by a
 * snapshot.  Sample s of the stream is rings[ring_row * ring_cap + s % ring_cap]; the caller keeps samples
 * [c0 * hop - pad, max(n_adv, n_snap)) there.  A call adds at most max_new_frames (1 .. 65536) final frames per row.
 *
 * Every descriptor is clamped on the device (rows into range, c0 into [0, 2^29], new frames to max_new_frames), so
 * nothing outside rings, state and out is read or written whatever desc or a state row holds.  A snapshot that cannot
 * be produced -- its final frames lie before the row's c0 or past c0 + max_new_frames, or n_snap is too short --
 * writes NaN to out[b]; n_snap <= 0 leaves out[b] alone.  Two items naming one state row race.  Two launches whatever
 * B (a ring STFT of each item's new and tail frames, then one CTA per item); the call only enqueues on `stream`, so it
 * can be captured in a CUDA graph once a call with the same B and max_new_frames has sized the workspace outside
 * capture (inside capture a larger workspace is OVC_ERR_STATE).  A checkpoint without ref_enc.* gives OVC_ERR_MISSING. */
OVC_API size_t ovc_reference_encoder_stream_state_floats(const ovc_ctx* ctx);
OVC_API int ovc_reference_encoder_stream(ovc_ctx* ctx, const float* rings, int ring_rows, int64_t ring_cap, float* state,
                                         int state_rows, const int64_t* desc, int B, int max_new_frames, float* out,
                                         void* stream);

/* Sample-rate conversion on the device, for waveforms that do not arrive at the model's rate (the reference resamples
 * every input on the host: librosa.load(path, sr=hps.data.sampling_rate), openvoice/api.py:123,144).  The arithmetic is
 * scipy.signal.resample_poly(x, up, down) at its defaults (Kaiser beta 5 window, 20 max(up, down) + 1 taps, constant
 * padding), up / down = sr_out / sr_in reduced; fp64 taps and accumulation, one rounding to fp32 -- within one ulp of
 * float32(resample_poly(float64(x))).  A rate that is not positive, or a reduced max(up, down) above 2048, is
 * OVC_ERR_INVALID (every common rate from 8 kHz to 192 kHz is accepted).  The context builds each pair's filter bank on
 * first use and keeps it: that first call uploads the bank on `stream` and waits for the stream to finish the copy.
 *   in          [B, in_pitch] fp32 (device): row b holds input samples [in_start, in_start + in_pitch) of item b
 *   in_lengths  [B] int64 (device): samples of item b's whole input; INT64_MAX = a stream that has not ended.  Samples
 *               outside [0, len) and outside the row read as 0
 *   out         [B, out_pitch] fp32 (device): row b receives y_b[out_start, out_start + out_pitch); outputs at or past
 *               n_out(len) = ceil(len * up / down) are written as 0
 * A whole-clip call has in_start = out_start = 0.  A windowed call gives the whole-clip samples bit for bit when its
 * rows hold every input sample the requested outputs read: ovc_resample_span says which.  Only enqueues on `stream`. */
OVC_API int ovc_resample(ovc_ctx* ctx, int sr_in, int sr_out, const float* in, const int64_t* in_lengths, int B,
                         int64_t in_pitch, int64_t in_start, float* out, int64_t out_pitch, int64_t out_start, void* stream);

/* Host-side geometry of ovc_resample for sr_in -> sr_out (no context, no device):
 *   out4[0] = n_out(n_in), output samples of a clip of n_in input samples
 *   out4[1] = outputs whose input support lies inside the first n_in samples (what a stream can emit before it ends)
 *   out4[2], out4[3] = input samples [lo, hi) read by outputs [m0, m1) (m1 > m0; lo may be negative) */
OVC_API int ovc_resample_span(int sr_in, int sr_out, int64_t n_in, int64_t m0, int64_t m1, int64_t* out4);

/* Build (once per context) the filter bank of sr_in -> sr_out and return its plan id in *id, for ovc_resample_rings.
 * The banks are those of ovc_resample (one per reduced pair, shared), and asking again for a pair returns the same id.
 * Uploads and waits for `stream`: call it at set-up, never inside a step.  Refuses the rates ovc_resample refuses
 * (OVC_ERR_INVALID). */
OVC_API int ovc_resample_plan(ovc_ctx* ctx, int sr_in, int sr_out, int32_t* id, void* stream);

/* ovc_resample for many live streams in one launch, each with its own plan: input from ring rows, output into ring
 * rows or a packed buffer.  Item b < B computes outputs [m0[b], m0[b] + count[b]) of plan plan[b] (an id of
 * ovc_resample_plan); it reads input sample j at in[in_row[b] * in_cap + j mod in_cap], zero outside [0, in_len[b])
 * (in_len INT64_MAX: a stream that has not ended), and writes output m at
 * out[out_row[b] * out_cap + (out_off[b] + m - m0[b]) mod out_cap].  out_off = m0 writes a ring row indexed by absolute
 * sample; an out_cap past every item's end makes `out` a packed buffer.  Outputs at or past n_out(in_len[b]) are
 * written as 0.
 *   plan                                          [B] int32 (device)
 *   in_row, in_len, m0, count, out_row, out_off   [B] int64 (device)
 *   in [in_rows, in_cap], out [out_rows, out_cap] fp32 (device); max_count bounds every count (the launch's width)
 * Every descriptor is clamped on the device, so nothing outside `in` and `out` is read or written whatever the arrays
 * hold: the plan id and rows into range, in_len to >= 0, m0 into [0, 2^63 / 16384], count into [0, max_count], out_off
 * mod out_cap.  Exactness: an output equals the whole-signal ovc_resample of the same stream bit for bit when its ring
 * row still holds every input sample that ovc_resample_span says it reads (and no other item writes where it reads).
 * Only enqueues on `stream` and takes stable pointers, so it can sit inside a captured graph. */
OVC_API int ovc_resample_rings(ovc_ctx* ctx, const int32_t* plan, const float* in, int in_rows, int64_t in_cap,
                               const int64_t* in_row, const int64_t* in_len, const int64_t* m0, const int64_t* count,
                               float* out, int out_rows, int64_t out_cap, const int64_t* out_row, const int64_t* out_off,
                               int B, int64_t max_count, void* stream);

/* ---- V1 base-speaker TTS front half: SynthesizerTrn.infer (openvoice/models.py:467-490), SURVEY.md section 8 row f3 ----
 * Available when the checkpoint passed through ovc_load_tensor holds enc_p.* / dp.* / sdp.* / emb_g.* (a V1 base
 * speaker, models.py:451-465); their hyper-parameters (n_vocab, heads, layers, window, filter sizes, n_speakers) are
 * read off the tensor shapes.  infer() is split where the reference itself synchronises (y_lengths -> mask sizes,
 * models.py:476-478):
 *
 *   ovc_tts_encode   x, m_p, logs_p = enc_p(tokens)                        models.py:468, 16-57; attentions.py:37-465
 *                    g = emb_g(sid)                                          models.py:470
 *                    logw = sdp(x, g, reverse) * ratio + dp(x, g) * (1 - ratio)   models.py:474-475, 60-180;
 *                                                                             modules.py:84-130, 459-516; transforms.py
 *                    w_ceil = ceil(exp(logw) * mask * length_scale); y_lengths = max(1, sum w_ceil)   models.py:477-479
 *   ovc_tts_decode   attn = generate_path(w_ceil); m_p, logs_p expanded; z_p = m_p + noise * exp(logs_p) * noise_scale;
 *                    z = flow(z_p, g, reverse); o = dec(z * y_mask, g)       models.py:480-490; commons.py:128-142
 *
 * tokens [B][T] int64 (padded), x_lengths [B] int64, sid [B] int64, noise_w [B][2][T] or NULL (Philox from `seed`);
 * y_lengths [B] int64 out; w_ceil / logw [B][T] optional outs.  All device pointers.  ovc_tts_decode uses the state the
 * last ovc_tts_encode left in the context: noise [B][inter][Ymax] or NULL (Philox), Ymax = max(y_lengths) (the
 * caller reads y_lengths back, as the reference does), max_len = the reference's max_len (0: none; the flow still runs
 * on all Ymax frames, only the generator is cut, models.py:489), ragged as in ovc_voice_conversion;
 * o [B][min(Ymax, max_len)*hop], z / z_p [B][inter][Ymax] optional.  ovc_tts_info: out8 = {has_tts, n_vocab, n_speakers, n_heads, n_layers, window, filter_channels, dp_filter}. */
OVC_API int ovc_tts_info(const ovc_ctx* ctx, int32_t* out8);
OVC_API int ovc_tts_encode(ovc_ctx* ctx, const int64_t* tokens, const int64_t* x_lengths, const int64_t* sid,
                           const float* noise_w, uint64_t seed, float noise_scale_w, float length_scale, float sdp_ratio,
                           int B, int T, int64_t* y_lengths, float* w_ceil, float* logw, void* stream);
OVC_API int ovc_tts_decode(ovc_ctx* ctx, const float* noise, uint64_t seed, float noise_scale, int B, int Ymax, int max_len,
                           int ragged, float* o, float* z, float* z_p, void* stream);
/* The two halves with per-item parameters (ovc_item_params; `items` a host pointer, NULL = none).  The Philox draws:
 * noise_w row r of item b = philox(key; stream, 0x7700 + r, t) with the encode key, z_p noise = philox(key; stream, c, y)
 * with the decode key (key = seed[b] or `seed`, stream = stream[b] or b).  Sentence j of a batch-1-per-request infer
 * with seed s is therefore reproduced inside any batch by seed = s (encode), s + 1 (decode), stream = j. */
OVC_API int ovc_tts_encode_items(ovc_ctx* ctx, const int64_t* tokens, const int64_t* x_lengths, const int64_t* sid,
                                 const float* noise_w, uint64_t seed, float noise_scale_w, float length_scale, float sdp_ratio,
                                 int B, int T, int64_t* y_lengths, float* w_ceil, float* logw, void* stream,
                                 const ovc_item_params* items);
OVC_API int ovc_tts_decode_items(ovc_ctx* ctx, const float* noise, uint64_t seed, float noise_scale, int B, int Ymax,
                                 int max_len, int ragged, float* o, float* z, float* z_p, void* stream,
                                 const ovc_item_params* items);

/* Duration fit: the encode with each fit group's length scale solved on the device, so that a run of rows (the
 * sentences of one request, say) lasts a given number of frames.  Group g is rows [row0[g], row1[g]) with a target of
 * target_frames[g] = F* frames.  Its frames at scale s are F(s) = sum over its rows of max(1, sum_t ceilf(expf(logw[t]) * s)),
 * the y_lengths the encode gives at length_scale = s, and its scale s* is the smallest float s in [scale_lo, scale_hi] with
 * F(s) >= F*, or scale_hi if there is none.  Every row of the group is then encoded at length_scale = s*, bit for bit as an
 * encode given s* as that row's per-item length_scale.  Rows outside every group keep the call's (or their per-item)
 * length_scale.  length_scale [B] receives every row's scale.  Device arrays are clamped on the device: row ranges into
 * [0, B), each to start at or after the previous group's end (groups never share a row), targets to at least 1.
 * The call only enqueues work. */
typedef struct ovc_tts_fit {
  const int64_t* row0;            /* [G], device: the group's first row */
  const int64_t* row1;            /* [G], device: one past its last row */
  const int64_t* target_frames;   /* [G], device */
  int G;                          /* 1 <= G <= B */
  float scale_lo, scale_hi;       /* 0 < scale_lo <= scale_hi, finite */
  float* length_scale;            /* [B], device out */
} ovc_tts_fit;
/* ovc_tts_encode_items / ovc_tts_encode_g with fit groups (`fit` a host pointer); exactly one of sid and g is given
 * (g_tokens as in ovc_tts_encode_g).  The ovc_tts_encode_state* calls and ovc_tts_decode work after it unchanged. */
OVC_API int ovc_tts_encode_fit(ovc_ctx* ctx, const int64_t* tokens, const int64_t* x_lengths, const int64_t* sid,
                               const float* g, int g_tokens, const float* noise_w, uint64_t seed, float noise_scale_w,
                               float length_scale, float sdp_ratio, int B, int T, int64_t* y_lengths, float* w_ceil,
                               float* logw, void* stream, const ovc_item_params* items, const ovc_tts_fit* fit);

/* Streaming decode: the decode half in time windows, from encode state the caller owns.
 *
 * ovc_tts_encode_state copies what the pending ovc_tts_encode left in the context into caller buffers (device to
 * device, only enqueued on `stream`): stats [B][T][2 inter] (m_p | logs_p per token), cum [B][T] int32 (cumulative
 * frame durations: token j covers frames [cum[j-1], cum[j])) and g [B][gin] (the speaker vectors emb_g(sid)).  Together
 * with the encode's y_lengths they are everything the decode reads, so a later ovc_tts_encode cannot disturb a decode
 * that uses the copies.
 *
 * ovc_tts_decode_windows decodes W windows of N such encoded rows (stats, cum, g, y_lengths [N], T as encoded).  Every
 * per-window value is a [W] device array:
 *   row          encoded row of window w (int64; clamped into [0, N))
 *   frame0, len  the window covers frames [frame0[w], frame0[w] + len[w]) of its row (int64)
 *   seed         decode key (uint64), stream (int64), noise_scale (float)
 * Window w's frame frame0[w] + t, t < len[w], is expanded exactly as the whole decode expands that frame: the token
 * of the absolute frame, the Philox draw at counter (key = seed[w]; stream[w], channel c, (frame0[w] + t) mod 2^32),
 * which is the whole decode's counter for that frame with the same key and stream (see ovc_tts_decode_items).  The flow
 * and the generator then run on the window alone, at its own length: the frames of it inside [0, y_lengths[row]),
 * at most Wmax.  A window [lo, hi) that extends its interior [e0, e1) by the decode's receptive field on both sides
 * (flow reverse +-32 frames, generator +-14; clipped at the row's ends) gives the whole decode's samples of
 * [e0, e1) to fp32 reordering; a window of the whole row gives them bit for bit.  Outputs:
 *   o    [W][hop * Wmax]      window w's samples, zero past hop * (its decode length)
 *   z_p  [W][inter][Wmax]     or NULL; the expanded prior sample, zero past the window's decode length
 * Frames outside the row, or past len[w], are zeros and nothing is read out of bounds whatever the arrays hold.  A call
 * that repeats its (W, Wmax, buffers, options) is replayed from a CUDA graph (OVC_OPT_GRAPH) and follows the arrays'
 * new contents.  Null buffers or non-positive sizes are OVC_ERR_INVALID. */
OVC_API int ovc_tts_encode_state(ovc_ctx* ctx, float* stats, int32_t* cum, float* g, void* stream);

/* Encode state written straight into rows of a pool: a grow-only set of N rows at token pitch Tp that holds the
 * sentences of many encodes (live streams whose text arrives over time), decoded together by ovc_tts_decode_windows with
 * (N, Tp) in place of (N, T).
 *
 * ovc_tts_encode_state_rows writes row b of the pending ovc_tts_encode (B rows of T tokens) into pool row dst_row[b]:
 * stats [N][Tp][2 inter], cum [N][Tp] int32, g [N][gin] and y_lengths [N] int64 (the encode's y_length of the row).
 * ovc_tts_state_rows does the same from caller-owned state (stats [B][T][2 inter], cum [B][T], g [B][gin],
 * y_lengths [B]), e.g. to re-pitch a pool into a larger one with dst_row = 0 .. B - 1.
 *
 * Padding rule.  Tokens T <= t < Tp of a pool row are filled as an encode fills the tokens of a short row inside its
 * batch: cum[t] = cum[T - 1] (the durations past a row's x_length are 0, so the cumulative sum stays put), and stats[t]
 * = 0 (an encode does not write a row's stats past its x_length; what lies there is never read for a row with frames).
 * ovc_tts_decode_windows finds frame f's token as the first t with cum[t] > f, so for every f < y_length the token, and
 * the samples, are those of the encode's own state bit for bit.  (A row whose durations all round to 0 has y_length 1
 * and expands its one frame from the last token of the pitch, padding included: with a larger pitch that token moves.)
 * Tokens t < T are copied as they are, including whatever the encode left past x_length.
 *
 *   dst_row  [B] int64 (device); clamped into [0, N) on the device, so nothing is written outside the pool whatever it
 *            holds.  Rows named twice get an unspecified one of their sources.
 * Tp < T, N < 1 or a null pointer is OVC_ERR_INVALID.  One grid-strided kernel; only enqueues on `stream` and takes
 * stable pointers, so it can sit inside a captured graph. */
OVC_API int ovc_tts_encode_state_rows(ovc_ctx* ctx, const int64_t* dst_row, int N, int Tp, float* stats, int32_t* cum,
                                      float* g, int64_t* y_lengths, void* stream);
OVC_API int ovc_tts_state_rows(ovc_ctx* ctx, const float* stats, const int32_t* cum, const float* g, const int64_t* y_lengths,
                               int B, int T, const int64_t* dst_row, int N, int Tp, float* d_stats, int32_t* d_cum,
                               float* d_g, int64_t* d_y_lengths, void* stream);

OVC_API int ovc_tts_decode_windows(ovc_ctx* ctx, const float* stats, const int32_t* cum, const float* g,
                                   const int64_t* y_lengths, int N, int T, const int64_t* row, const int64_t* frame0,
                                   const int64_t* len, int W, int Wmax, const uint64_t* seed, const int64_t* stream,
                                   const float* noise_scale, float* o, float* z_p, void* cuda_stream);

/* Speaking style from caller-supplied speaker vectors instead of emb_g(sid): blends of emb_g rows, or vectors that
 * change from token to token (every conditioning layer of the reference's dp / sdp / flow / dec is a 1x1 conv added to
 * per-token or per-frame activations, so each accepts g [B, gin, T]).
 *
 * ovc_tts_encode_g is ovc_tts_encode_items with `g` (device, fp32) in place of sid:
 *   g_tokens 0   g [B][gin], one vector per row.  Everything after the encode is the sid path with g = that vector;
 *                a row whose vector equals emb_g[id] gives the results of sid = id bit for bit.
 *   g_tokens 1   g [B][gin][T] (ovc_tone_track_expand's layout), token t of row b at g[(b * gin + c) * T + t].  The
 *                duration predictors add cond(g[b][:][t]) to token t (the same fmaf chain as the per-row vector, so a
 *                token whose vector equals the row's gets bit-identical values).  The decode expands g along the
 *                alignment path exactly as it expands m_p: frame y takes the vector of the token covering it, and
 *                frames no token covers (past y_length) take 0.  The flow reverse and the generator are then
 *                conditioned per frame; only their 6 656 target-side columns are computed per frame.
 * The context keeps its own copy of g, so the caller may reuse the buffer after the call.  ovc_tts_decode(_items)
 * needs nothing more.  Workspace: a per-token encode adds B * gin * T floats to the text-side workspace; its decode adds
 * B * Ymax * (gin + 6 656) floats (the per-frame vectors and their conditioning columns) to the decode workspace.
 *
 * After a per-token encode ovc_tts_encode_state and ovc_tts_encode_state_rows fail with OVC_ERR_STATE (their g holds
 * one vector per row); ovc_tts_encode_state_tokens copies the state with g [B][gin][T] instead, and fails with
 * OVC_ERR_STATE after any other encode.  ovc_tts_encode_state_rows_tokens / ovc_tts_state_rows_tokens are the pool
 * writes of ovc_tts_encode_state_rows / ovc_tts_state_rows with a per-token pool g [N][gin][Tp] (source g [B][gin][T]);
 * tokens T <= t < Tp get g = 0, as their stats.  A checkpoint whose generator ignores g (zero_g) refuses per-token
 * vectors with OVC_ERR_INVALID.  ovc_tts_decode_windows_tokens is ovc_tts_decode_windows on such state
 * (g [N][gin][T], T as encoded): window w's frame frame0[w] + t gets the vector the whole decode gives that frame, and
 * the same exactness rules hold.  Its workspace adds W * Wmax * (gin + 6 656) floats. */
OVC_API int ovc_tts_encode_g(ovc_ctx* ctx, const int64_t* tokens, const int64_t* x_lengths, const float* g, int g_tokens,
                             const float* noise_w, uint64_t seed, float noise_scale_w, float length_scale, float sdp_ratio,
                             int B, int T, int64_t* y_lengths, float* w_ceil, float* logw, void* stream,
                             const ovc_item_params* items);
OVC_API int ovc_tts_encode_state_tokens(ovc_ctx* ctx, float* stats, int32_t* cum, float* g, void* stream);
OVC_API int ovc_tts_encode_state_rows_tokens(ovc_ctx* ctx, const int64_t* dst_row, int N, int Tp, float* stats, int32_t* cum,
                                             float* g, int64_t* y_lengths, void* stream);
OVC_API int ovc_tts_state_rows_tokens(ovc_ctx* ctx, const float* stats, const int32_t* cum, const float* g,
                                      const int64_t* y_lengths, int B, int T, const int64_t* dst_row, int N, int Tp,
                                      float* d_stats, int32_t* d_cum, float* d_g, int64_t* d_y_lengths, void* stream);
OVC_API int ovc_tts_decode_windows_tokens(ovc_ctx* ctx, const float* stats, const int32_t* cum, const float* g,
                                          const int64_t* y_lengths, int N, int T, const int64_t* row, const int64_t* frame0,
                                          const int64_t* len, int W, int Wmax, const uint64_t* seed, const int64_t* stream,
                                          const float* noise_scale, float* o, float* z_p, void* cuda_stream);

/* Arithmetic of the convolutions (generator ResBlocks = 90 % of the FLOPs, WaveNet stacks, upsamplers):
 *   0            fp32 FFMA on the CUDA cores
 *   1 (default of the Python surface)  split-precision "3xFP16" on the Hopper tensor cores (wgmma):
 *                x = hi + lo / 2^11 with hi = fp16(x), lo = fp16((x - hi) * 2^11); every product is
 *                a_hi*b_hi + (a_lo*b_hi + a_hi*b_lo) / 2^11, fp32 accumulation, cross terms in their own
 *                accumulator -- fp32-grade error, same parity gate as mode 0.  Operands must be < 65504 in magnitude.
 *   2            single-pass fp16 on the tensor cores (11-bit operands): the precision class the REFERENCE itself
 *                gets on a GPU by default (cuDNN TF32, torch.backends.cudnn.allow_tf32 = True); own looser gate */
OVC_API int ovc_set_precision(ovc_ctx* ctx, int mode);

/* Tuning / diagnostics switches (never change results beyond fp32 reordering):
 *   OVC_OPT_TTS_SIMPLE    1: one-thread-per-element text-side kernels (the CPU-checked element functions) instead of
 *                         the warp-cooperative LayerNorm / fused attention
 *   OVC_OPT_GRAPH         1 (default): replay the launch sequence of a repeated (shape, buffers) call from a CUDA graph
 *   OVC_OPT_PDL           programmatic stream serialization of the tensor-core conv launches (the prologue of kernel n+1 --
 *                         barriers, weight TMA -- overlaps the drain of kernel n): 0 off, 1 all of them, 2 (default)
 *                         the WaveNet stacks only */
#define OVC_OPT_TTS_SIMPLE 2
#define OVC_OPT_GRAPH 3
#define OVC_OPT_PDL 5
#define OVC_OPT_BRANCHES 7   /* 1 (default): latency-bound calls (B * Tmax <= 512 frames) run the three ResBlock branches of an
                              * MRF stage concurrently (three streams, a third of the SMs per kernel); results are bit-identical */
#define OVC_OPT_PAIR 8       /* 1 (default): the HBM-bound ResBlock conv pairs (C <= 64, k = 3) run as ONE kernel each
                              * (tcconv_kernel<C, true>): the intermediate activation stays in shared memory */
#define OVC_OPT_PAIR_OCC 9   /* 1 (default): the conv pairs of the C = 32 / 64 stages run two CTAs per SM where that is
                              * measured faster (tc_pair_occ), so one tile's MMAs overlap another's epilogue; 0: one CTA
                              * per SM everywhere.  Results are bit-identical */
#define OVC_OPT_STAGED_EPI 10 /* 1 (default): the tensor-core convs of column tile 128 and the C = 128 conv pairs stage each
                               * tile's conv result in shared memory and a fourth warpgroup runs its epilogue (bias, residual,
                               * MRF accumulate, scale, stores) while the MMA warpgroups compute the next tile; 0: the MMA
                               * warpgroups run it themselves.  Applied where it is measured faster (split precision,
                               * k >= 5: tc_stage_pays).  Results are bit-identical */
OVC_API int ovc_set_option(ovc_ctx* ctx, int key, int value);

/* Number of kernels the last ovc_voice_conversion / ovc_convert_waveform call launched. */
OVC_API int ovc_last_launch_count(const ovc_ctx* ctx);

/* Number of ovc_voice_conversion / ovc_convert_waveform calls served by replaying a captured CUDA graph (OVC_OPT_GRAPH)
 * since the context was created.  A (shapes, buffers, options) signature is captured the second time it is seen and
 * replayed from the third call on; results are bit-identical to the directly launched sequence. */
OVC_API int ovc_graph_replays(const ovc_ctx* ctx);

/* Per-call timing hook for bench.py's roofline: when enabled, the dominant kernel family
 * (generator ResBlock convolutions) is bracketed with CUDA events on `stream`.  After the
 * stream has been synchronised, ovc_profile_read returns the accumulated milliseconds, the
 * number of launches, their algorithmic FLOPs and their algorithmic (layer-granular) bytes
 * since the last reset. */
OVC_API int ovc_profile_enable(ovc_ctx* ctx, int enable);
OVC_API int ovc_profile_read(ovc_ctx* ctx, double* ms, int64_t* launches, double* flops, double* bytes);
/* Per-launch detail of every conv kernel since the last reset (call before ovc_profile_read):
 * kernel-variant name (16 bytes each), milliseconds, algorithmic FLOPs / bytes, family (1 = generator
 * ResBlock convs).  Returns the number of entries written (<= max). */
OVC_API int ovc_profile_detail(ovc_ctx* ctx, int max, char* names, double* ms, double* flops, double* bytes,
                               int* family);

/* Debug taps (tests only): when enabled, named intermediate tensors of the next call are
 * copied aside; ovc_debug_fetch copies one to host memory.  Names: "enc.pre", "enc.wn",
 * "dec.pre", "dec.ups0".."dec.ups3", "dec.stage0".."dec.stage3", "cond". */
OVC_API int ovc_debug_enable(ovc_ctx* ctx, int enable);
OVC_API int ovc_debug_fetch(ovc_ctx* ctx, const char* name, float* host_out, size_t max_floats,
                    int64_t* shape4 /* B, C, T, pitch */);

#ifdef __cplusplus
}
#endif
#endif /* OVC_B200_H */

/* whisper_b200 — C ABI of the H100-native Whisper hot path.
 *
 * This is the thin extern-"C" layer BASELINE.json's north_star asks for: plain pointers and sizes, no C++ or torch types.
 * The COM-style iModel / iContext shells of the reference (include/whisper_b200_com.h) sit on top of it, exactly where the
 * reference's own back-ends sit behind Whisper/modelFactory.cpp:5-20.
 *
 * Each entry point names the reference interface it stands in for (paths relative to the reference tree):
 *   wsp_model_open            Whisper/Whisper/WhisperModel.cpp:434-492 (WhisperModel::load) == Whisper/source/whisper.cpp:451-1072
 *   wsp_engine_create         Whisper/Whisper/WhisperModel.cpp:257-340 (loadGpu: tensors -> VRAM)
 *   wsp_context_create        Whisper/Whisper/ModelImpl.cpp:14 (createContext), KV sizing Whisper/Whisper/WhisperContext.cpp:291-308
 *   wsp_pcm_to_mel            Whisper/source/whisper.h:97 whisper_pcm_to_mel      (Whisper/Whisper/Spectrogram.cpp:64-121)
 *   wsp_pcm_to_mel_window     Whisper/Whisper/MelStreamer.cpp:128-236 (MelStreamer::makeTransposedBuffer / makeBuffer: one window of a streamed clip)
 *   wsp_set_mel               Whisper/source/whisper.h:107 whisper_set_mel
 *   wsp_encode                Whisper/source/whisper.h:117 whisper_encode          (Whisper/Whisper/WhisperContext.cpp:310 encode)
 *   wsp_set_audio_ctx         Whisper/API/sFullParams.h:75 sFullParams::audio_ctx  (whisper_context::exp_n_audio_ctx, Whisper/source/whisper.cpp:2836)
 *   wsp_set_speed_up          Whisper/API/sFullParams.h:33 eFullParamsFlags::SpeedupAudio (whisper_pcm_to_mel_phase_vocoder, Whisper/source/whisper.cpp:2299-2311)
 *   wsp_decode                Whisper/source/whisper.h:128 whisper_decode + :140-150 whisper_sample_best/timestamp
 *                             (Whisper/Whisper/WhisperContext.cpp:578 decode, Whisper/Whisper/ContextImpl.cpp:71-157 sampleBest)
 *   wsp_get_logits/probs      Whisper/source/whisper.h:166 whisper_get_probs
 *   wsp_run_chunks            the fixed-length greedy chunk loop of BASELINE.md §2 (mel + encode + n_decode x (decode + sample))
 *   wsp_run_chunks_until_eot  the same loop, each chunk cut at its first EOT and the batch stopped soon after its last one
 *   wsp_get_chunk_languages   whisper_lang_auto_detect (Whisper/source/whisper.cpp:2428-2495) per chunk of a run_chunks* call
 *   wsp_run_chunks_window     the same loop, each chunk decoded and ended as whisper_full's first window (whisper.cpp:2910-3003)
 *   wsp_run_spans_window      the same, each row whisper_full's first window at a span's offset_ms / duration_ms (whisper.cpp:2810-2818)
 *   wsp_window_segments       whisper_full's segments of one window (whisper.cpp:3026-3119)
 *   wsp_set_token_timestamps  whisper_full_params::token_timestamps (Whisper/API/sFullParams.h eFullParamsFlags::TokenTimestamps): the
 *                             signal energy of get_signal_energy (whisper.cpp:3356-3372), computed on the device
 *   wsp_window_token_times    those segments with whisper_full's token times (whisper.cpp:3374-3600) and max_len wrapping (:2713-2763)
 *   wsp_upload_pcm_stereo     a stereo chunk, downmixed on the device as Whisper/MF/AudioBuffer.cpp:57-93 (appendDownmixedStereo)
 *   wsp_chunk_speakers        iContext::detectSpeaker (Whisper/Whisper/ContextImpl.diarize.cpp:73-108) for every segment of a batch
 *   wsp_get_tensor            the reference's named trace points, Whisper/Utils/Trace/tracing.h (names as in whisper.cpp:1121-1869)
 *
 * Error handling mirrors the reference's HRESULT convention (SURVEY.md §8b): every function returns a wsp_status that the COM
 * shell maps 1:1 to an HRESULT; no exception crosses this boundary.  There is NO CPU fallback: if the CUDA device or the
 * sm_90a kernels are unavailable the calls fail with WSP_E_CUDA.
 *
 * Threading: a wsp_model / wsp_engine is immutable after creation and may be shared; a wsp_context is single-threaded state
 * (KV memories, workspaces), one per concurrent stream — the same contract as iModel / iContext (Whisper/Whisper/WhisperModel.h:28-31).
 */
#ifndef WHISPER_B200_H
#define WHISPER_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef int32_t wsp_status;
enum
{
	WSP_OK = 0,
	WSP_S_FALSE = 1,          /* "did nothing" (S_FALSE) */
	WSP_E_INVALIDARG = -1,
	WSP_E_POINTER = -2,
	WSP_E_FILE = -3,          /* cannot open / truncated */
	WSP_E_FORMAT = -4,        /* not a ggml whisper file, missing or mis-shaped tensors */
	WSP_E_CUDA = -5,          /* CUDA runtime / driver failure, or no sm_90a device */
	WSP_E_OUTOFMEMORY = -6,
	WSP_E_BOUNDS = -7,        /* batch, token count or context length beyond what the context was created for */
	WSP_E_NOTIMPL = -8,
};

typedef struct wsp_model wsp_model;
typedef struct wsp_engine wsp_engine;
typedef struct wsp_context wsp_context;

/* whisper_token_data (Whisper/source/whisper.h:71-85) without the token-level timestamp fields */
typedef struct wsp_token_data
{
	int32_t id;      /* sampled token */
	int32_t tid;     /* most probable timestamp token */
	float p;         /* probability of `id` */
	float pt;        /* probability of `tid` among timestamp tokens */
	float ptsum;     /* total probability of all timestamp tokens */
} wsp_token_data;

/* decode flags */
enum
{
	WSP_DECODE_FORCE_TIMESTAMP = 1,   /* whisper_sample_timestamp */
	WSP_DECODE_INITIAL = 2,           /* is_initial: first timestamp <= 1.00 s */
	WSP_DECODE_ALL_LOGITS = 4,        /* keep logits/probs for every prompt token (n_tokens <= 8), as the oracle does */
	WSP_DECODE_DEVICE_TOKENS = 8,     /* feed the tokens sampled by the previous call (no host round trip); n_past continues */
	WSP_DECODE_NO_SAMPLE = 16,
};

/* ---- library ---- */
const char* wsp_version( void );
const char* wsp_last_error( void );              /* thread-local text of the last failure */
int32_t wsp_device_count( void );
wsp_status wsp_device_name( int32_t device, char* dst, size_t cap );   /* replaces listGPUs (Whisper/D3D/listGPUs.cpp) */
/* number of kernels this library has launched since load (bench.py's gpu_launches evidence) */
uint64_t wsp_launch_count( void );

/* ---- model file (host) ---- */
wsp_status wsp_model_open( const char* path_utf8, wsp_model** out );
void wsp_model_close( wsp_model* m );
/* n_vocab, n_audio_ctx, n_audio_state, n_audio_head, n_audio_layer, n_text_ctx, n_text_state, n_text_head, n_text_layer, n_mels, f16 */
wsp_status wsp_model_hparams( const wsp_model* m, int32_t out11[ 11 ] );
/* eot, sot, prev, solm, not, beg, translate, transcribe */
wsp_status wsp_model_special_tokens( const wsp_model* m, int32_t out8[ 8 ] );
const char* wsp_model_token_text( const wsp_model* m, int32_t id );
int32_t wsp_model_is_multilingual( const wsp_model* m );
/* raw file image, for broadcasting to peer GPUs before wsp_engine_create_from_image */
const void* wsp_model_file_data( const wsp_model* m, uint64_t* size );
/* the small host-side part (hparams, filters, vocabulary, tensor directory) as a relocatable blob */
wsp_status wsp_model_meta_serialize( const wsp_model* m, void* dst, uint64_t cap, uint64_t* size );
wsp_status wsp_model_from_meta( const void* meta, uint64_t size, wsp_model** out );

/* ---- engine: weights resident on one device ---- */
wsp_status wsp_engine_create( const wsp_model* m, int32_t device, wsp_engine** out );
/* same, but the tensor data is taken from a device-resident copy of the file image (e.g. received by an NCCL broadcast) */
wsp_status wsp_engine_create_from_image( const wsp_model* m, int32_t device, const void* dev_file_image, uint64_t size, wsp_engine** out );
void wsp_engine_destroy( wsp_engine* e );
uint64_t wsp_engine_weight_bytes( const wsp_engine* e );

/* ---- context: per-stream state for up to max_batch independent 30 s chunks ---- */
wsp_status wsp_context_create( wsp_engine* e, int32_t max_batch, wsp_context** out );
void wsp_context_destroy( wsp_context* c );
wsp_status wsp_synchronize( wsp_context* c );
/* device memory held by the context: workspaces, KV caches, mel slots (ContextImpl::getMemoryUse, Whisper/Whisper/ContextImpl.misc.cpp:170-182) */
uint64_t wsp_context_device_bytes( const wsp_context* c );

/* a1: 16 kHz mono f32 PCM (host) -> log-mel of chunk slot `slot`, kept on the device.  n_len = n_samples / 160 frames
 * (n_samples / 320 with wsp_set_speed_up). */
wsp_status wsp_pcm_to_mel( wsp_context* c, int32_t slot, const float* pcm, int32_t n_samples );
/* a1, streamed flavour (iContext::runStreamed): log-mel of frames [0, n_frames) of `pcm` — which should extend 240 samples past the
 * last frame unless the stream ends there — normalised by the maximum over these frames only, floored at 1e-20; `forced_max` (may be
 * NULL) replaces that maximum, `max_out` (may be NULL) receives the maximum found.  The slot then holds n_frames frames. */
wsp_status wsp_pcm_to_mel_window( wsp_context* c, int32_t slot, const float* pcm, int32_t n_samples, int32_t n_frames, const float* forced_max, float* max_out );
wsp_status wsp_set_mel( wsp_context* c, int32_t slot, const float* mel, int32_t n_len );     /* [80][n_len] */
int32_t wsp_mel_len( wsp_context* c, int32_t slot );
wsp_status wsp_get_mel( wsp_context* c, int32_t slot, float* dst, size_t cap_floats );

/* a2-a12: encoder + cross-KV for slots [0,batch); mel_offsets[b] = first frame of the 2n-frame window (NULL = 0), n = the audio context below */
wsp_status wsp_encode( wsp_context* c, const int32_t* mel_offsets, int32_t batch );

/* sFullParams::audio_ctx (Whisper/API/sFullParams.h:75): encode only the first n of the model's n_audio_ctx (1500) audio positions.
 * As in the reference (whisper.cpp:1092-1167, 1479-1480, 1528; Whisper/Whisper/ContextImpl.cpp:24, 55, 489), the encoder then reads mel
 * frames [offset, offset + 2n) — zero past the clip's end — convolves them with zero padding at frame 2n, adds the first n rows of the
 * positional embedding and attends over n keys; the cross-K/V memories hold n rows per layer and every decoder cross-attention runs
 * over those n keys.  Encoder work and cross-KV traffic fall in proportion to n.
 * n <= 0 selects the default (n_audio_ctx); n > n_audio_ctx is WSP_E_INVALIDARG (the reference does not check it and would read past
 * its positional table).  The value is context state and takes effect at the next wsp_encode, wsp_run_chunks* or wsp_detect_language;
 * every decode attends over the n of the last encode, so the cross-KV layout and the decoder always agree.  wsp_get_tensor shapes
 * follow that encode: "enc.input" [2n][80], "enc.conv1" [2n][d], "enc.x" / "encode-out" [n][d], "cross_k" / "cross_v" [L][H][n][64]. */
wsp_status wsp_set_audio_ctx( wsp_context* c, int32_t n );

/* whisper_full_params::speed_up (Whisper/API/sFullParams.h:33 eFullParamsFlags::SpeedupAudio): on = 1 computes whole-clip log-mels with
 * the reference's phase vocoder, whisper_pcm_to_mel_phase_vocoder (Whisper/source/whisper.cpp:2299-2311, 2060-2181 with speed_up): an
 * 800-point Hann window and transform every 320 samples, the power spectrum's adjacent bins averaged back onto the model's 201 bins.
 * The spectrum is compressed 2x in frequency, so the mel reads like audio played twice as fast: n_len = n_samples / 320 frames and one
 * 3000-frame encoder window covers 60 s of audio (reduced accuracy, as the reference's -su option says).  on = 0 (the default) is the
 * 400-point transform; any other value is WSP_E_INVALIDARG.  The value is context state and takes effect at the next log-mel of
 * wsp_pcm_to_mel, wsp_run_chunks and wsp_run_chunks_resident; wsp_mel_len, wsp_get_mel and wsp_get_tensor("mel") follow that mel.
 * While it is on, wsp_pcm_to_mel_window returns WSP_E_NOTIMPL (the reference has no streamed phase-vocoder window); wsp_set_mel is
 * unaffected. */
wsp_status wsp_set_speed_up( wsp_context* c, int32_t on );

/* a13-a18: one decoder call for `batch` chunks, n_tokens new tokens each (tokens[b*n_tokens + i]), after n_past cached ones.
 * sampled (nullable) receives the greedy choice per chunk from the last token's distribution. */
wsp_status wsp_decode( wsp_context* c, const int32_t* tokens, int32_t n_tokens, int32_t n_past, int32_t batch, uint32_t flags, wsp_token_data* sampled );
/* logits / probabilities of the last wsp_decode: [batch][n_vocab], or [batch*n_tokens][n_vocab] after WSP_DECODE_ALL_LOGITS */
wsp_status wsp_get_logits( wsp_context* c, float* dst, size_t cap_floats );
wsp_status wsp_get_probs( wsp_context* c, float* dst, size_t cap_floats );

/* whisper_lang_auto_detect (Whisper/source/whisper.cpp:2428-2495): encode slot 0's window at mel frame `offset_frames`, decode [sot],
 * then — like the reference — a softmax over the language tokens' PROBABILITIES; lang_probs[n_langs] (nullable), *lang_id = the arg-max */
wsp_status wsp_detect_language( wsp_context* c, int32_t offset_frames, int32_t n_langs, float* lang_probs, int32_t* lang_id );

/* Prompt token of wsp_run_chunks, wsp_run_chunks_resident and wsp_run_chunks_until_eot (and of wsp_replicas_run_chunks, which passes
 * its prompt through): "detect this chunk's language".  A prompt may hold it at most once, e.g. [sot, WSP_TOKEN_LANGUAGE_AUTO, transcribe].
 * The call then detects each chunk's language from that chunk's own encode, as whisper_lang_auto_detect does at offset 0 (one decoder
 * pass over [sot] for the whole batch, the reference's softmax over the language tokens' probabilities, arg-max), and decodes chunk b
 * with the sentinel replaced by its language token sot + 1 + lang_b.  The languages considered are the n_langs = translate - sot - 1
 * tokens after sot (99 on the multilingual vocabulary); on a model that is not multilingual the sentinel is WSP_E_INVALIDARG.  Detection
 * sees the context's current audio_ctx and speed-up, like the batch's own encode; stage_ms[2] includes it.  Every other prompt id
 * must satisfy 0 <= id < n_vocab, else the call is WSP_E_INVALIDARG and launches nothing. */
enum { WSP_TOKEN_LANGUAGE_AUTO = -1 };

/* The measured path: for `batch` chunks of host PCM — mel, encode, then n_decode greedy steps (first step samples with
 * is_initial timestamp rules, as whisper_full does, whisper.cpp:2943) entirely on the device with sampled tokens fed back
 * without host round trips.  tokens_out[b*n_decode + i].  stage_ms (nullable): { h2d+mel, encode, decode } from CUDA events. */
wsp_status wsp_run_chunks( wsp_context* c, const float* const* pcm, const int32_t* n_samples, int32_t batch,
	const int32_t* prompt, int32_t n_prompt, int32_t n_decode, int32_t* tokens_out, float* stage_ms );
/* keep a chunk's PCM resident in HBM (slot-owned copy) ... */
wsp_status wsp_upload_pcm( wsp_context* c, int32_t slot, const float* pcm, int32_t n_samples );
/* ... and run the same path from it: mel + encode + decode with no host->device input copy inside (bench.py's `value` leg) */
wsp_status wsp_run_chunks_resident( wsp_context* c, int32_t batch, const int32_t* prompt, int32_t n_prompt, int32_t n_decode, int32_t* tokens_out, float* stage_ms );
/* The batch path of wsp_run_chunks, ending each chunk at its first EOT: chunk b's output is its greedy tokens up to and including
 * the first EOT, or max_decode tokens if it samples none; n_out[b] = that count; tokens_out[b*max_decode + i] for i < n_out[b]
 * (tokens_out may be NULL; entries past n_out[b] are not written).  EOT and max_decode are the only stop rules: whisper_full's others
 * (a timestamp past the window's end, max_tokens) do not apply here; wsp_run_chunks_window applies them.  A chunk that has ended stays in the batch and keeps being decoded
 * until the batch stops; its later tokens are not part of its output.  The steps go out in blocks of 8 and the host reads the
 * number of ended chunks one block behind, so the batch stops at most 16 steps after its last chunk's EOT.
 * pcm == NULL runs from the slots' resident PCM (wsp_upload_pcm), as wsp_run_chunks_resident does; otherwise n_samples is required.
 * Bounds, errors and stage_ms are those of wsp_run_chunks; stage_ms[2] covers the steps actually run, and afterwards wsp_get_logits
 * and wsp_get_tensor("self_k" / "self_v") hold the state of the last of them. */
wsp_status wsp_run_chunks_until_eot( wsp_context* c, const float* const* pcm, const int32_t* n_samples, int32_t batch,
	const int32_t* prompt, int32_t n_prompt, int32_t max_decode, int32_t* tokens_out, int32_t* n_out, float* stage_ms );
/* The languages the last wsp_run_chunks* call on this context detected, when its prompt held WSP_TOKEN_LANGUAGE_AUTO: lang_ids[batch]
 * as wsp_detect_language reports them (0 = en; chunk b's language token is sot + 1 + lang_ids[b]) and, if lang_probs is not NULL,
 * lang_probs[b*n_langs + l] for b < batch, which needs cap_floats >= batch * n_langs.  They come back with that call's tokens.
 * WSP_S_FALSE, writing nothing, when that call had no sentinel (or there was none); WSP_E_BOUNDS for a batch above that call's or a
 * short cap_floats. */
wsp_status wsp_get_chunk_languages( wsp_context* c, int32_t batch, int32_t* lang_ids, float* lang_probs, size_t cap_floats );

/* ---- whisper_full's first window on the batch path ---- */
typedef struct wsp_window_params
{
	int32_t max_tokens;       /* whisper_full_params::max_tokens: a segment ends after token max_tokens (<= 0: no limit) */
	int32_t single_segment;   /* whisper_full_params::single_segment */
} wsp_window_params;
typedef struct wsp_window_result
{
	int32_t n_sampled;        /* tokens the window sampled, a token that went back in time included */
	int32_t n_tokens;         /* result_len: the first n_tokens of them are the window's result */
	int32_t seek_delta;       /* frames the window advances by */
	int32_t failed;           /* no usable timestamp (whisper.cpp:2977, 3000-3003): whisper_full drops the window */
} wsp_window_result;
/* The batch path of wsp_run_chunks, with each chunk decoded as whisper_full decodes its first window (Whisper/source/whisper.cpp:
 * 2910-3003): a window at seek 0 over the chunk's n_len = wsp_mel_len frames (n_samples / 160, or / 320 under speed-up), ended by
 * EOT, by max_tokens, by a timestamp at or past n_len - 100 frames, by a timestamp that goes back in time, or after n_max =
 * n_text_ctx / 2 - 4 tokens, where it fails unless it holds a timestamp of at least 15 s.  Every chunk keeps the one caller prompt,
 * as whisper_full's first window does with no prompt past.  Chunk b's tokens with their probabilities go to tokens_out[b*cap + i]
 * for i < results[b].n_sampled (tokens_out may be NULL; cap >= n_max, else WSP_E_BOUNDS).  A chunk of at most 100 frames runs no
 * window (whisper.cpp:2871): its result is all zeros.  The batch never runs more than n_max steps and stops at most 16 steps after
 * its last window ends.  pcm == NULL runs from the slots' resident PCM; the prompt may hold WSP_TOKEN_LANGUAGE_AUTO; audio_ctx and
 * speed-up apply as they do to wsp_run_chunks.  Every argument is checked before anything is enqueued; stage_ms as in
 * wsp_run_chunks_until_eot. */
wsp_status wsp_run_chunks_window( wsp_context* c, const float* const* pcm, const int32_t* n_samples, int32_t batch, const int32_t* prompt,
	int32_t n_prompt, const wsp_window_params* params, wsp_token_data* tokens_out, int32_t cap, wsp_window_result* results, float* stage_ms );

/* A time interval of a resident clip: whisper_full_params::offset_ms and duration_ms (sFullParams.h:51-52) of slot `slot`'s PCM. */
typedef struct wsp_window_span
{
	int32_t slot;             /* the source: the slot's resident PCM (wsp_upload_pcm, or the downmix of wsp_upload_pcm_stereo) */
	int32_t offset_ms;        /* >= 0 */
	int32_t duration_ms;      /* 0: to the end of the clip; < 0: no window, as in the reference */
} wsp_window_span;
/* wsp_run_chunks_window over spans: row b is the first window of whisper_full( the clip of spans[b].slot, offset_ms, duration_ms ) with
 * no past prompt (whisper.cpp:2810-2818, 2910-3003).  With n_len = the whole clip's mel length (n_samples / 160, or / 320 under
 * speed-up), seek = offset_ms / 10 and seek_end = seek + (duration_ms == 0 ? n_len : duration_ms / 10):
 *   - a row with seek_end <= seek + 100 runs no window (:2816, 2871): its result is all zeros;
 *   - the row's encode reads frames [seek, seek + 2n) of the source's whole-clip log-mel, normalised over the whole clip, frames past
 *     n_len zero (:1112-1120): the encoder sees the audio past seek_end, as the reference's does;
 *   - the window rule runs at seek over seek_end, and wsp_window_segments( ..., seek, ... ) gives the row's segments at absolute times
 *     in the clip (:3028, 3042).
 * Under speed-up seek and seek_end count frames at the vocoder's hop of 320 samples, as in the reference: an offset then lands at twice
 * its time in the clip, and segment times are doubled.  Rows naming one slot share its log-mel, and its signal energy while token
 * timestamps are on: each named slot's are computed once per call, in the batched launches of wsp_run_chunks_window, and a slot no row
 * names is not touched.  WSP_TOKEN_LANGUAGE_AUTO detects each row's language from the row's own encode, as whisper_lang_auto_detect(
 * offset_ms ) does (:2428-2495); whisper_full itself detects at offset 0 whatever offset_ms is (:2792), so a row gets the language
 * spoken in its span.  Every row keeps the one caller prompt and n_past.  Outputs, cap, stage_ms, audio_ctx and the other settings are
 * those of wsp_run_chunks_window.  Every argument is checked before anything is enqueued, and an error launches nothing: a null
 * pointer is WSP_E_POINTER (tokens_out and stage_ms may be NULL); a batch outside [1, max_batch] or a slot outside max_batch
 * WSP_E_BOUNDS; a slot without resident PCM, a negative offset_ms (undefined in the reference, which reads before the mel) or the
 * sentinel on a row whose seek is at or past its source's n_len (the reference's -2, :2440-2443) WSP_E_INVALIDARG.  The seek
 * arithmetic cannot overflow int32: each of its terms is below 2^31 / 10. */
wsp_status wsp_run_spans_window( wsp_context* c, const wsp_window_span* spans, int32_t batch, const int32_t* prompt, int32_t n_prompt,
	const wsp_window_params* params, wsp_token_data* tokens_out, int32_t cap, wsp_window_result* results, float* stage_ms );

/* segmentation flags */
enum
{
	WSP_SEGMENT_SINGLE = 1,          /* whisper_full_params::single_segment: timestamps do not split */
	WSP_SEGMENT_PRINT_SPECIAL = 2,   /* print_special: special tokens count as text */
	WSP_SEGMENT_SPEED_UP = 4,        /* speed_up: times are doubled (whisper.cpp:3044, 3088) */
};
typedef struct wsp_segment
{
	int64_t t0, t1;           /* 10 ms units */
	int32_t i0, i1;           /* the segment's tokens are [i0, i1) of the window's */
} wsp_segment;
/* Host only: whisper_full's segments of one window at `seek` (whisper.cpp:3026-3119), from its result and its first result->n_tokens
 * tokens.  A timestamp token closes a segment unless single-segment; consecutive timestamps are skipped, and a segment is emitted only
 * if its text is not empty.  A segment's text is the text of its tokens [i0, i1), special tokens (id >= eot) left out unless
 * WSP_SEGMENT_PRINT_SPECIAL.  A failed window has none.  *n_segs = the number of segments; the first min(*n_segs, cap) are written
 * (segs may be NULL when cap is 0), and more than cap is WSP_E_BOUNDS.  n_tokens + 1 always suffices. */
wsp_status wsp_window_segments( const wsp_model* m, const wsp_token_data* tokens, const wsp_window_result* result, int32_t seek,
	uint32_t flags, wsp_segment* segs, int32_t cap, int32_t* n_segs );

/* ---- token-level timestamps of whisper_full's first window on the batch path ---- */
/* whisper_full_params::token_timestamps.  on = 1 makes the signal energy of get_signal_energy (whisper.cpp:3356-3372) context state:
 * e[i] = (sum over j = -32..32 with 0 <= i + j < n of |x[i + j]|) / 65, summed in f32 in that order, bit-identical to the reference.
 * While it is on, wsp_run_chunks_window computes it on the device for every chunk of its batch, from the PCM the call used (host or
 * resident; under speed-up the original samples), right after the log-mel and inside stage_ms[0], and brings it back with the call's
 * tokens; wsp_pcm_to_mel computes it for its slot.  wsp_get_tensor("energy", slot) returns it.  on = 0 (the default) changes nothing
 * in any call; any other value is WSP_E_INVALIDARG. */
wsp_status wsp_set_token_timestamps( wsp_context* c, int32_t on );
typedef struct wsp_token_time
{
	int64_t t0, t1;           /* whisper_token_data::t0 / t1, 10 ms units; -1 for a token outside every segment */
	float vlen;               /* whisper_token_data::vlen: voice length of the token's text */
} wsp_token_time;
typedef struct wsp_token_time_params
{
	float thold_pt;           /* whisper_full_params::thold_pt (default 0.01) */
	float thold_ptsum;        /* whisper_full_params::thold_ptsum (default 0.01) */
	int32_t max_len;          /* whisper_full_params::max_len: wrap segments at this many characters (<= 0: no wrapping) */
} wsp_token_time_params;
/* Host only: chunk `chunk`'s segments of this context's last wsp_run_chunks_window or wsp_run_spans_window call as whisper_full emits
 * them with token_timestamps on.  tokens and result are that call's for the chunk, flags as for wsp_window_segments.  The window is
 * cut by wsp_window_segments at the chunk's seek (0, or a span's offset_ms / 10, so times are absolute in the clip); then, segment by
 * segment in order and from the state whisper_full starts a call with (t_beg = t_last = 0, :2803-2808), the token times of
 * whisper.cpp:3374-3600 run over the signal energy of the chunk's whole clip, clamped at its last sample (:3320-3322): a span's first
 * segment that does not open with beg reads energy before the span.  A spans call keeps each source's energy in the row of its slot
 * of [max_batch][longest clip] f32 on the device and again in pinned host memory, so an hour-long source costs
 * max_batch x 57.6 M samples x 4 B in each.  With max_len > 0 each segment is wrapped right after its token
 * times (:3063-3070, 3107-3114).  Under WSP_SEGMENT_SPEED_UP this is what the reference does: segment times are doubled, the
 * timestamp token times t_beg + 2 (tid - beg) are not, and the energy is that of the original samples.  segs receives the segments
 * after wrapping, the first min(*n_segs, cap) of them (a segment's text is that of its non-special tokens once wrapped);
 * times[i] = window token i's times for i < result->n_tokens.  A failed window, or a chunk of at most 100 frames, has no segments.
 * Errors, checked before anything is written: WSP_E_POINTER for a null pointer (tokens and times may be NULL only when the window
 * has no result tokens), WSP_E_INVALIDARG when the last window call ran with the energy off or there was none, WSP_E_BOUNDS for a
 * chunk outside that call's batch or, with *n_segs set, more segments than cap. */
wsp_status wsp_window_token_times( wsp_context* c, int32_t chunk, const wsp_token_data* tokens, const wsp_window_result* result,
	uint32_t flags, const wsp_token_time_params* p, wsp_segment* segs, int32_t cap, int32_t* n_segs, wsp_token_time* times );

/* ---- stereo chunks and per-segment speakers on the batch path (iContext::detectSpeaker, the CLI's --diarize) ---- */
/* Interleaved 16 kHz f32 stereo lr[n_frames][2] (left, right) into slot `slot`: the pairs are kept on the device, and one kernel launch
 * writes the slot's resident mono PCM as (l + r) * 0.5f per frame, AudioBuffer::appendDownmixedStereo's mix (Whisper/MF/AudioBuffer.cpp:
 * 57-93) and the one the WAV reader gives runFull for two channels, bit for bit.  wsp_run_chunks_resident, and wsp_run_chunks_until_eot /
 * wsp_run_chunks_window with pcm == NULL, then run from that mono exactly as after wsp_upload_pcm of it (language sentinel, audio_ctx,
 * speed-up and token timestamps included).  Returns once the slot holds the data.  The pairs stay the slot's stereo until the next
 * wsp_upload_pcm_stereo or wsp_upload_pcm to the slot: wsp_upload_pcm drops them.  Their device memory counts in
 * wsp_context_device_bytes.  lr may be NULL when n_frames is 0; a slot outside max_batch is WSP_E_BOUNDS, a negative n_frames
 * WSP_E_INVALIDARG. */
wsp_status wsp_upload_pcm_stereo( wsp_context* c, int32_t slot, const float* lr, int32_t n_frames );
/* iContext::detectSpeaker's answers (Whisper/Whisper/ContextImpl.diarize.cpp:73-108), the values of eSpeakerChannel */
enum
{
	WSP_SPEAKER_UNSURE = 0,
	WSP_SPEAKER_LEFT = 1,
	WSP_SPEAKER_RIGHT = 2,
	WSP_SPEAKER_NO_STEREO = 255,
	WSP_SPEAKER_OUT_OF_RANGE = -1,   /* the segment starts outside the clip: the reference's E_BOUNDS (Spectrogram.cpp:142-168) */
};
/* The speaker of every segment of a batch, as detectSpeaker answers it for the clip alone, bit for bit, in one kernel launch with one
 * copy in and one copy out.  Chunk b's segments are segs[seg_start[b] .. seg_start[b + 1]) and are read against slot b's stereo;
 * speakers[i] receives segment i's answer.  The segments are whatever the caller emits for the chunk, wsp_window_segments or the wrapped
 * segments of wsp_window_token_times: t0 / t1 in 10 ms units from the chunk's start (under speed-up already doubled, so real time over
 * the original samples).  For a segment with begin = t0, end = t1:
 *   end - begin <= 0                                   WSP_SPEAKER_UNSURE
 *   else, slot b holds no stereo (or none of n_frames)  WSP_SPEAKER_NO_STEREO
 *   else, begin < 0 or begin * 160 >= n_frames          WSP_SPEAKER_OUT_OF_RANGE
 *   else the frames [begin * 160, end * 160) cut at the end of the clip (the reference's zero fill after it adds nothing): |L| and |R|
 *   are summed in the reference's SSE lane order, even frames and odd frames in separate f32 accumulators, each a chain in frame order,
 *   then left = L even + L odd and right = R even + R odd (ContextImpl.diarize.cpp:17-52), and the answer is
 *   (left > right * 1.1f) | (right > left * 1.1f) << 1 (:54-70): WSP_SPEAKER_LEFT, WSP_SPEAKER_RIGHT or WSP_SPEAKER_UNSURE.
 * The chains are kept as chains on the device: a pairwise sum would round differently and move decisions within rounding of 1.1.
 * Every argument is checked before anything is enqueued: a null pointer is WSP_E_POINTER (segs may be NULL when seg_start[batch] is 0),
 * seg_start[0] != 0 or a decreasing seg_start is WSP_E_INVALIDARG, a batch outside [1, max_batch] is WSP_E_BOUNDS.  A batch without
 * segments launches nothing. */
wsp_status wsp_chunk_speakers( wsp_context* c, int32_t batch, const int32_t* seg_start, const wsp_segment* segs, int32_t* speakers );

/* ---- several devices in one process (csrc/replicas.cpp) ----
 * Chunks are independent (SURVEY.md §8e): one engine + context per listed device (a device may be listed twice: two contexts on one
 * GPU), the model file read ONCE and its image copied device-to-device from devices[0] (cudaMemcpyPeer over NVLink) — the C++ form of
 * bench.py's NCCL broadcast; reference analogues: iModel::clone (Whisper/Whisper/ModelImpl.cpp:40-60), whisper_full_parallel
 * (Whisper/source/whisper.cpp:3127-3268). */
typedef struct wsp_replicas wsp_replicas;
typedef struct wsp_replica_stats
{
	int32_t device;
	int32_t batches_done, chunks_done;
	int32_t failed;          /* the replica returned an error and was retired; its batch went back to the queue */
	float busy_ms;           /* host wall time spent inside wsp_run_chunks */
	float load_ms;           /* engine + context creation, including the image copy */
} wsp_replica_stats;
wsp_status wsp_replicas_create( const wsp_model* m, const int32_t* devices, int32_t n_devices, int32_t max_batch, wsp_replicas** out );
int32_t wsp_replicas_count( const wsp_replicas* r );
/* n_chunks clips through a host work queue: batches of <= max_batch chunks go to whichever replica is free; a batch whose replica fails
 * is re-queued for the others.  tokens_out[chunk * n_decode + i]; stats (nullable) [n_devices]. */
wsp_status wsp_replicas_run_chunks( wsp_replicas* r, const float* const* pcm, const int32_t* n_samples, int32_t n_chunks, const int32_t* prompt,
	int32_t n_prompt, int32_t n_decode, int32_t* tokens_out, wsp_replica_stats* stats );
/* test hook: replica i fails its next batch (exercises retire + re-queue) */
wsp_status wsp_replicas_debug_fail_next( wsp_replicas* r, int32_t replica );
void wsp_replicas_destroy( wsp_replicas* r );

/* CUDA-event stopwatch on the context's stream (the stream every kernel of this library is launched on) */
wsp_status wsp_timer_start( wsp_context* c );
wsp_status wsp_timer_stop( wsp_context* c, float* ms );
/* instrumented decoder pass for roofline accounting: n_steps more single-token steps, launched kernel by kernel with an event pair
 * around every launch.  kinds: 0 skinny GEMM, 1 cross-attention, 2 self-attention, 3 other (embedding, sampler) */
wsp_status wsp_profile_decode( wsp_context* c, int32_t batch, int32_t n_steps, float ms_by_kind[ 4 ], int32_t launches_by_kind[ 4 ] );

/* test hook: named intermediates of chunk `slot`, as f32.  n = the audio positions of the last encode (1500 unless wsp_set_audio_ctx
 * chose fewer), d = n_audio_state, H = n_audio_head, L = n_text_layer, Tp = 1536 (n_audio_ctx rounded up to 128).  The encoder
 * tensors are those of the last encode; with wsp_debug_set_encoder_layers(k) the per-layer ones belong to layer k - 1.
 *   "mel"                  [80][n_len]  log-mel of the slot
 *   "enc.input"            [2n][80]     f16 mel window, frames [offset, offset + 2n), zero past n_len
 *   "enc.conv1"            [2n][d]      f16 gelu(conv1 + bias)
 *   "enc.x"                [n][d]       f32 residual stream: the input of layer k (all layers: the input of ln_post)
 *   "enc.xn", "encode-out" [n][d]       f16 ln_post output
 *   "enc.q", "enc.k"       [H][n][64]   f16 attention Q, K of the last encoded layer
 *   "enc.vt"               [H][64][Tp]  f16 transposed V; columns [n, n rounded up to 128) are zero
 *   "enc.attn"             [n][d]       f16 attention output (head h in columns [64h, 64h + 64))
 *   "enc.h"                [n][4d]      f16 MLP hidden gelu(LN2(x) W1^T + b1) of the last encoded layer
 *   "cross_k", "cross_v"   [L][H][n][64] f16 cross-attention memories (K scaled by 64^-0.25)
 *   "self_k", "self_v"     [L][H][n_text_ctx][64] f16 decoder self-KV cache (K scaled by 64^-0.25); row j = text position j
 * The decoder tensors are the rows of chunk `slot` in the last decoder pass that ran kernel by kernel (every pass while a decoder stop
 * is set; N = that pass's tokens per chunk, d = n_text_state):
 *   "dec.x"                [N][d]       f32 residual stream
 *   "dec.q"                [N][d]       f32 query of the last self or cross attention (scaled by 64^-0.25)
 *   "dec.attn"             [N][d]       f16 output of the last self or cross attention (head h in columns [64h, 64h + 64))
 *   "dec.h"                [N][4d]      f16 MLP hidden gelu(LN3(x) W1^T + b1)
 *   "energy"               [n_samples]  f32 signal energy of the chunk's PCM (wsp_set_token_timestamps); empty before any
 *   "pcm"                  [n_samples]  f32 the slot's resident mono PCM (wsp_upload_pcm, or the downmix of wsp_upload_pcm_stereo)
 *   "pcm_stereo"           [n_frames][2] f32 the slot's stereo pairs (wsp_upload_pcm_stereo); empty after wsp_upload_pcm */
wsp_status wsp_get_tensor( wsp_context* c, const char* name, int32_t slot, float* dst, size_t cap_floats, size_t* n_floats );
/* debug: run only the first n encoder layers (negative = all) */
wsp_status wsp_debug_set_encoder_layers( wsp_context* c, int32_t n );
/* debug: end every decoder pass after op `op` of decoder layer `layer` (0 LN + QKV with the self-KV append, 1 self attention, 2 self
 * out-projection + residual, 3 LN + cross Q, 4 cross attention, 5 cross out-projection + residual, 6 LN + fc1 + GELU, 7 fc2 + residual);
 * layer -1 ends it after the embedding.  While a stop is set every wsp_decode runs kernel by kernel whatever its n_tokens and the step
 * mode, without the CUDA graph, the final LayerNorm, the logits or the probabilities, and a call that would sample fails with
 * WSP_E_INVALIDARG.  (-1, -1) clears the stop. */
wsp_status wsp_debug_set_decoder_stop( wsp_context* c, int32_t layer, int32_t op );
/* The CPU reference accumulates the decoder's V^T*P product in f16, per thread (Whisper/source/ggml.c:4680-4722), so its logits
 * depend on its thread count.  n = the cpuThreads the reference would be run with (sFullParams::cpuThreads; default 4 =
 * whisper_full_default_params, Whisper/source/whisper.cpp:2605); the decoder reproduces that arithmetic for n = 1..16 in every
 * step mode.  Any other n returns WSP_E_INVALIDARG. */
wsp_status wsp_set_reference_threads( wsp_context* c, int32_t n );
/* debug: 0 = launch the N = 1 decoder step kernel by kernel instead of replaying the captured CUDA graph */
wsp_status wsp_debug_set_graph( wsp_context* c, int32_t on );
/* debug: how the single-token decoder step runs: 2 = one dataflow kernel (decode_flow.cu, default), 1 = round 1's persistent kernel with
 * grid barriers (decode_mega.cu, kept for same-box A/B runs), 0 = one kernel per op */
wsp_status wsp_debug_set_step_mode( wsp_context* c, int32_t mode );
/* debug: record %globaltimer marks (ns) of CTA 0 at every phase boundary of the decoder-step kernel; read them back after a step */
wsp_status wsp_debug_enable_step_timing( wsp_context* c, int32_t on );
wsp_status wsp_debug_step_timing( wsp_context* c, uint64_t* dst, int32_t cap );
/* pinned host memory for callers that want asynchronous H2D copies of PCM (bench.py's e2e leg) */
void* wsp_host_alloc( size_t bytes );
void wsp_host_free( void* p );
/* per-phase device time accumulated by the context (CUDA events): { mel, encode, decode, sample } in ms, and call counts */
wsp_status wsp_timings( wsp_context* c, float ms4[ 4 ], int32_t calls4[ 4 ], int32_t reset );

/* ---- kernel-level test hooks (tests/ only) ---- */
/* D[M][N] = A[M][K] * B[N][K]^T with the wgmma GEMM; A,B f16 bit patterns (uint16), D f32; all host pointers */
wsp_status wsp_test_gemm( int32_t device, int32_t M, int32_t N, int32_t K, const uint16_t* A, const uint16_t* B, float* D, int32_t bn, int32_t iters, float* ms );
/* encoder attention: Q,K [BH][T][64], V [BH][T][64] f16 bit patterns -> out f32 [BH][T][64] */
wsp_status wsp_test_attention( int32_t device, int32_t BH, int32_t T, const uint16_t* Q, const uint16_t* K, const uint16_t* V, float* out, int32_t iters, float* ms );
/* skinny GEMM: out[cols][nOut] = x[cols][K] * W[nOut][K]^T */
wsp_status wsp_test_skinny( int32_t device, int32_t nOut, int32_t K, int32_t cols, const uint16_t* W, const uint16_t* X, float* out, int32_t iters, float* ms );
/* sampler alone: rows of logits -> probs (softmax with the reference's f16-table exp, may be NULL) and one sampled token per row under
 * the rules of whisper_sample_best / whisper_sample_timestamp (whisper.cpp:1875-1964); special4 = { beg, sot, solm, not } */
wsp_status wsp_test_sample( int32_t device, int32_t rows, int32_t n_vocab, const float* logits, const int32_t special4[ 4 ], int32_t force_timestamp,
	int32_t is_initial, float* probs, wsp_token_data* out );
/* host only: whisper_full's window rule (csrc/window_rule.h, the code runFull and the sampler epilogue run) over ids[n] from step 0 of
 * a window at `seek` over seek_end frames; rule4 = { eot, beg, max_tokens, single_segment }, n_max = n_text_ctx / 2 - 4.  out5 =
 * { has_ts, seek_delta, result_len, failed, ended }; *n_steps = the tokens it consumed (the one that ended the window included). */
wsp_status wsp_test_window_rule( const int32_t rule4[ 4 ], int32_t n_max, int32_t seek, int32_t seek_end, const int32_t* ids, int32_t n, int32_t out5[ 5 ], int32_t* n_steps );
/* host only: whisper_full's token times (csrc/token_times.h, the code runFull and wsp_window_token_times run) for one segment of
 * tokens[n] over [t0, t1] with vlen[n], energy[n_samples] and the state state3 = { t_beg, t_last, tid_last } carried in and out;
 * special2 = { beg, eot }; times[n] holds the times on entry (-1 where none) and on return.  WSP_S_FALSE, changing nothing, without
 * energy (n_samples 0). */
wsp_status wsp_test_token_times( const wsp_token_data* tokens, const float* vlen, int32_t n, int64_t t0, int64_t t1, const int32_t special2[ 2 ],
	const float* energy, int32_t n_samples, float thold_pt, float thold_ptsum, int64_t state3[ 3 ], wsp_token_time* times );
/* host only: detectSpeaker's rule (csrc/speaker.h, the code iContext::detectSpeaker and the kernel of wsp_chunk_speakers run) for
 * segs[n_segs] over interleaved lr[n_frames][2] -> speakers[n_segs], as wsp_chunk_speakers answers them; lr may be NULL when n_frames
 * is 0 (no stereo) */
wsp_status wsp_test_speakers( const float* lr, int32_t n_frames, const wsp_segment* segs, int32_t n_segs, int32_t* speakers );
/* signal_energy_kernel alone over `batch` host clips pcm[b][n_samples[b]] -> energy[b][n_samples[b]] (host); with iters > 0, *ms = the
 * mean time of one launch over `iters` more launches between CUDA events */
wsp_status wsp_test_signal_energy( int32_t device, const float* const* pcm, const int32_t* n_samples, int32_t batch, float* const* energy,
	int32_t iters, float* ms );
/* the all-logits vocabulary softmax alone: rows of n logits -> probs with the reference's f16-table exp (host pointers) */
wsp_status wsp_test_softmax_rows( int32_t device, int32_t rows, int32_t n, const float* logits, float* probs );
/* LayerNorm rows x d f32 -> f16 bit patterns */
wsp_status wsp_test_layernorm( int32_t device, int32_t rows, int32_t d, const float* x, const float* gamma, const float* beta, uint16_t* out );

#ifdef __cplusplus
}
#endif
#endif

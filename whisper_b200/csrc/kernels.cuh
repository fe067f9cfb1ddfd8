// Non-GEMM kernels of the hot path (HBM-bound): log-mel front end, LayerNorm, encoder window gather, token embedding,
// and the decoder's per-token kernels (skinny weight-streaming GEMM, self/cross attention over the f16 KV memories, sampler).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include "window_rule.h"

namespace kern
{
	// Launch with the programmatic-stream-serialization attribute (PDL).  Kernels launched this way call pdl_launch_dependents() first
	// thing and pdl_wait() before touching anything a predecessor wrote.
	template<class... KArgs, class... Args>
	inline cudaError_t launchPdl( void ( *kernel )( KArgs... ), dim3 grid, dim3 block, size_t smem, cudaStream_t s, Args... args )
	{
		cudaLaunchConfig_t cfg{};
		cfg.gridDim = grid;
		cfg.blockDim = block;
		cfg.dynamicSmemBytes = smem;
		cfg.stream = s;
		cudaLaunchAttribute at[ 1 ];
		at[ 0 ].id = cudaLaunchAttributeProgrammaticStreamSerialization;
		at[ 0 ].val.programmaticStreamSerializationAllowed = 1;
		cfg.attrs = at;
		cfg.numAttrs = 1;
		return cudaLaunchKernelEx( &cfg, kernel, static_cast<KArgs>( args )... );
	}

	// ---- log-mel (a1: whisper.cpp:2060-2181) -------------------------------------------------------------------
	struct MelTables
	{
		const float* hann = nullptr;     // [400]  f32( 0.5*(1-cos(2*pi*i/400)) )
		const double* cosT = nullptr;    // [400]  cos(2*pi*m/400)
		const double* sinT = nullptr;    // [400]
		const float* filters = nullptr;  // [80][201] from the model file
		const double2* twiddle = nullptr; // [400]  { cosT, sinT } interleaved: one 16-byte shared-memory read per DFT term
		const short2* band = nullptr;     // [80]   [x, y) = the bins where the band's filter row is non-zero (real filter banks are triangular)
	};
	// The phase vocoder (speed-up, whisper.cpp:2299-2311) takes a second MelTables of the same layout: hann [800] and twiddle [800] of the
	// 800-point transform, cosT / sinT unset, filters and band shared with the 400-point tables.
	// up to MEL_BATCH chunks transformed and normalised by one launch each (power, normalise); single clips and streamed windows are
	// a batch of one.  Chunk b: pcm [nSamples] -> log10 mel [80][nLen] (row = band), its maximum (ordered-int encoded float) in maxSlots[b]
	constexpr int MEL_BATCH = 16;
	struct MelBatch
	{
		const float* pcm[ MEL_BATCH ];
		float* mel[ MEL_BATCH ];       // [80][nLen[b]]
		int nSamples[ MEL_BATCH ];
		int nLen[ MEL_BATCH ];
		int* maxSlots;                 // [count] consecutive
		int count;
	};
	// raw log10 mel and maxSlots; speedUp: the phase vocoder (800-point transform, hop 320, tb = its tables) instead of the 400-point
	// one (hop 160)
	cudaError_t melBatchPower( const MelTables& tb, const MelBatch& mb, bool speedUp, cudaStream_t s );
	// in place: clamp to (maxSlots[b] - 8), (x + 4) / 4
	cudaError_t melBatchNormalize( const MelBatch& mb, cudaStream_t s );
	// mel f32 [80][nLen] at frame offset -> time-major f16 window [1 + frames + 1][80], halo rows (conv padding) written as zeros;
	// frames = 2 * audio_ctx (3000 by default)
	cudaError_t melWindow( const float* mel, int nLen, int offset, __half* dst, int frames, cudaStream_t s );

	// ---- signal energy of token-level timestamps (get_signal_energy, whisper.cpp:3356-3372) ----------------------------------
	// every chunk of a batch in one launch: chunk b's pcm[b][nSamples[b]] -> out[row[b] * stride + i] = (sum over j = -32..32 with
	// 0 <= i + j < n of |x[i + j]|) / 65, the sum in f32 in that order of j, so the result is bit-identical to the reference's
	constexpr int ENERGY_BATCH = 256;
	constexpr int ENERGY_HW = 32;
	struct EnergyBatch
	{
		const float* pcm[ ENERGY_BATCH ];
		int nSamples[ ENERGY_BATCH ];
		uint8_t row[ ENERGY_BATCH ];   // the output row of chunk b (a context slot, < 256)
		float* out;                    // [rows][stride]
		int64_t stride;
		int count;
	};
	cudaError_t signalEnergy( const EnergyBatch& eb, cudaStream_t s );

	// ---- stereo chunks and their speakers (wsp_upload_pcm_stereo, wsp_chunk_speakers) -------------------------------------------
	// mono[i] = (lr[2i] + lr[2i+1]) * 0.5f for i < nFrames (AudioBuffer::appendDownmixedStereo); one launch, also for nFrames = 0
	cudaError_t downmixStereo( const float* lr, float* mono, int nFrames, cudaStream_t s );
	// one segment of detectSpeaker (speaker.h): pre != wsp::kSpeakerSums is the answer already; otherwise the lane sums of the count
	// frames at lr (16-byte aligned) decide it
	struct SpeakerJob
	{
		const float* lr;
		int64_t count;
		int32_t pre;
		int32_t pad;
	};
	// out[i] = the answer of jobs[i] for i < n, one warp per segment; n >= 1
	cudaError_t chunkSpeakers( const SpeakerJob* jobs, int32_t* out, int n, cudaStream_t s );

	// ---- LayerNorm + affine -> f16 (a5, a11) -------------------------------------------------------------------------
	cudaError_t layerNormF16( const float* x, const float* gamma, const float* beta, __half* out, int rows, int d, cudaStream_t s );

	// ---- decoder -------------------------------------------------------------------------------------------------------
	// x[b*N+i][:] = f32(te[token[b*N+i]][:]) + pe[nPast+i][:]     (a13)
	cudaError_t embedTokens( const __half* te, const float* pe, const int* tokens, const int* dNPast, float* x, int B, int N, int d, cudaStream_t s );

	enum SkinnyEpi : int
	{
		SK_QKV = 0,        // rows [0,d): q f32 = (acc+b)*s ; [d,2d): K cache f16 = acc*s ; [2d,3d): V cache f16 = acc+b
		SK_BIAS_RESID = 1, // x f32 += acc + b
		SK_Q_SCALE = 2,    // q f32 = (acc+b)*s
		SK_GELU_F16 = 3,   // h f16 = gelu(acc+b)
		SK_LOGITS = 4,     // logits f32 = acc
	};
	struct SkinnyArgs
	{
		const __half* W = nullptr;     // [nOut][K] f16 row-major
		int nOut = 0, K = 0;
		// input columns: either f32 rows + LayerNorm (gamma != null) or f16 rows
		const float* xF32 = nullptr;
		const __half* xF16 = nullptr;
		int64_t xStride = 0;           // elements between consecutive columns
		const float* gamma = nullptr;
		const float* beta = nullptr;
		int nCols = 0;
		// epilogue
		int epi = 0;
		const float* bias = nullptr;
		float scale = 1.0f;
		float* outF32 = nullptr;       // q / x / logits  [col][ld]
		__half* outF16 = nullptr;      // h             [col][ld]
		int ld = 0;
		__half* kCache = nullptr;      // [B][H][nTextCtx][64] for this layer (head-major)
		__half* vCache = nullptr;
		int d = 0, N = 0, nTextCtx = 0;
		const int* dNPast = nullptr;
	};
	cudaError_t skinnyGemm( const SkinnyArgs& a, cudaStream_t s );

	// refThreads (1..kMaxRefThreads): reproduce the reference's f16-accumulated V^T*P for that many CPU threads (ref_arith.cuh)
	// self attention over the f16 self-KV cache, causal: query i of chunk b sees keys [0, nPast+i]   (a14)
	cudaError_t selfAttnDecode( const float* q, const __half* kCache, const __half* vCache, __half* out, int B, int N, int H, int d, int nTextCtx, const int* dNPast, int refThreads, cudaStream_t s );
	// cross attention over the f16 cross-KV memory [b][h][T][64]                                       (a15)
	cudaError_t crossAttnDecode( const float* q, const __half* kMem, const __half* vMem, __half* out, int B, int N, int H, int d, int T, int refThreads, cudaStream_t s );

	// softmax + greedy sampling with the Whisper timestamp rules (a17 softmax, a18: whisper.cpp:1875-1964)
	struct TokenData
	{
		int id, tid;
		float p, pt, ptsum;
	};
	struct SampleArgs
	{
		const float* logits = nullptr;  // [B][nVocab] (last token of each chunk)
		float* probs = nullptr;         // [B][nVocab] out
		int B = 0, nVocab = 0;
		int tokenBeg = 0, tokenSot = 0, tokenSolm = 0, tokenNot = 0;
		const int* dForceTs = nullptr;  // device flags: [0] force_timestamp, [1] is_initial (so one CUDA graph serves every step)
		TokenData* out = nullptr;       // [B]
		int* nextTokens = nullptr;      // [B] device feedback for the next step (may be null)
		int* dNPast = nullptr;          // advanced by N after sampling (may be null)
		int N = 0;
		int* history = nullptr;         // optional [B][histCap] token log, written at column *dStep
		int histCap = 0;
		int* dStep = nullptr;
		int* tieScratch = nullptr;      // required: [B][nVocab + 1024] ints, survivor lists of the exact tie emulation
		// end-of-text log (null = unarmed): the first time row b samples tokenEot, endStep[b] (zeroed by the caller) = *dStep + 1
		// and *nEnded is incremented; the advance kernel then copies *nEnded to *nEndedHost (mapped pinned host memory)
		int tokenEot = 0;
		int* endStep = nullptr;
		int* nEnded = nullptr;
		volatile int* nEndedHost = nullptr;
		// armed callers also pass these (wsp_run_chunks_window): the step's TokenData goes to tokenLog[b][*dStep], and while
		// winCtl[0] is set a row ends by whisper_full's window rule (window_rule.h) instead of at its first EOT.  winCtl = { on,
		// max_tokens, single_segment, n_max }, then seek_end - seek of each row [B] (the rule runs at seek 0 over it, which decides
		// as at seek over seek_end); winState[B] is the rows' state, and a row whose endStep the caller set non-zero never runs the rule
		const int* winCtl = nullptr;
		wsp::WindowState* winState = nullptr;
		TokenData* tokenLog = nullptr;
	};
	// one cluster of 4 CTAs per row (any nVocab >= 8 whose quarter fits shared memory), then the 1-thread advance of n_past / flags / step
	cudaError_t sampleGreedy( const SampleArgs& a, cudaStream_t s );

	// row-wise softmax of [rows][n] (all-logits test mode)
	cudaError_t softmaxRows( const float* logits, float* probs, int rows, int n, cudaStream_t s );

	// whisper_lang_auto_detect's choice for every row of a batch (whisper.cpp:2428-2495), after the [sot] pass and softmaxRows: the
	// language tokens' probabilities probs[b][tokLang0 + l], l < nLangs, ordered descending (equal values: lower l first), exp() of
	// each summed in that order in f32, langProbs[b][l] = exp(p_l) / sum, langIds[b] = the top l.  Row b's prompt is then written to
	// tokens[b * nPrompt + i]: tmpl[i], with tmpl[autoPos] replaced by tokLang0 + langIds[b].
	constexpr int kLangPromptMax = 256;
	struct LangPickArgs
	{
		const float* probs = nullptr;   // [B][nVocab]
		int nVocab = 0, tokLang0 = 0, nLangs = 0;
		int* langIds = nullptr;         // [B]
		float* langProbs = nullptr;     // [B][nLangs]
		int* tokens = nullptr;          // [B][nPrompt]
		int nPrompt = 0, autoPos = 0;
		int tmpl[ kLangPromptMax ];
	};
	cudaError_t langPick( const LangPickArgs& a, int B, cudaStream_t s );
	// one-time function attributes (dynamic shared memory opt-in) so that nothing but launches happens under stream capture
	cudaError_t prepare( int maxK );

	// tiny helpers
	cudaError_t setInts( int* dst, int a, int b, cudaStream_t s );
}

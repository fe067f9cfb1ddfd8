// Engine (weights on one H100) and Context (per-stream state for up to maxBatch independent 30 s chunks).
//
// Reference counterparts: ModelBuffers (Whisper/Whisper/ModelBuffers.h:8-111) / WhisperModel (loader), and WhisperContext
// (Whisper/Whisper/WhisperContext.cpp:138-639 — the network definition) with its KeyValueBuffers (KeyValueBuffers.h:7-53).
// Oracle: whisper_encode / whisper_decode (Whisper/source/whisper.cpp:1084-1872).
#pragma once
#include "../../include/whisper_b200.h"
#include "attn_enc.cuh"
#include "decode_flow.cuh"
#include "decode_mega.cuh"
#include "gemm_tc.cuh"
#include "kernels.cuh"
#include "model.h"
#include <atomic>
#include <string>
#include <vector>

namespace wsp
{
	extern thread_local std::string g_lastError;
	extern std::atomic<uint64_t> g_launchCount;
	int fail( int status, const std::string& what );
	int cudaFail( cudaError_t e, const char* what );

#define WSP_CUDA( expr )                                                        \
	do {                                                                        \
		cudaError_t _e = ( expr );                                              \
		if( _e != cudaSuccess ) return ::wsp::cudaFail( _e, #expr );            \
	} while( 0 )
#define WSP_CHECK( expr )                                                       \
	do {                                                                        \
		int _s = ( expr );                                                      \
		if( _s < 0 ) return _s;                                                 \
	} while( 0 )

	constexpr int kFrames = 3000;          // mel frames per 30 s window
	constexpr int kFramesPad = 3002;       // + one zero halo row each side (conv padding = 1)
	constexpr int kConv1KTap = 128;        // 80 input channels padded to two 64-wide K blocks per tap
	constexpr int kMaxDecodeTokens = 256;  // tokens per chunk in one decoder call (prompt <= 224 + 4)
	constexpr int kAllLogitsTokens = 8;
	constexpr int kStepMarks = 4608;       // 64-bit debug marks the decoder-step kernels may write (wsp_debug_step_timing)

	struct LnW { float* g = nullptr; float* b = nullptr; };
	struct EncLayerW
	{
		LnW ln1, ln2;
		__half* wqkv = nullptr; float* bqkv = nullptr;   // [3d][d], (q.b | 0 | v.b)
		__half* wo = nullptr; float* bo = nullptr;
		__half* w1 = nullptr; float* b1 = nullptr;       // [4d][d]
		__half* w2 = nullptr; float* b2 = nullptr;       // [d][4d]
	};
	struct DecLayerW
	{
		LnW ln1, lnc, ln3;
		__half* wqkv = nullptr; float* bqkv = nullptr;
		__half* wo = nullptr; float* bo = nullptr;
		__half* wcq = nullptr; float* bcq = nullptr;
		__half* wco = nullptr; float* bco = nullptr;
		__half* w1 = nullptr; float* b1 = nullptr;
		__half* w2 = nullptr; float* b2 = nullptr;
	};

	struct Engine
	{
		int device = 0;
		int numSMs = 132;
		HParams hp{};
		int tokEot = 0, tokSot = 0, tokPrev = 0, tokSolm = 0, tokNot = 0, tokBeg = 0;
		int nLangs = 0;                 // language tokens sot + 1 .. sot + nLangs (99 on the multilingual vocabulary, 0 otherwise)
		uint8_t* arena = nullptr;
		size_t arenaSize = 0, arenaUsed = 0;

		__half* conv1w = nullptr; float* conv1b = nullptr;   // [d][3*128]
		__half* conv2w = nullptr; float* conv2b = nullptr;   // [d][3*d]
		float* encPos = nullptr;                             // [1500][d]
		LnW encLnPost;
		std::vector<EncLayerW> enc;
		__half* crossW = nullptr; float* crossB = nullptr;   // [L*2d][d] (K_l | V_l), bias (0 | v.b)
		float* decPos = nullptr;                             // [n_text_ctx][d]
		__half* tokEmb = nullptr;                            // [n_vocab][d]
		LnW decLn;
		std::vector<DecLayerW> dec;
		kern::MelTables mel;
		kern::MelTables melVocoder;   // the phase vocoder's 800-point window and twiddles, mel's filters (speed-up)
		std::vector<std::string> tokenText;   // the vocabulary, for the host-side segment rules of wsp_window_token_times

		~Engine();
	};

	int createEngine( const ModelFile& m, int device, const void* devImage, uint64_t imageSize, Engine** out );

	struct MelSlot
	{
		float* mel = nullptr;   // [80][nLen]
		int cap = 0;            // frames allocated
		int nLen = 0;
		float* pcm = nullptr;   // optional device-resident PCM (wsp_upload_pcm), for the HBM-resident bench leg
		int pcmCap = 0;
		int pcmSamples = 0;
		float* stereo = nullptr;   // [stereoCap][2] interleaved pairs of wsp_upload_pcm_stereo, whose downmix is `pcm`
		int stereoCap = 0;
		int stereoFrames = 0;      // 0: the slot has no stereo (wsp_upload_pcm drops it)
	};

	// one row of a window call: the slot whose log-mel it encodes and whisper_full's seek_start / seek_end, in mel frames
	struct WindowRow
	{
		int slot, seek, seekEnd;
	};

	// per-kernel-kind device time of the decoder, collected by an instrumented (un-graphed) pass: wsp_profile_decode
	enum KernelKind { KK_SKINNY = 0, KK_CROSS = 1, KK_SELF = 2, KK_OTHER = 3, KK_COUNT = 4 };
	struct KernelProfile
	{
		bool on = false;
		std::vector<cudaEvent_t> pool;
		std::vector<int> kinds;     // kind of interval i = [pool[2i], pool[2i+1]]
		size_t used = 0;
	};

	// What a captured N = 1 step graph depends on.  The launches in it took their arguments by value at capture time, so every
	// Context field that decodeEnqueue reads by value for the N = 1 path is a member: decodeSubmit re-captures when the key differs.
	struct StepGraphKey
	{
		int batch = 0, encCtx = 0, refThreads = 0, stepMode = 0;
		bool timing = false;
		bool eot = false;
		bool operator==( const StepGraphKey& o ) const
		{
			return batch == o.batch && encCtx == o.encCtx && refThreads == o.refThreads && stepMode == o.stepMode && timing == o.timing && eot == o.eot;
		}
	};

	struct Context
	{
		Engine* e = nullptr;
		int maxB = 0;
		cudaStream_t stream = nullptr;
		std::vector<MelSlot> slots;
		int* melMax = nullptr;          // [maxB] ordered-int maxima of one mel launch's chunks
		float* pcmDev = nullptr; size_t pcmCap = 0;
		uint64_t devBytes = 0;          // device memory this context holds (timingsPrint's memory table)
		bool speedUp = false;           // whole-clip log-mels through the 2x phase vocoder (wsp_set_speed_up)

		// encoder workspaces
		// sized for n_audio_ctx = 1500; an encode over n <= 1500 audio positions (audio_ctx) packs its chunks densely with n in
		// place of 1500 (2n + 2 rows per chunk in melF16 / conv1), inside the same allocations and tensor maps
		__half* melF16 = nullptr;       // [maxB][3002][80]
		__half* conv1 = nullptr;        // [maxB][3002][d]
		float* x = nullptr;             // [maxB*1500][d] residual stream
		__half* xn = nullptr;           // [maxB*1500][d]
		__half* q = nullptr;            // [maxB][H][1500][64]
		__half* k = nullptr;
		__half* vt = nullptr;           // [maxB][H][64][Tp] (row length Tp whatever n is)
		__half* attn = nullptr;         // [maxB*1500][d]
		__half* h = nullptr;            // [maxB*1500][4d]
		__half* crossK = nullptr;       // [L][maxB][H][1500][64]; with n audio positions each layer holds [maxB][H][n][64] at the same stride
		__half* crossV = nullptr;
		int Tp = 0;
		int audioCtx = 0;               // audio positions the next encode uses (wsp_set_audio_ctx; 0 = the model's n_audio_ctx)
		int encCtx = 0;                 // audio positions of the last encode: rows of the cross-KV memories every decode attends over

		// decoder state
		__half* selfK = nullptr;        // [L][maxB][H][n_text_ctx][64] (head-major rows)
		__half* selfV = nullptr;
		float* xd = nullptr;            // [maxB*kMaxDecodeTokens][d]
		float* qd = nullptr;
		__half* attnD = nullptr;
		__half* hD = nullptr;           // [maxB*kMaxDecodeTokens][4d]
		float* logits = nullptr;        // [maxB*kAllLogitsTokens][n_vocab]
		float* probs = nullptr;
		int* tieScratch = nullptr;      // [maxB][n_vocab + 1024]: survivor lists of the sampler's exact tie emulation
		int* tokensDev = nullptr;       // [maxB*kMaxDecodeTokens]
		int* dNPast = nullptr;          // device scalars: n_past | flags[2] | step
		int* dFlags = nullptr;
		int* dStep = nullptr;
		kern::TokenData* sampled = nullptr;   // [maxB]
		int* history = nullptr;         // [maxB][histCap]
		int histCap = 0;
		// end-of-text log of wsp_run_chunks_until_eot: the sampler fills it only while eotArmed is set
		bool eotArmed = false;
		int* endStep = nullptr;         // [maxB] 1 + the step of each chunk's first EOT, 0 = none yet
		int* nEnded = nullptr;          // device counter of chunks with an EOT (in the dNPast block)
		int* nEndedHost = nullptr;      // mapped pinned copy of nEnded, written by the last kernel of every step
		int* nEndedMapped = nullptr;    // its device address
		cudaEvent_t blockEv[ 2 ] = { nullptr, nullptr };   // ends of the last two enqueued step blocks
		// whisper_full's window rule of the window calls, passed to the armed sampler of both calls; winCtl[0] = 0 (EOT) or 1 (rule)
		int* winCtl = nullptr;          // [4 + maxB] on | max_tokens | single_segment | n_max, then each row's seek_end - seek
		wsp::WindowState* winState = nullptr;   // [maxB]
		kern::TokenData* tokenLog = nullptr;    // [maxB][histCap] every armed step's TokenData
		// per-chunk language detection of a run_chunks* call whose prompt holds WSP_TOKEN_LANGUAGE_AUTO (lang_pick_kernel)
		int* langIds = nullptr;         // [maxB]
		float* langProbs = nullptr;     // [maxB][nLangs]
		std::vector<int32_t> lastLangIds;   // host copies from the last run_chunks* call (wsp_get_chunk_languages); empty: it had no sentinel
		std::vector<float> lastLangProbs;   // [batch][nLangs]
		// signal energy of token-level timestamps (wsp_set_token_timestamps): computed only while tokenTimestamps is set
		bool tokenTimestamps = false;
		float* energy = nullptr;        // [maxB][energyCap] on the device
		float* energyHost = nullptr;    // [maxB][energyCap] pinned: the last window call's energy, copied back with its tokens
		size_t energyCap = 0;
		std::vector<int> energyLen;     // [maxB] samples of each slot's device energy
		int windowEnergyBatch = 0;      // batch of the last window call if it computed the energy, else 0
		std::vector<int> windowEnergyLen;   // [that batch] samples of each chunk's source energy in energyHost
		std::vector<WindowRow> windowRows;  // [that batch] each chunk's source slot (its energy's row in energyHost) and seek
		// wsp_chunk_speakers: the segments' jobs, then their answers, in one device buffer
		uint8_t* speakerBuf = nullptr;
		size_t speakerCap = 0;          // segments it holds
		int lastLogitRows = 0;
		int nPastHost = 0;              // host mirror of the device-resident n_past (it advances on the device between graph replays)
		int debugEncLayers = -1;
		// wsp_debug_set_decoder_stop: every decoder pass runs kernel by kernel and ends after op debugDecOp of layer debugDecLayer
		// (layer -1: after the embedding), without logits or sampling; (-1, -1) = no stop
		int debugDecLayer = -1, debugDecOp = -1;
		bool decoderStopped() const { return debugDecLayer >= 0 || debugDecOp >= 0; }
		int lastPerOpN = 0;             // tokens per chunk of the last kernel-by-kernel decoder pass: the rows of c.xd, qd, attnD, hD
		int refThreads = 4;            // reference CPU thread count whose V^T*P arithmetic the decoder reproduces (1..16)

		// tensor maps (built once; M of a launch limits the rows touched)
		CUtensorMap mapMel, mapConv1Even, mapConv1Odd, mapXn, mapAttn, mapH;
		CUtensorMap mapConv1W, mapConv2W, mapCrossW;
		std::vector<CUtensorMap> mapWqkv, mapWo, mapW1, mapW2;
		CUtensorMap mapQ, mapK, mapVt;
		int bnD = 128, bn3D = 128, bn4D = 128, bnCross = 128;

		// per-layer pointer table of both decoder-step kernels, on the device
		kern::DecStepLayer* stepLayers = nullptr;
		// persistent decoder-step kernel (decode_mega.cu): grid-barrier counter
		unsigned* megaBarrier = nullptr;
		// dataflow decoder-step kernel (decode_flow.cu): per-CTA bias slabs, exchange buffers, launch epoch
		float* flowBias = nullptr;
		uint8_t* flowExch = nullptr;
		unsigned* flowCtrl = nullptr;
		kern::FlowGeom flowGeom;
		// N = 1 decoder step (wsp_debug_set_step_mode): 2 = dataflow kernel (default), 1 = round 1's barrier kernel, 0 = one kernel per op
		int stepMode = 2;
		unsigned long long* stepMarks = nullptr;   // [kStepMarks] debug marks of the step kernels, read by wsp_debug_step_timing
		bool stepTiming = false;        // the step kernels record %globaltimer marks into stepMarks (wsp_debug_enable_step_timing)
		int stepTimingCta = 0;          // CTA whose marks the dataflow kernel records (WSP_TIMING_CTA; the barrier kernel's is CTA 0)

		// decode CUDA graph (N = 1 steady state)
		cudaGraphExec_t stepGraph = nullptr;
		StepGraphKey stepGraphKey;      // what stepGraph was captured for
		int stepGraphLaunches = 0;
		bool useGraph = true;

		KernelProfile prof;
		cudaEvent_t timerEv[ 2 ] = { nullptr, nullptr };

		// timing
		cudaEvent_t ev[ 4 ] = { nullptr, nullptr, nullptr, nullptr };
		float ms[ 4 ] = { 0, 0, 0, 0 };
		int calls[ 4 ] = { 0, 0, 0, 0 };

		~Context();
	};

	int createContext( Engine* e, int maxBatch, Context** out );
	int ctxPcmToMel( Context& c, int slot, const float* pcmHost, int nSamples );
	int ctxPcmToMelWindow( Context& c, int slot, const float* pcmHost, int nSamples, int nFrames, const float* forcedMax, float* maxOut );
	int ctxSetMel( Context& c, int slot, const float* melHost, int nLen );
	int ctxEncode( Context& c, const int32_t* offsets, int batch );
	int ctxSetAudioCtx( Context& c, int n );
	int ctxSetSpeedUp( Context& c, int on );
	int ctxSetTokenTimestamps( Context& c, int on );
	int ctxDecode( Context& c, const int32_t* tokensHost, int nTokens, int nPast, int batch, uint32_t flags, wsp_token_data* sampledHost );
	int ctxUploadPcm( Context& c, int slot, const float* pcmHost, int nSamples );
	int ctxUploadPcmStereo( Context& c, int slot, const float* lrHost, int nFrames );
	int ctxChunkSpeakers( Context& c, int batch, const int32_t* segStart, const wsp_segment* segs, int32_t* speakers );
	int ctxProfileDecode( Context& c, int batch, int nSteps, float* msByKind, int* launchesByKind );
	// wsp_run_chunks_window's outputs
	struct WindowOut
	{
		wsp_window_params params;
		wsp_token_data* tokens;         // [batch][cap], may be null
		int cap;
		wsp_window_result* results;     // [batch]
	};
	// nOut == nullptr and window == nullptr: nDecode steps for every chunk (wsp_run_chunks*); nOut: each chunk ends at its first EOT
	// (wsp_run_chunks_until_eot); window: each chunk ends by whisper_full's window rule, nDecode = n_max (wsp_run_chunks_window).
	// rows (window calls from resident PCM only): chunk b is rows[b]'s window, else chunk b is slot b's at seek 0 over its mel length.
	int ctxRunChunks( Context& c, const float* const* pcm, const int32_t* nSamples, int batch, const int32_t* prompt, int nPrompt, int nDecode,
		int32_t* tokensOut, int32_t* nOut, float* stageMs, bool resident, const WindowOut* window = nullptr, const WindowRow* rows = nullptr );
	// wsp_run_spans_window
	int ctxRunSpans( Context& c, const wsp_window_span* spans, int batch, const int32_t* prompt, int nPrompt, int nDecode, float* stageMs,
		const WindowOut& window );
}

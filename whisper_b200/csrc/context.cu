// Context: workspaces, tensor maps, encoder / decoder orchestration (the network definition).
// Reference: WhisperContext::encode / ::decode (Whisper/Whisper/WhisperContext.cpp:310-388, 578-639); oracle whisper_encode /
// whisper_decode (Whisper/source/whisper.cpp:1084-1872).  All launches go to one stream; the N = 1 decoder step is a CUDA graph.
#include "engine.h"
#include "speaker.h"
#include <algorithm>
#include <math.h>
#include <memory>
#include <stdlib.h>
#include <string.h>

namespace wsp
{
	namespace
	{
		thread_local uint64_t t_allocated = 0;   // bytes handed out by devAlloc on this thread (read by its callers)
		template<class T> int devAlloc( T*& p, size_t count, bool zero = false )
		{
			void* v = nullptr;
			cudaError_t e = cudaMalloc( &v, count * sizeof( T ) );
			if( e != cudaSuccess ) return cudaFail( e, "cudaMalloc" );
			if( zero )
			{
				e = cudaMemset( v, 0, count * sizeof( T ) );
				if( e != cudaSuccess ) return cudaFail( e, "cudaMemset" );
			}
			p = static_cast<T*>( v );
			t_allocated += count * sizeof( T );
			return WSP_OK;
		}
		inline void launched( int n = 1 ) { g_launchCount.fetch_add( (uint64_t)n, std::memory_order_relaxed ); }
		inline int pickBN( int N ) { return ( N % 256 == 0 ) ? 256 : 128; }
	}

	Context::~Context()
	{
		if( e ) cudaSetDevice( e->device );
		if( stepGraph ) cudaGraphExecDestroy( stepGraph );
		for( auto& s : slots ) { if( s.mel ) cudaFree( s.mel ); if( s.pcm ) cudaFree( s.pcm ); if( s.stereo ) cudaFree( s.stereo ); }
		for( auto& v : prof.pool ) cudaEventDestroy( v );
		for( auto& v : timerEv ) if( v ) cudaEventDestroy( v );
		void* bufs[] = { stepLayers, flowBias, flowExch, flowCtrl, megaBarrier, stepMarks, melMax, pcmDev, melF16, conv1, x, xn, q, k, vt, attn, h, crossK, crossV, selfK, selfV, xd, qd, attnD, hD, logits, probs, tieScratch,
			tokensDev, dNPast, sampled, history, endStep, langIds, langProbs, winCtl, winState, tokenLog, energy, speakerBuf };
		for( void* b : bufs ) if( b ) cudaFree( b );
		if( nEndedHost ) cudaFreeHost( nEndedHost );
		if( energyHost ) cudaFreeHost( energyHost );
		for( auto& v : ev ) if( v ) cudaEventDestroy( v );
		for( auto& v : blockEv ) if( v ) cudaEventDestroy( v );
		if( stream ) cudaStreamDestroy( stream );
	}

	int createContext( Engine* e, int maxBatch, Context** out )
	{
		if( !e || maxBatch < 1 || maxBatch > 256 ) return fail( WSP_E_INVALIDARG, "max_batch must be in [1, 256]" );
		WSP_CUDA( cudaSetDevice( e->device ) );
		std::unique_ptr<Context> cp( new Context() );
		Context& c = *cp;
		c.e = e;
		c.maxB = maxBatch;
		t_allocated = 0;
		struct Tally { Context& c; ~Tally() { c.devBytes += t_allocated; t_allocated = 0; } } tally{ c };
		const HParams& hp = e->hp;
		const int d = hp.n_audio_state, H = hp.n_audio_head, T = hp.n_audio_ctx, L = hp.n_text_layer;
		if( T * 2 != kFrames ) return fail( WSP_E_FORMAT, "n_audio_ctx must be 1500" );
		c.Tp = ( ( T + 127 ) / 128 ) * 128;
		c.encCtx = T;
		WSP_CUDA( cudaStreamCreateWithFlags( &c.stream, cudaStreamNonBlocking ) );
		for( auto& v : c.ev ) WSP_CUDA( cudaEventCreate( &v ) );
		for( auto& v : c.timerEv ) WSP_CUDA( cudaEventCreate( &v ) );
		for( auto& v : c.blockEv ) WSP_CUDA( cudaEventCreateWithFlags( &v, cudaEventDisableTiming ) );
		c.slots.resize( maxBatch );
		c.energyLen.assign( maxBatch, 0 );
		const size_t B = (size_t)maxBatch;
		WSP_CHECK( devAlloc( c.melMax, B ) );
		// the halo rows are rewritten by every encode (mel_window_kernel, EPI_CONV1) except row 0, which no packing moves
		WSP_CHECK( devAlloc( c.melF16, B * kFramesPad * 80, true ) );
		WSP_CHECK( devAlloc( c.conv1, B * kFramesPad * d, true ) );
		WSP_CHECK( devAlloc( c.x, B * T * d ) );
		WSP_CHECK( devAlloc( c.xn, B * T * d ) );
		WSP_CHECK( devAlloc( c.q, B * T * d ) );
		WSP_CHECK( devAlloc( c.k, B * T * d ) );
		WSP_CHECK( devAlloc( c.vt, B * H * 64 * c.Tp, true ) );                // pad columns are re-zeroed by the QKV epilogue
		WSP_CHECK( devAlloc( c.attn, B * T * d ) );
		WSP_CHECK( devAlloc( c.h, B * T * 4 * d ) );
		WSP_CHECK( devAlloc( c.crossK, (size_t)L * B * T * d ) );
		WSP_CHECK( devAlloc( c.crossV, (size_t)L * B * T * d ) );
		WSP_CHECK( devAlloc( c.selfK, (size_t)L * B * hp.n_text_ctx * d, true ) );
		WSP_CHECK( devAlloc( c.selfV, (size_t)L * B * hp.n_text_ctx * d, true ) );
		WSP_CHECK( devAlloc( c.xd, B * kMaxDecodeTokens * d ) );
		WSP_CHECK( devAlloc( c.qd, B * kMaxDecodeTokens * d ) );
		WSP_CHECK( devAlloc( c.attnD, B * kMaxDecodeTokens * d ) );
		WSP_CHECK( devAlloc( c.hD, B * kMaxDecodeTokens * 4 * d ) );
		WSP_CHECK( devAlloc( c.logits, B * kAllLogitsTokens * hp.n_vocab ) );
		WSP_CHECK( devAlloc( c.probs, B * kAllLogitsTokens * hp.n_vocab ) );
		WSP_CHECK( devAlloc( c.tieScratch, B * ( (size_t)hp.n_vocab + 1024 ) ) );
		WSP_CHECK( devAlloc( c.tokensDev, B * kMaxDecodeTokens, true ) );
		WSP_CHECK( devAlloc( c.dNPast, 8, true ) );
		c.dFlags = c.dNPast + 2;
		c.dStep = c.dNPast + 4;
		c.nEnded = c.dNPast + 6;
		WSP_CHECK( devAlloc( c.sampled, B ) );
		c.histCap = hp.n_text_ctx;
		WSP_CHECK( devAlloc( c.history, B * c.histCap, true ) );
		WSP_CHECK( devAlloc( c.endStep, B, true ) );
		WSP_CHECK( devAlloc( c.winCtl, 4 + B, true ) );
		WSP_CHECK( devAlloc( c.winState, B, true ) );
		WSP_CHECK( devAlloc( c.tokenLog, B * c.histCap, true ) );
		if( e->nLangs > 0 )
		{
			WSP_CHECK( devAlloc( c.langIds, B, true ) );
			WSP_CHECK( devAlloc( c.langProbs, B * e->nLangs, true ) );
		}
		WSP_CUDA( cudaHostAlloc( (void**)&c.nEndedHost, sizeof( int ), cudaHostAllocMapped ) );
		*c.nEndedHost = 0;
		WSP_CUDA( cudaHostGetDevicePointer( (void**)&c.nEndedMapped, c.nEndedHost, 0 ) );

		// ---- tensor maps ----
		c.bnD = pickBN( d ); c.bn3D = pickBN( 3 * d ); c.bn4D = pickBN( 4 * d ); c.bnCross = pickBN( L * 2 * d );
		bool ok = true;
		// A operands (activations): box rows = 128
		ok &= gemm::makeMap2D( &c.mapMel, c.melF16, 80, B * kFramesPad, 80 * 2, gemm::BM );
		ok &= gemm::makeMap2D( &c.mapConv1Even, c.conv1, d, B * ( kFramesPad / 2 ), (uint64_t)2 * d * 2, gemm::BM );
		ok &= gemm::makeMap2D( &c.mapConv1Odd, c.conv1 + d, d, B * ( kFramesPad / 2 ), (uint64_t)2 * d * 2, gemm::BM );
		ok &= gemm::makeMap2D( &c.mapXn, c.xn, d, B * T, (uint64_t)d * 2, gemm::BM );
		ok &= gemm::makeMap2D( &c.mapAttn, c.attn, d, B * T, (uint64_t)d * 2, gemm::BM );
		ok &= gemm::makeMap2D( &c.mapH, c.h, 4 * d, B * T, (uint64_t)4 * d * 2, gemm::BM );
		// B operands (weights): box rows = BN of the GEMM that uses them
		ok &= gemm::makeMap2D( &c.mapConv1W, e->conv1w, 3 * kConv1KTap, d, (uint64_t)3 * kConv1KTap * 2, c.bnD );
		ok &= gemm::makeMap2D( &c.mapConv2W, e->conv2w, 3 * d, d, (uint64_t)3 * d * 2, c.bnD );
		ok &= gemm::makeMap2D( &c.mapCrossW, e->crossW, d, (uint64_t)L * 2 * d, (uint64_t)d * 2, c.bnCross );
		const int Le = hp.n_audio_layer;
		c.mapWqkv.resize( Le ); c.mapWo.resize( Le ); c.mapW1.resize( Le ); c.mapW2.resize( Le );
		for( int i = 0; i < Le; i++ )
		{
			ok &= gemm::makeMap2D( &c.mapWqkv[ i ], e->enc[ i ].wqkv, d, 3 * d, (uint64_t)d * 2, c.bn3D );
			ok &= gemm::makeMap2D( &c.mapWo[ i ], e->enc[ i ].wo, d, d, (uint64_t)d * 2, c.bnD );
			ok &= gemm::makeMap2D( &c.mapW1[ i ], e->enc[ i ].w1, d, 4 * d, (uint64_t)d * 2, c.bn4D );
			ok &= gemm::makeMap2D( &c.mapW2[ i ], e->enc[ i ].w2, 4 * d, d, (uint64_t)4 * d * 2, c.bnD );
		}
		// attention operands
		ok &= gemm::makeMap2D( &c.mapQ, c.q, 64, B * H * T, 128, 128 );
		ok &= gemm::makeMap2D( &c.mapK, c.k, 64, B * H * T, 128, 128 );
		ok &= gemm::makeMap2D( &c.mapVt, c.vt, c.Tp, B * H * 64, (uint64_t)c.Tp * 2, 64 );
		if( !ok ) return fail( WSP_E_CUDA, "cuTensorMapEncodeTiled failed (driver too old for TMA?)" );
		// per-layer pointer table of the two decoder-step kernels: the persistent one (decode_mega.cu) and the dataflow one
		// (decode_flow.cu, which also gets per-CTA bias slabs and sentinel-filled exchange buffers)
		{
			const kern::FlowGeom g = kern::flowGeometry( d, hp.n_vocab, e->numSMs );
			c.flowGeom = g;
			const size_t slabLayer = (size_t)g.grid * g.slabFloats;
			WSP_CHECK( devAlloc( c.flowBias, slabLayer * L ) );
			std::vector<kern::DecStepLayer> sl( (size_t)L );
			for( int i = 0; i < L; i++ )
			{
				const DecLayerW& W = e->dec[ i ];
				kern::DecStepLayer& m = sl[ i ];
				m.ln1g = W.ln1.g; m.ln1b = W.ln1.b; m.lncg = W.lnc.g; m.lncb = W.lnc.b; m.ln3g = W.ln3.g; m.ln3b = W.ln3.b;
				m.wqkv = W.wqkv; m.wo = W.wo; m.wcq = W.wcq; m.wco = W.wco; m.w1 = W.w1; m.w2 = W.w2;
				m.bqkv = W.bqkv; m.bo = W.bo; m.bcq = W.bcq; m.bco = W.bco; m.b1 = W.b1; m.b2 = W.b2;
				m.biasSlab = c.flowBias + (size_t)i * slabLayer;
				m.kCache = c.selfK + (size_t)i * B * hp.n_text_ctx * d;
				m.vCache = c.selfV + (size_t)i * B * hp.n_text_ctx * d;
				m.crossK = c.crossK + (size_t)i * B * T * d;
				m.crossV = c.crossV + (size_t)i * B * T * d;
				WSP_CUDA( kern::flowBuildBiasSlab( c.flowBias + (size_t)i * slabLayer, g, d, W.bqkv, W.bo, W.bcq, W.bco, W.b1, W.b2, c.stream ) );
			}
			WSP_CHECK( devAlloc( c.stepLayers, (size_t)L ) );
			WSP_CUDA( cudaMemcpy( c.stepLayers, sl.data(), sl.size() * sizeof( kern::DecStepLayer ), cudaMemcpyHostToDevice ) );
			WSP_CHECK( devAlloc( c.megaBarrier, 64, true ) );
			const size_t exBytes = kern::flowExchangeBytes( d, maxBatch, L );
			WSP_CHECK( devAlloc( c.flowExch, exBytes ) );
			WSP_CUDA( cudaMemset( c.flowExch, 0xFF, exBytes ) );
			WSP_CHECK( devAlloc( c.flowCtrl, 8, true ) );
			WSP_CHECK( devAlloc( c.stepMarks, kStepMarks, true ) );
			const char* env = getenv( "WSP_TIMING_CTA" );
			if( env ) c.stepTimingCta = atoi( env );
		}
		WSP_CUDA( kern::prepare( 4 * d ) );
		WSP_CUDA( kern::megaPrepare( d ) );
		WSP_CUDA( kern::flowPrepare( d ) );
		WSP_CUDA( cudaDeviceSynchronize() );
		*out = cp.release();
		return WSP_OK;
	}

	// ===============================================================================================================
	// stage timing (wsp_timings): 0 = mel, 1 = encoder, 2 = decoder
	// ===============================================================================================================
	static float addStage( Context& c, int stage, cudaEvent_t from, cudaEvent_t to, int calls )
	{
		float ms = 0;
		cudaEventElapsedTime( &ms, from, to );
		c.ms[ stage ] += ms; c.calls[ stage ] += calls;
		return ms;
	}
	// one call of a stage: what work() enqueues is timed, what after() enqueues (results on their way back) is not; returns synchronised
	template<class W, class A>
	static int timeStage( Context& c, int stage, W work, A after )
	{
		WSP_CUDA( cudaEventRecord( c.ev[ 0 ], c.stream ) );
		WSP_CHECK( work() );
		WSP_CUDA( cudaEventRecord( c.ev[ 1 ], c.stream ) );
		WSP_CHECK( after() );
		WSP_CUDA( cudaStreamSynchronize( c.stream ) );
		addStage( c, stage, c.ev[ 0 ], c.ev[ 1 ], 1 );
		return WSP_OK;
	}
	template<class W>
	static int timeStage( Context& c, int stage, W work ) { return timeStage( c, stage, work, []() -> int { return WSP_OK; } ); }

	// ===============================================================================================================
	// mel
	// ===============================================================================================================
	static int ensureMelSlot( Context& c, int slot, int nLen )
	{
		if( slot < 0 || slot >= c.maxB ) return fail( WSP_E_BOUNDS, "chunk slot out of range" );
		MelSlot& s = c.slots[ slot ];
		if( nLen > s.cap )
		{
			if( s.mel ) cudaFree( s.mel );
			s.mel = nullptr;
			const int cap = nLen < kFrames ? kFrames : nLen;
			c.devBytes -= (uint64_t)80 * s.cap * 4;
			WSP_CHECK( devAlloc( s.mel, (size_t)80 * cap ) );
			c.devBytes += (uint64_t)80 * cap * 4;
			s.cap = cap;
		}
		s.nLen = nLen;
		return WSP_OK;
	}

	// frames of the whole-clip log-mel of nSamples samples: n / hop (whisper.cpp:2080), hop 160 for whisper_pcm_to_mel and 320 for the
	// phase vocoder of whisper_pcm_to_mel_phase_vocoder (:2299-2311) that speed-up selects
	static int melFrames( const Context& c, int nSamples ) { return nSamples / ( c.speedUp ? 320 : 160 ); }
	static const kern::MelTables& melTables( const Context& c ) { return c.speedUp ? c.e->melVocoder : c.e->mel; }

	// log-mel of chunks [0, batch) into slots slotOf( b ), in one triple of launches per 16 chunks: pcmOf( b ) / samplesOf( b ) name
	// chunk b's device PCM.  Chunk b's maximum goes to melMax[b], which only this launch reads.
	template<class S, class P, class N>
	static int melBatchFromDevicePcm( Context& c, int batch, S slotOf, P pcmOf, N samplesOf )
	{
		for( int b0 = 0; b0 < batch; b0 += kern::MEL_BATCH )
		{
			kern::MelBatch mb{};
			mb.count = batch - b0 < kern::MEL_BATCH ? batch - b0 : kern::MEL_BATCH;
			mb.maxSlots = c.melMax + b0;
			for( int i = 0; i < mb.count; i++ )
			{
				const int n = samplesOf( b0 + i );
				const int nLen = melFrames( c, n );
				WSP_CHECK( ensureMelSlot( c, slotOf( b0 + i ), nLen ) );
				mb.pcm[ i ] = pcmOf( b0 + i );
				mb.mel[ i ] = c.slots[ slotOf( b0 + i ) ].mel;
				mb.nSamples[ i ] = n;
				mb.nLen[ i ] = nLen;
			}
			WSP_CUDA( kern::melBatchPower( melTables( c ), mb, c.speedUp, c.stream ) );
			WSP_CUDA( kern::melBatchNormalize( mb, c.stream ) );
			launched( 3 );
		}
		return WSP_OK;
	}

	static int ensurePcm( Context& c, size_t floats )
	{
		if( floats <= c.pcmCap ) return WSP_OK;
		if( c.pcmDev ) { WSP_CUDA( cudaStreamSynchronize( c.stream ) ); cudaFree( c.pcmDev ); c.pcmDev = nullptr; }
		c.devBytes -= (uint64_t)c.pcmCap * 4;
		WSP_CHECK( devAlloc( c.pcmDev, floats ) );
		c.devBytes += (uint64_t)floats * 4;
		c.pcmCap = floats;
		return WSP_OK;
	}

	// room for `samples` of signal energy per slot, on the device and, for window calls, in pinned host memory; what the slots hold
	// is kept
	static int ensureEnergy( Context& c, size_t samples, bool host )
	{
		if( samples > c.energyCap )
		{
			WSP_CUDA( cudaStreamSynchronize( c.stream ) );
			float* grown = nullptr;
			WSP_CHECK( devAlloc( grown, (size_t)c.maxB * samples ) );
			if( c.energy )
			{
				WSP_CUDA( cudaMemcpy2D( grown, samples * 4, c.energy, c.energyCap * 4, c.energyCap * 4, (size_t)c.maxB, cudaMemcpyDeviceToDevice ) );
				cudaFree( c.energy );
			}
			if( c.energyHost )
			{
				float* grownHost = nullptr;
				WSP_CUDA( cudaHostAlloc( (void**)&grownHost, (size_t)c.maxB * samples * 4, cudaHostAllocDefault ) );
				for( size_t b = 0; b < (size_t)c.maxB; b++ ) memcpy( grownHost + b * samples, c.energyHost + b * c.energyCap, c.energyCap * 4 );
				cudaFreeHost( c.energyHost );
				c.energyHost = grownHost;
			}
			c.devBytes += (uint64_t)c.maxB * ( samples - c.energyCap ) * 4;
			c.energy = grown;
			c.energyCap = samples;
		}
		if( host && !c.energyHost ) WSP_CUDA( cudaHostAlloc( (void**)&c.energyHost, (size_t)c.maxB * c.energyCap * 4, cudaHostAllocDefault ) );
		return WSP_OK;
	}
	// signal energy of chunks [0, batch) into slots slotOf( b ) in one launch; pcmOf( b ) / samplesOf( b ) name chunk b's device PCM.
	// ensureEnergy has made room.
	template<class S, class P, class N>
	static int energyFromDevicePcm( Context& c, int batch, S slotOf, P pcmOf, N samplesOf )
	{
		kern::EnergyBatch eb{};
		eb.out = c.energy;
		eb.stride = (int64_t)c.energyCap;
		eb.count = batch;
		for( int b = 0; b < batch; b++ )
		{
			eb.pcm[ b ] = pcmOf( b );
			eb.nSamples[ b ] = samplesOf( b );
			eb.row[ b ] = (uint8_t)slotOf( b );
			c.energyLen[ (size_t)slotOf( b ) ] = eb.nSamples[ b ];
		}
		WSP_CUDA( kern::signalEnergy( eb, c.stream ) );
		launched();
		return WSP_OK;
	}
	static_assert( kern::ENERGY_BATCH >= 256, "one energy launch covers the largest context" );

	// whisper_full_params::token_timestamps: the signal energy of window calls and pcm_to_mel
	int ctxSetTokenTimestamps( Context& c, int on )
	{
		if( on != 0 && on != 1 ) return fail( WSP_E_INVALIDARG, "token timestamps must be 0 or 1" );
		c.tokenTimestamps = on != 0;
		return WSP_OK;
	}

	// one clip's host PCM into c.pcmDev, then melOf() enqueues its log-mel; both are timed as the mel stage
	template<class M>
	static int pcmToMelTimed( Context& c, const float* pcmHost, int nSamples, M melOf )
	{
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		WSP_CHECK( ensurePcm( c, (size_t)( nSamples > 0 ? nSamples : 1 ) ) );
		return timeStage( c, 0, [ & ]() -> int {
			if( nSamples > 0 )
				WSP_CUDA( cudaMemcpyAsync( c.pcmDev, pcmHost, (size_t)nSamples * 4, cudaMemcpyHostToDevice, c.stream ) );
			return melOf();
		} );
	}

	int ctxPcmToMel( Context& c, int slot, const float* pcmHost, int nSamples )
	{
		if( ( !pcmHost && nSamples != 0 ) || nSamples < 0 ) return fail( WSP_E_INVALIDARG, "pcm" );
		if( c.tokenTimestamps ) WSP_CHECK( ensureEnergy( c, (size_t)( nSamples > 0 ? nSamples : 1 ), false ) );
		return pcmToMelTimed( c, pcmHost, nSamples, [ & ]() -> int {
			auto slotOf = [ & ]( int ) { return slot; };
			auto pcmOf = [ & ]( int ) { return (const float*)c.pcmDev; };
			auto samplesOf = [ & ]( int ) { return nSamples; };
			WSP_CHECK( melBatchFromDevicePcm( c, 1, slotOf, pcmOf, samplesOf ) );
			return c.tokenTimestamps ? energyFromDevicePcm( c, 1, slotOf, pcmOf, samplesOf ) : WSP_OK;
		} );
	}

	// One window of a streamed clip (Whisper/Whisper/MelStreamer.cpp:128-236): frames [0, nFrames) of the PCM handed in — the PCM may
	// (and, except at the end of a stream, does) extend past the last frame so that every frame sees its full 400 samples — normalised
	// by the maximum over THESE frames only, floored at 1e-20 (:136), or by `forcedMax` when the streamer re-uses the maximum of the
	// previous, longer window that ended at the same frame (:152-166).  Same kernels as the whole-clip path.
	int ctxPcmToMelWindow( Context& c, int slot, const float* pcmHost, int nSamples, int nFrames, const float* forcedMax, float* maxOut )
	{
		if( ( !pcmHost && nSamples != 0 ) || nSamples < 0 || nFrames < 0 ) return fail( WSP_E_INVALIDARG, "pcm / frame count" );
		// the reference streams only the 400-point transform (MelStreamer.cpp); it has no streamed phase-vocoder window to follow
		if( c.speedUp ) return fail( WSP_E_NOTIMPL, "no streamed log-mel window with speed-up on" );
		return pcmToMelTimed( c, pcmHost, nSamples, [ & ]() -> int {
			WSP_CHECK( ensureMelSlot( c, slot, nFrames ) );
			kern::MelBatch mb{};
			mb.pcm[ 0 ] = c.pcmDev;
			mb.mel[ 0 ] = c.slots[ slot ].mel;
			mb.nSamples[ 0 ] = nSamples;
			mb.nLen[ 0 ] = nFrames;
			mb.maxSlots = c.melMax + slot;
			mb.count = 1;
			WSP_CUDA( kern::melBatchPower( c.e->mel, mb, false, c.stream ) );
			int32_t ordered = 0;
			WSP_CUDA( cudaMemcpyAsync( &ordered, c.melMax + slot, 4, cudaMemcpyDeviceToHost, c.stream ) );
			WSP_CUDA( cudaStreamSynchronize( c.stream ) );
			// the device keeps the maximum as an order-preserving integer (kernels_frontend.cu: orderedFromFloat)
			auto toFloat = []( int32_t i ) { const int32_t b = i >= 0 ? i : i ^ 0x7FFFFFFF; float f; memcpy( &f, &b, 4 ); return f; };
			auto toOrdered = []( float f ) { int32_t b; memcpy( &b, &f, 4 ); return b >= 0 ? b : b ^ 0x7FFFFFFF; };
			float mmax = toFloat( ordered );
			if( !( mmax > 1e-20f ) ) mmax = 1e-20f;
			if( maxOut ) *maxOut = mmax;
			if( forcedMax ) mmax = *forcedMax;
			const int32_t wanted = toOrdered( mmax );
			if( wanted != ordered )
				WSP_CUDA( cudaMemcpyAsync( c.melMax + slot, &wanted, 4, cudaMemcpyHostToDevice, c.stream ) );
			WSP_CUDA( kern::melBatchNormalize( mb, c.stream ) );
			launched( 3 );
			return WSP_OK;
		} );
	}

	int ctxSetMel( Context& c, int slot, const float* melHost, int nLen )
	{
		if( !melHost || nLen < 0 ) return fail( WSP_E_INVALIDARG, "mel" );
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		WSP_CHECK( ensureMelSlot( c, slot, nLen ) );
		WSP_CUDA( cudaMemcpyAsync( c.slots[ slot ].mel, melHost, (size_t)80 * nLen * 4, cudaMemcpyHostToDevice, c.stream ) );
		WSP_CUDA( cudaStreamSynchronize( c.stream ) );
		return WSP_OK;
	}

	// ===============================================================================================================
	// encoder
	// ===============================================================================================================
	// chunk b's window is frames [offsets[b], offsets[b] + 2n) of slot slots[b]'s log-mel (slots == nullptr: slot b; offsets == nullptr: 0)
	static int encodeAsync( Context& c, const int32_t* slots, const int32_t* offsets, int batch )
	{
		Engine& e = *c.e;
		const HParams& hp = e.hp;
		const int d = hp.n_audio_state, H = hp.n_audio_head, L = hp.n_text_layer;
		// audio positions of this encode (whisper.cpp:1092): the window is 2T mel frames, every chunk takes 2T + 2 rows (halo, frames,
		// halo) in melF16 / conv1 and T rows everywhere after conv2
		const int T = c.audioCtx > 0 ? c.audioCtx : hp.n_audio_ctx;
		const int frames = 2 * T, rowsPad = frames + 2;
		cudaStream_t s = c.stream;
		for( int b = 0; b < batch; b++ )
		{
			const int slot = slots ? slots[ b ] : b;
			const MelSlot& ms = c.slots[ slot ];
			if( !ms.mel ) return fail( WSP_E_INVALIDARG, "no mel in slot " + std::to_string( slot ) );
			const int off = offsets ? offsets[ b ] : 0;
			if( off < 0 ) return fail( WSP_E_INVALIDARG, "negative mel offset" );
			WSP_CUDA( kern::melWindow( ms.mel, ms.nLen, off, c.melF16 + (size_t)b * rowsPad * 80, frames, s ) );
			launched();
		}
		// from here on the cross-KV memories are (being) rewritten with T rows per chunk: decodes attend over T keys
		c.encCtx = T;
		gemm::Launch g;
		// conv1 + bias + GELU -> f16, time-major with halo (a3)
		g = gemm::Launch();
		g.mapA = c.mapMel; g.mapA2 = c.mapMel; g.mapB = c.mapConv1W;
		g.M = batch * rowsPad - 2; g.N = d; g.K = 3 * kConv1KTap; g.kTap = kConv1KTap / gemm::BK;
		g.ep.M = g.M; g.ep.N = d; g.ep.ld = d; g.ep.bias = e.conv1b; g.ep.out_a = c.conv1;
		g.ep.rows_per_chunk = rowsPad; g.ep.valid_per_chunk = frames; g.ep.nchunks = batch;
		WSP_CUDA( gemm::launch( g, gemm::EPI_CONV1, gemm::A_CONV_S1, c.bnD, e.numSMs, s ) );
		// conv2 (stride 2) + bias + GELU + positional embedding -> f32 residual stream (a4)
		g = gemm::Launch();
		g.mapA = c.mapConv1Even; g.mapA2 = c.mapConv1Odd; g.mapB = c.mapConv2W;
		g.M = batch * ( rowsPad / 2 ) - 1; g.N = d; g.K = 3 * d; g.kTap = d / gemm::BK;
		g.ep.M = g.M; g.ep.N = d; g.ep.ld = d; g.ep.bias = e.conv2b; g.ep.pos = e.encPos; g.ep.out_f32 = c.x;
		g.ep.rows_per_chunk = rowsPad / 2; g.ep.valid_per_chunk = T; g.ep.nchunks = batch; g.ep.T = T; g.ep.d = d;
		WSP_CUDA( gemm::launch( g, gemm::EPI_CONV2, gemm::A_CONV_S2, c.bnD, e.numSMs, s ) );
		launched( 2 );

		const int M = batch * T;
		const int nLayers = ( c.debugEncLayers >= 0 && c.debugEncLayers < hp.n_audio_layer ) ? c.debugEncLayers : hp.n_audio_layer;
		for( int il = 0; il < nLayers; il++ )
		{
			const EncLayerW& W = e.enc[ il ];
			WSP_CUDA( kern::layerNormF16( c.x, W.ln1.g, W.ln1.b, c.xn, M, d, s ) );
			// Q | K | V projections in one GEMM; epilogue writes head-major f16 Q, K and transposed V (a6, a7)
			g = gemm::Launch();
			g.mapA = c.mapXn; g.mapA2 = c.mapXn; g.mapB = c.mapWqkv[ il ];
			g.M = M; g.N = 3 * d; g.K = d;
			g.ep.M = M; g.ep.N = 3 * d; g.ep.bias = W.bqkv; g.ep.out_a = c.q; g.ep.out_b = c.k; g.ep.out_c = c.vt;
			g.ep.T = T; g.ep.Tp = c.Tp; g.ep.H = H; g.ep.d = d;
			WSP_CUDA( gemm::launch( g, gemm::EPI_QKV, gemm::A_PLAIN, c.bn3D, e.numSMs, s ) );
			// fused flash attention (a8)
			attn::EncParams ap;
			ap.T = T; ap.H = H; ap.nBH = batch * H; ap.d = d; ap.out = c.attn;
			ap.scale_log2 = (float)( ( 1.0 / sqrt( 64.0 ) ) * 1.4426950408889634 );
			WSP_CUDA( attn::launchEnc( c.mapQ, c.mapK, c.mapVt, ap, s ) );
			// output projection + bias + residual (a9)
			g = gemm::Launch();
			g.mapA = c.mapAttn; g.mapA2 = c.mapAttn; g.mapB = c.mapWo[ il ];
			g.M = M; g.N = d; g.K = d;
			g.ep.M = M; g.ep.N = d; g.ep.ld = d; g.ep.bias = W.bo; g.ep.resid = c.x; g.ep.out_f32 = c.x;
			WSP_CUDA( gemm::launch( g, gemm::EPI_BIAS_RESID, gemm::A_PLAIN, c.bnD, e.numSMs, s ) );
			// MLP (a10)
			WSP_CUDA( kern::layerNormF16( c.x, W.ln2.g, W.ln2.b, c.xn, M, d, s ) );
			g = gemm::Launch();
			g.mapA = c.mapXn; g.mapA2 = c.mapXn; g.mapB = c.mapW1[ il ];
			g.M = M; g.N = 4 * d; g.K = d;
			g.ep.M = M; g.ep.N = 4 * d; g.ep.ld = 4 * d; g.ep.bias = W.b1; g.ep.out_a = c.h;
			WSP_CUDA( gemm::launch( g, gemm::EPI_BIAS_GELU_F16, gemm::A_PLAIN, c.bn4D, e.numSMs, s ) );
			g = gemm::Launch();
			g.mapA = c.mapH; g.mapA2 = c.mapH; g.mapB = c.mapW2[ il ];
			g.M = M; g.N = d; g.K = 4 * d;
			g.ep.M = M; g.ep.N = d; g.ep.ld = d; g.ep.bias = W.b2; g.ep.resid = c.x; g.ep.out_f32 = c.x;
			WSP_CUDA( gemm::launch( g, gemm::EPI_BIAS_RESID, gemm::A_PLAIN, c.bnD, e.numSMs, s ) );
			launched( 7 );
		}
		// ln_post (a11) and the cross-attention K/V memories of every decoder layer in one GEMM (a12)
		WSP_CUDA( kern::layerNormF16( c.x, e.encLnPost.g, e.encLnPost.b, c.xn, M, d, s ) );
		g = gemm::Launch();
		g.mapA = c.mapXn; g.mapA2 = c.mapXn; g.mapB = c.mapCrossW;
		g.M = M; g.N = L * 2 * d; g.K = d;
		g.ep.M = M; g.ep.N = g.N; g.ep.bias = e.crossB; g.ep.out_a = c.crossK; g.ep.out_b = c.crossV;
		g.ep.T = T; g.ep.H = H; g.ep.d = d; g.ep.nchunks = c.maxB;
		g.ep.layer_stride = (size_t)c.maxB * hp.n_audio_ctx * d;   // [L][maxB][H][T][64] inside the 1500-row layers of the pointer tables
		g.ep.scale = (float)pow( 64.0, -0.25 );   // whisper.cpp:1465
		WSP_CUDA( gemm::launch( g, gemm::EPI_CROSSKV, gemm::A_PLAIN, c.bnCross, e.numSMs, s ) );
		launched( 2 );
		return WSP_OK;
	}

	// whisper_full's audio_ctx (whisper.cpp:1092, 1528, 2836): encode only the first n audio positions; n <= 0 = the model's own
	int ctxSetAudioCtx( Context& c, int n )
	{
		if( n > c.e->hp.n_audio_ctx ) return fail( WSP_E_INVALIDARG, "audio_ctx exceeds the model's n_audio_ctx" );
		c.audioCtx = n > 0 ? n : 0;
		return WSP_OK;
	}

	// whisper_full_params::speed_up (sFullParams.h:33 SpeedupAudio): whole-clip log-mels through the phase vocoder
	int ctxSetSpeedUp( Context& c, int on )
	{
		if( on != 0 && on != 1 ) return fail( WSP_E_INVALIDARG, "speed-up must be 0 or 1" );
		c.speedUp = on != 0;
		return WSP_OK;
	}

	int ctxEncode( Context& c, const int32_t* offsets, int batch )
	{
		if( batch < 1 || batch > c.maxB ) return fail( WSP_E_BOUNDS, "batch exceeds the context's max_batch" );
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		return timeStage( c, 1, [ & ]() -> int { return encodeAsync( c, nullptr, offsets, batch ); } );
	}

	// ===============================================================================================================
	// decoder
	// ===============================================================================================================
	namespace
	{
		struct ProfScope
		{
			Context& c;
			bool active;
			ProfScope( Context& ctx, int kind ) : c( ctx ), active( ctx.prof.on )
			{
				if( !active ) return;
				KernelProfile& p = c.prof;
				if( p.used + 2 > p.pool.size() )
				{
					for( int i = 0; i < 2; i++ ) { cudaEvent_t e; cudaEventCreate( &e ); p.pool.push_back( e ); }
				}
				p.kinds.push_back( kind );
				cudaEventRecord( p.pool[ p.used ], c.stream );
			}
			~ProfScope()
			{
				if( !active ) return;
				cudaEventRecord( c.prof.pool[ c.prof.used + 1 ], c.stream );
				c.prof.used += 2;
			}
		};
	}
#define WSP_KERNEL( kind, expr ) do { ProfScope _ps( c, kind ); WSP_CUDA( expr ); } while( 0 )

	// Greedy sampling of the last token of every chunk from c.logits (sampler + advance kernel): the next tokens, n_past and the
	// step counter stay on the device
	static int enqueueSampler( Context& c, int N, int batch )
	{
		const Engine& e = *c.e;
		kern::SampleArgs sa;
		sa.logits = c.logits; sa.probs = c.probs; sa.tieScratch = c.tieScratch; sa.B = batch; sa.nVocab = e.hp.n_vocab;
		sa.tokenBeg = e.tokBeg; sa.tokenSot = e.tokSot; sa.tokenSolm = e.tokSolm; sa.tokenNot = e.tokNot;
		sa.dForceTs = c.dFlags; sa.out = c.sampled; sa.nextTokens = c.tokensDev; sa.dNPast = c.dNPast; sa.N = N;
		sa.history = c.history; sa.histCap = c.histCap; sa.dStep = c.dStep;
		if( c.eotArmed )
		{
			sa.tokenEot = e.tokEot; sa.endStep = c.endStep; sa.nEnded = c.nEnded; sa.nEndedHost = c.nEndedMapped;
			sa.winCtl = c.winCtl; sa.winState = c.winState; sa.tokenLog = c.tokenLog;
		}
		WSP_KERNEL( KK_OTHER, kern::sampleGreedy( sa, c.stream ) );
		return WSP_OK;
	}

	// One decoder pass kernel by kernel (kernels_decode.cu): embedding, 8 launches per layer, final LN + logits
	static int enqueuePerOp( Context& c, int N, int batch, bool allLogits, int& n )
	{
		Engine& e = *c.e;
		const HParams& hp = e.hp;
		// T = cross-attention keys: the audio positions of the last encode (whisper.cpp:1528)
		const int d = hp.n_text_state, H = hp.n_text_head, T = c.encCtx, nCtx = hp.n_text_ctx;
		cudaStream_t s = c.stream;
		const int cols = batch * N;
		const float qkScale = (float)pow( 64.0, -0.25 );   // whisper.cpp:1588, 1595, 1700
		// y = epi( W x + bias ) for every column: x = LayerNorm( c.xd ) with `ln`, or the f16 rows xF16 when ln is null
		auto skinny = [ & ]( const __half* W, const float* bias, int nOut, int K, const LnW* ln, const __half* xF16, kern::SkinnyEpi epi, float* outF32, __half* outF16 = nullptr ) {
			kern::SkinnyArgs a;
			a.W = W; a.nOut = nOut; a.K = K; a.xStride = K; a.nCols = cols;
			if( ln ) { a.xF32 = c.xd; a.gamma = ln->g; a.beta = ln->b; }
			else a.xF16 = xF16;
			a.epi = epi; a.bias = bias; a.outF32 = outF32; a.outF16 = outF16;
			if( epi == kern::SK_QKV || epi == kern::SK_Q_SCALE ) a.scale = qkScale;
			a.ld = epi == kern::SK_QKV ? d : nOut;
			return a;
		};
		c.lastPerOpN = N;
		// wsp_debug_set_decoder_stop: the pass ends after op `op` of layer `il` (0 QKV, 1 self attention, 2 self-out, 3 cross Q,
		// 4 cross attention, 5 cross-out, 6 fc1, 7 fc2)
		auto stopAfter = [ & ]( int il, int op ) { return c.decoderStopped() && c.debugDecLayer == il && ( il < 0 || c.debugDecOp == op ); };
		WSP_KERNEL( KK_OTHER, kern::embedTokens( e.tokEmb, e.decPos, c.tokensDev, c.dNPast, c.xd, batch, N, d, s ) ); n++;
		if( stopAfter( -1, 0 ) ) return WSP_OK;
		for( int il = 0; il < hp.n_text_layer; il++ )
		{
			const DecLayerW& W = e.dec[ il ];
			__half* kc = c.selfK + (size_t)il * c.maxB * nCtx * d;
			__half* vc = c.selfV + (size_t)il * c.maxB * nCtx * d;
			// LN + (Q | K | V); K, V appended to the f16 self-KV cache in the epilogue (a14)
			kern::SkinnyArgs a = skinny( W.wqkv, W.bqkv, 3 * d, d, &W.ln1, nullptr, kern::SK_QKV, c.qd );
			a.kCache = kc; a.vCache = vc; a.d = d; a.N = N; a.nTextCtx = nCtx; a.dNPast = c.dNPast;
			WSP_KERNEL( KK_SKINNY, kern::skinnyGemm( a, s ) ); n++;
			if( stopAfter( il, 0 ) ) return WSP_OK;
			WSP_KERNEL( KK_SELF, kern::selfAttnDecode( c.qd, kc, vc, c.attnD, batch, N, H, d, nCtx, c.dNPast, c.refThreads, s ) ); n++;
			if( stopAfter( il, 1 ) ) return WSP_OK;
			WSP_KERNEL( KK_SKINNY, kern::skinnyGemm( skinny( W.wo, W.bo, d, d, nullptr, c.attnD, kern::SK_BIAS_RESID, c.xd ), s ) ); n++;
			if( stopAfter( il, 2 ) ) return WSP_OK;
			// cross attention (a15)
			WSP_KERNEL( KK_SKINNY, kern::skinnyGemm( skinny( W.wcq, W.bcq, d, d, &W.lnc, nullptr, kern::SK_Q_SCALE, c.qd ), s ) ); n++;
			if( stopAfter( il, 3 ) ) return WSP_OK;
			const size_t crossOff = (size_t)il * c.maxB * hp.n_audio_ctx * d;   // layer stride of the pointer tables, whatever T is
			WSP_KERNEL( KK_CROSS, kern::crossAttnDecode( c.qd, c.crossK + crossOff, c.crossV + crossOff, c.attnD, batch, N, H, d, T, c.refThreads, s ) ); n++;
			if( stopAfter( il, 4 ) ) return WSP_OK;
			WSP_KERNEL( KK_SKINNY, kern::skinnyGemm( skinny( W.wco, W.bco, d, d, nullptr, c.attnD, kern::SK_BIAS_RESID, c.xd ), s ) ); n++;
			if( stopAfter( il, 5 ) ) return WSP_OK;
			// MLP (a16)
			WSP_KERNEL( KK_SKINNY, kern::skinnyGemm( skinny( W.w1, W.b1, 4 * d, d, &W.ln3, nullptr, kern::SK_GELU_F16, nullptr, c.hD ), s ) ); n++;
			if( stopAfter( il, 6 ) ) return WSP_OK;
			WSP_KERNEL( KK_SKINNY, kern::skinnyGemm( skinny( W.w2, W.b2, d, 4 * d, nullptr, c.hD, kern::SK_BIAS_RESID, c.xd ), s ) ); n++;
			if( stopAfter( il, 7 ) ) return WSP_OK;
		}
		if( c.decoderStopped() ) return WSP_OK;
		// final LN + logits = tok_emb^T x (a17): only the last token of each chunk unless all logits were requested
		kern::SkinnyArgs a = skinny( e.tokEmb, nullptr, hp.n_vocab, d, &e.decLn, nullptr, kern::SK_LOGITS, c.logits );
		if( !allLogits ) { a.xF32 = c.xd + (size_t)( N - 1 ) * d; a.xStride = (int64_t)N * d; a.nCols = batch; }
		WSP_KERNEL( KK_SKINNY, kern::skinnyGemm( a, s ) ); n++;
		return WSP_OK;
	}

	// what both step kernels are handed alike
	static kern::DecStepArgs stepArgs( const Context& c, int batch )
	{
		const Engine& e = *c.e;
		const HParams& hp = e.hp;
		kern::DecStepArgs a;
		a.layers = c.stepLayers; a.L = hp.n_text_layer; a.B = batch; a.maxB = c.maxB; a.H = hp.n_text_head; a.nTextCtx = hp.n_text_ctx;
		a.T = c.encCtx;   // cross-attention keys: the audio positions of the last encode (whisper.cpp:1528)
		a.nVocab = hp.n_vocab; a.refThreads = c.refThreads;
		a.tokEmb = e.tokEmb; a.decPos = e.decPos; a.lnfg = e.decLn.g; a.lnfb = e.decLn.b;
		a.tokens = c.tokensDev; a.dNPast = c.dNPast; a.logits = c.logits; a.timing = c.stepTiming ? c.stepMarks : nullptr;
		return a;
	}

	// Enqueue one decoder pass for `batch` chunks x N tokens.  Reads tokens from c.tokensDev, n_past / sampling flags from device
	// scalars (so the N = 1 instance can be captured once as a CUDA graph and replayed for every step).
	static int decodeEnqueue( Context& c, int N, int batch, bool allLogits, bool sample, int* launchesOut )
	{
		const Engine& e = *c.e;
		const int d = e.hp.n_text_state;
		if( c.decoderStopped() && sample && !allLogits ) return fail( WSP_E_INVALIDARG, "no sampling while a decoder stop is set" );
		// the steady state: embedding + all layers + logits in ONE kernel (a stopped pass runs kernel by kernel)
		const bool step = N == 1 && !allLogits && !c.decoderStopped();
		const kern::DecStepArgs sa = stepArgs( c, batch );
		int n = 0;
		if( step && c.stepMode == 2 && kern::flowSupported( d, batch, sa.T, sa.H, sa.nTextCtx, c.refThreads, c.flowGeom ) )
		{
			kern::FlowArgs fa{ sa };   // the dataflow kernel (decode_flow.cu)
			fa.exch = c.flowExch; fa.ctrl = c.flowCtrl; fa.g = c.flowGeom; fa.timingCta = c.stepTimingCta;
			WSP_KERNEL( KK_SKINNY, kern::decodeStepFlow( fa, d, e.numSMs, c.stream ) ); n++;
		}
		else if( step && c.stepMode == 1 && kern::megaSupported( d, batch, sa.T ) )
		{
			kern::MegaArgs ma{ sa };   // the persistent barrier kernel (decode_mega.cu)
			ma.x = c.xd; ma.q = c.qd; ma.attn = c.attnD; ma.h = c.hD; ma.barrier = c.megaBarrier;
			WSP_KERNEL( KK_SKINNY, kern::decodeStepMega( ma, d, e.numSMs, c.stream ) ); n++;
		}
		else
			WSP_CHECK( enqueuePerOp( c, N, batch, allLogits, n ) );
		if( sample && !allLogits ) { WSP_CHECK( enqueueSampler( c, N, batch ) ); n += 2; }
		if( launchesOut ) *launchesOut = n;
		return WSP_OK;
	}

	// Submit one decoder pass: the captured CUDA graph for the N = 1 steady state, plain launches otherwise.
	static int decodeSubmit( Context& c, int N, int batch, bool allLogits, bool sample )
	{
		int n = 0;
		if( N == 1 && !allLogits && sample && c.useGraph && !c.prof.on && !c.decoderStopped() )
		{
			const StepGraphKey key{ batch, c.encCtx, c.refThreads, c.stepMode, c.stepTiming, c.eotArmed };
			if( !c.stepGraph || !( c.stepGraphKey == key ) )
			{
				if( c.stepGraph ) { cudaGraphExecDestroy( c.stepGraph ); c.stepGraph = nullptr; }
				cudaGraph_t graph = nullptr;
				WSP_CUDA( cudaStreamBeginCapture( c.stream, cudaStreamCaptureModeThreadLocal ) );
				const int rc = decodeEnqueue( c, 1, batch, false, true, &n );
				cudaError_t ce = cudaStreamEndCapture( c.stream, &graph );
				if( rc < 0 ) { if( graph ) cudaGraphDestroy( graph ); return rc; }
				WSP_CUDA( ce );
				ce = cudaGraphInstantiate( &c.stepGraph, graph, 0 );
				cudaGraphDestroy( graph );
				WSP_CUDA( ce );
				c.stepGraphKey = key;
				c.stepGraphLaunches = n;
			}
			WSP_CUDA( cudaGraphLaunch( c.stepGraph, c.stream ) );
			g_launchCount.fetch_add( (uint64_t)c.stepGraphLaunches, std::memory_order_relaxed );
			return WSP_OK;
		}
		WSP_CHECK( decodeEnqueue( c, N, batch, allLogits, sample, &n ) );
		launched( n );
		if( allLogits && !c.decoderStopped() )
		{
			// probabilities for every row (the oracle keeps logits and probs of all N tokens, whisper.cpp:1855-1859); no sampling
			WSP_CUDA( kern::softmaxRows( c.logits, c.probs, batch * N, c.e->hp.n_vocab, c.stream ) );
			launched();
		}
		return WSP_OK;
	}

	int ctxDecode( Context& c, const int32_t* tokensHost, int nTokens, int nPast, int batch, uint32_t flags, wsp_token_data* sampledHost )
	{
		const HParams& hp = c.e->hp;
		const bool devTokens = ( flags & WSP_DECODE_DEVICE_TOKENS ) != 0;
		const bool allLogits = ( flags & WSP_DECODE_ALL_LOGITS ) != 0;
		const bool sample = ( flags & WSP_DECODE_NO_SAMPLE ) == 0;
		if( batch < 1 || batch > c.maxB ) return fail( WSP_E_BOUNDS, "batch exceeds the context's max_batch" );
		if( nTokens < 1 || nTokens > kMaxDecodeTokens ) return fail( WSP_E_BOUNDS, "n_tokens out of range" );
		if( allLogits && nTokens > kAllLogitsTokens ) return fail( WSP_E_BOUNDS, "ALL_LOGITS supports at most 8 tokens" );
		if( devTokens && nTokens != 1 ) return fail( WSP_E_INVALIDARG, "DEVICE_TOKENS implies n_tokens == 1" );
		if( !devTokens && !tokensHost ) return fail( WSP_E_POINTER, "tokens" );
		if( !devTokens && ( nPast < 0 || nPast + nTokens > hp.n_text_ctx ) ) return fail( WSP_E_BOUNDS, "n_past + n_tokens exceeds n_text_ctx" );
		// device-fed tokens continue from the device's n_past: its host mirror guards the KV cache and the positional table
		if( devTokens && c.nPastHost + nTokens > hp.n_text_ctx ) return fail( WSP_E_BOUNDS, "n_past + n_tokens exceeds n_text_ctx" );
		if( !devTokens )
			for( int i = 0; i < batch * nTokens; i++ )
				if( tokensHost[ i ] < 0 || tokensHost[ i ] >= hp.n_vocab ) return fail( WSP_E_INVALIDARG, "token id out of range" );
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		cudaStream_t s = c.stream;
		return timeStage( c, 2, [ & ]() -> int {
			if( !devTokens )
			{
				WSP_CUDA( cudaMemcpyAsync( c.tokensDev, tokensHost, (size_t)batch * nTokens * 4, cudaMemcpyHostToDevice, s ) );
				WSP_CUDA( kern::setInts( c.dNPast, nPast, 0, s ) );
				WSP_CUDA( kern::setInts( c.dFlags, ( flags & WSP_DECODE_FORCE_TIMESTAMP ) ? 1 : 0, ( flags & WSP_DECODE_INITIAL ) ? 1 : 0, s ) );
				launched( 2 );
			}
			WSP_CHECK( decodeSubmit( c, nTokens, batch, allLogits, sample ) );
			// the device advances n_past only when it samples (advance_kernel): mirror exactly that
			if( !devTokens ) c.nPastHost = nPast;
			if( sample && !allLogits ) c.nPastHost += nTokens;
			c.lastLogitRows = allLogits ? batch * nTokens : batch;
			return WSP_OK;
		}, [ & ]() -> int {
			if( sampledHost && sample && !allLogits )
				WSP_CUDA( cudaMemcpyAsync( sampledHost, c.sampled, (size_t)batch * sizeof( wsp_token_data ), cudaMemcpyDeviceToHost, s ) );
			return WSP_OK;
		} );
	}

	int ctxUploadPcm( Context& c, int slot, const float* pcmHost, int nSamples )
	{
		if( slot < 0 || slot >= c.maxB ) return fail( WSP_E_BOUNDS, "chunk slot out of range" );
		if( ( !pcmHost && nSamples != 0 ) || nSamples < 0 ) return fail( WSP_E_INVALIDARG, "pcm" );
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		MelSlot& s = c.slots[ slot ];
		if( nSamples > s.pcmCap )
		{
			if( s.pcm ) { WSP_CUDA( cudaStreamSynchronize( c.stream ) ); cudaFree( s.pcm ); s.pcm = nullptr; }
			WSP_CHECK( devAlloc( s.pcm, (size_t)( nSamples > 0 ? nSamples : 1 ) ) );
			s.pcmCap = nSamples;
		}
		s.pcmSamples = nSamples;
		s.stereoFrames = 0;
		WSP_CUDA( cudaMemcpyAsync( s.pcm, pcmHost, (size_t)nSamples * 4, cudaMemcpyHostToDevice, c.stream ) );
		WSP_CUDA( cudaStreamSynchronize( c.stream ) );
		return WSP_OK;
	}

	// the stereo pairs into the slot, and their downmix as its resident mono PCM
	int ctxUploadPcmStereo( Context& c, int slot, const float* lrHost, int nFrames )
	{
		if( slot < 0 || slot >= c.maxB ) return fail( WSP_E_BOUNDS, "chunk slot out of range" );
		if( ( !lrHost && nFrames != 0 ) || nFrames < 0 ) return fail( WSP_E_INVALIDARG, "pcm" );
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		MelSlot& s = c.slots[ slot ];
		if( nFrames > s.stereoCap )
		{
			if( s.stereo ) { WSP_CUDA( cudaStreamSynchronize( c.stream ) ); cudaFree( s.stereo ); s.stereo = nullptr; }
			c.devBytes -= (uint64_t)s.stereoCap * 8;
			s.stereoCap = 0;
			WSP_CHECK( devAlloc( s.stereo, (size_t)2 * nFrames ) );
			c.devBytes += (uint64_t)nFrames * 8;
			s.stereoCap = nFrames;
		}
		if( nFrames > s.pcmCap )
		{
			if( s.pcm ) { WSP_CUDA( cudaStreamSynchronize( c.stream ) ); cudaFree( s.pcm ); s.pcm = nullptr; }
			WSP_CHECK( devAlloc( s.pcm, (size_t)nFrames ) );
			s.pcmCap = nFrames;
		}
		s.pcmSamples = nFrames;
		s.stereoFrames = nFrames;
		if( nFrames > 0 ) WSP_CUDA( cudaMemcpyAsync( s.stereo, lrHost, (size_t)nFrames * 8, cudaMemcpyHostToDevice, c.stream ) );
		WSP_CUDA( kern::downmixStereo( s.stereo, s.pcm, nFrames, c.stream ) );
		launched();
		WSP_CUDA( cudaStreamSynchronize( c.stream ) );
		return WSP_OK;
	}

	// detectSpeaker for every segment of a batch: speakerSpan on the host picks each segment's frames (or its answer), then one launch
	// folds and decides them all between one copy in and one copy out
	int ctxChunkSpeakers( Context& c, int batch, const int32_t* segStart, const wsp_segment* segs, int32_t* speakers )
	{
		if( batch < 1 || batch > c.maxB ) return fail( WSP_E_BOUNDS, "batch exceeds the context's max_batch" );
		if( segStart[ 0 ] != 0 ) return fail( WSP_E_INVALIDARG, "seg_start[0] must be 0" );
		for( int b = 0; b < batch; b++ )
			if( segStart[ b + 1 ] < segStart[ b ] ) return fail( WSP_E_INVALIDARG, "seg_start decreases" );
		const size_t n = (size_t)segStart[ batch ];
		if( n == 0 ) return WSP_OK;
		if( !segs ) return fail( WSP_E_POINTER, "segs" );
		std::vector<kern::SpeakerJob> jobs( n );
		for( int b = 0; b < batch; b++ )
		{
			const MelSlot& s = c.slots[ b ];
			for( int32_t i = segStart[ b ]; i < segStart[ b + 1 ]; i++ )
			{
				int64_t first = 0, count = 0;
				const int pre = speakerSpan( segs[ i ].t0, segs[ i ].t1, s.stereoFrames, first, count );
				jobs[ (size_t)i ] = kern::SpeakerJob{ pre == kSpeakerSums ? s.stereo + 2 * first : nullptr, count, pre, 0 };
			}
		}
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		const size_t outOffset = ( n * sizeof( kern::SpeakerJob ) + 15 ) & ~(size_t)15;
		if( n > c.speakerCap )
		{
			if( c.speakerBuf ) { WSP_CUDA( cudaStreamSynchronize( c.stream ) ); cudaFree( c.speakerBuf ); c.speakerBuf = nullptr; }
			c.devBytes -= (uint64_t)c.speakerCap * ( sizeof( kern::SpeakerJob ) + 4 );
			c.speakerCap = 0;
			WSP_CHECK( devAlloc( c.speakerBuf, outOffset + n * 4 ) );
			c.devBytes += (uint64_t)n * ( sizeof( kern::SpeakerJob ) + 4 );
			c.speakerCap = n;
		}
		kern::SpeakerJob* dJobs = reinterpret_cast<kern::SpeakerJob*>( c.speakerBuf );
		int32_t* dOut = reinterpret_cast<int32_t*>( c.speakerBuf + outOffset );
		WSP_CUDA( cudaMemcpyAsync( dJobs, jobs.data(), n * sizeof( kern::SpeakerJob ), cudaMemcpyHostToDevice, c.stream ) );
		WSP_CUDA( kern::chunkSpeakers( dJobs, dOut, (int)n, c.stream ) );
		launched();
		WSP_CUDA( cudaMemcpyAsync( speakers, dOut, n * 4, cudaMemcpyDeviceToHost, c.stream ) );
		WSP_CUDA( cudaStreamSynchronize( c.stream ) );
		return WSP_OK;
	}

	// Instrumented decoder pass: nSteps single-token steps launched kernel by kernel with a CUDA event pair around every launch
	// (on the launching stream).  Continues from the context's current decoder state; used by bench.py for the roofline figure.
	int ctxProfileDecode( Context& c, int batch, int nSteps, float* msByKind, int* launchesByKind )
	{
		if( batch < 1 || batch > c.maxB || nSteps < 1 ) return fail( WSP_E_INVALIDARG, "batch / steps" );
		if( c.nPastHost + nSteps > c.e->hp.n_text_ctx ) return fail( WSP_E_BOUNDS, "n_past + n_steps exceeds n_text_ctx" );
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		c.prof.on = true;
		c.prof.used = 0;
		c.prof.kinds.clear();
		int rc = WSP_OK;
		for( int i = 0; i < nSteps && rc >= 0; i++ ) { rc = decodeSubmit( c, 1, batch, false, true ); if( rc >= 0 ) c.nPastHost++; }
		c.prof.on = false;
		if( rc < 0 ) return rc;
		WSP_CUDA( cudaStreamSynchronize( c.stream ) );
		for( int k = 0; k < KK_COUNT; k++ ) { msByKind[ k ] = 0; launchesByKind[ k ] = 0; }
		for( size_t i = 0; i < c.prof.kinds.size(); i++ )
		{
			float ms = 0;
			cudaEventElapsedTime( &ms, c.prof.pool[ 2 * i ], c.prof.pool[ 2 * i + 1 ] );
			msByKind[ c.prof.kinds[ i ] ] += ms;
			launchesByKind[ c.prof.kinds[ i ] ]++;
		}
		return WSP_OK;
	}

	// ===============================================================================================================
	// the measured path: mel + encode + n_decode greedy steps, tokens fed back on the device
	// ===============================================================================================================
	// whisper_lang_auto_detect for every chunk of the batch from its own encode (whisper.cpp:2428-2495): one N = 1 decoder pass over
	// [sot] at n_past 0 without sampling (the default step kernel; it writes self-KV row 0, which the prompt pass then rewrites), the
	// vocabulary softmax of the all-logits path, and langPick, which records each chunk's language and writes its prompt to tokensDev.
	// c.tokensDev[b] = sot and n_past = 0 are the caller's.
	static int enqueueLanguageDetection( Context& c, int batch, const int32_t* prompt, int nPrompt, int autoPos )
	{
		const Engine& e = *c.e;
		int n = 0;
		{
			// the step-timing marks (wsp_debug_step_timing) stay those of the sampled steps: this pass records none
			struct NoTiming { Context& c; bool was; NoTiming( Context& x ) : c( x ), was( x.stepTiming ) { c.stepTiming = false; } ~NoTiming() { c.stepTiming = was; } } nt( c );
			WSP_CHECK( decodeEnqueue( c, 1, batch, false, false, &n ) );
		}
		WSP_CUDA( kern::softmaxRows( c.logits, c.probs, batch, e.hp.n_vocab, c.stream ) );
		kern::LangPickArgs la{};
		la.probs = c.probs; la.nVocab = e.hp.n_vocab; la.tokLang0 = e.tokSot + 1; la.nLangs = e.nLangs;
		la.langIds = c.langIds; la.langProbs = c.langProbs; la.tokens = c.tokensDev; la.nPrompt = nPrompt; la.autoPos = autoPos;
		for( int i = 0; i < nPrompt; i++ ) la.tmpl[ i ] = prompt[ i ];
		WSP_CUDA( kern::langPick( la, batch, c.stream ) );
		launched( n + 2 );
		return WSP_OK;
	}
	static_assert( kMaxDecodeTokens <= kern::kLangPromptMax, "a prompt template must fit LangPickArgs" );

	// steps per block of wsp_run_chunks_until_eot: the host checks block k - 1's end-of-text count while block k runs
	constexpr int kEotLag = 8;

	int ctxRunChunks( Context& c, const float* const* pcm, const int32_t* nSamples, int batch, const int32_t* prompt, int nPrompt, int nDecode,
		int32_t* tokensOut, int32_t* nOut, float* stageMs, bool resident, const WindowOut* window, const WindowRow* rows )
	{
		const HParams& hp = c.e->hp;
		if( batch < 1 || batch > c.maxB ) return fail( WSP_E_BOUNDS, "batch exceeds the context's max_batch" );
		auto slotOf = [ & ]( int b ) { return rows ? rows[ b ].slot : b; };
		if( !prompt || nPrompt < 1 || nPrompt > kMaxDecodeTokens ) return fail( WSP_E_INVALIDARG, "prompt" );
		// every id indexes the embedding table, as ctxDecode's tokens do; at most one is the language sentinel
		int autoPos = -1;
		for( int i = 0; i < nPrompt; i++ )
		{
			if( prompt[ i ] == WSP_TOKEN_LANGUAGE_AUTO )
			{
				if( autoPos >= 0 ) return fail( WSP_E_INVALIDARG, "the prompt holds WSP_TOKEN_LANGUAGE_AUTO more than once" );
				autoPos = i;
			}
			else if( prompt[ i ] < 0 || prompt[ i ] >= hp.n_vocab ) return fail( WSP_E_INVALIDARG, "prompt token id out of range" );
		}
		const bool detect = autoPos >= 0;
		if( detect && c.e->nLangs < 1 ) return fail( WSP_E_INVALIDARG, "WSP_TOKEN_LANGUAGE_AUTO needs a multilingual model" );
		if( nDecode < 1 || nPrompt + nDecode > hp.n_text_ctx || nDecode > c.histCap ) return fail( WSP_E_BOUNDS, "n_prompt + n_decode exceeds n_text_ctx" );
		if( !resident && ( !pcm || !nSamples ) ) return fail( WSP_E_POINTER, "pcm" );
		for( int b = 0; b < batch; b++ )
		{
			if( !resident && nSamples[ b ] < 0 ) return fail( WSP_E_INVALIDARG, "n_samples" );
			if( resident && !c.slots[ slotOf( b ) ].pcm )
				return fail( WSP_E_INVALIDARG, "no resident PCM in slot " + std::to_string( slotOf( b ) ) + " (call wsp_upload_pcm)" );
			// whisper_lang_auto_detect( offset_ms ) refuses an offset at or past the end of the mel (whisper.cpp:2440-2443)
			if( rows && detect && rows[ b ].seek >= melFrames( c, c.slots[ rows[ b ].slot ].pcmSamples ) )
				return fail( WSP_E_INVALIDARG, "WSP_TOKEN_LANGUAGE_AUTO with a span offset at or past the end of its source" );
		}
		const bool untilEot = nOut != nullptr;
		if( window && window->cap < nDecode ) return fail( WSP_E_BOUNDS, "cap is below n_max" );
		// each window runs from its seek to its seek_end (whisper.cpp:2810-2818): seek 0 and the chunk's mel length, or a row's span; one
		// of at most 100 frames runs none (:2816, 2871).  The window rule reads the two only as seek_end - seek.
		std::vector<int32_t> toEnd( window ? (size_t)batch : 0 );
		for( size_t b = 0; b < toEnd.size(); b++ )
			toEnd[ b ] = rows ? rows[ b ].seekEnd - rows[ b ].seek : melFrames( c, resident ? c.slots[ b ].pcmSamples : nSamples[ b ] );
		// the slots whose log-mel (and energy) the call computes: each chunk's own, or each source slot of the rows once
		std::vector<int> srcs;
		if( rows )
		{
			std::vector<char> named( (size_t)c.maxB, 0 );
			for( int b = 0; b < batch; b++ )
				if( !named[ (size_t)rows[ b ].slot ] ) { named[ (size_t)rows[ b ].slot ] = 1; srcs.push_back( rows[ b ].slot ); }
		}
		else
			for( int b = 0; b < batch; b++ ) srcs.push_back( b );
		const int nSrc = (int)srcs.size();
		auto srcSlot = [ & ]( int i ) { return srcs[ (size_t)i ]; };
		c.lastLangIds.clear();
		c.lastLangProbs.clear();
		WSP_CUDA( cudaSetDevice( c.e->device ) );
		// a window call with token timestamps on computes every source's signal energy right after the log-mel
		const bool energy = window && c.tokenTimestamps;
		if( window ) c.windowEnergyBatch = 0;
		std::vector<int> energyLen( energy ? (size_t)batch : 0 );   // of each chunk's source
		if( energy )
		{
			size_t most = 1;
			for( int b = 0; b < batch; b++ )
			{
				energyLen[ (size_t)b ] = resident ? c.slots[ slotOf( b ) ].pcmSamples : nSamples[ b ];
				most = std::max( most, (size_t)energyLen[ (size_t)b ] );
			}
			WSP_CHECK( ensureEnergy( c, most, true ) );
		}
		cudaStream_t s = c.stream;
		WSP_CUDA( cudaEventRecord( c.ev[ 0 ], s ) );
		if( resident )
		{
			// inputs already in HBM (wsp_upload_pcm): the log-mel front end still runs inside the timed region
			auto pcmOf = [ & ]( int i ) { return (const float*)c.slots[ srcSlot( i ) ].pcm; };
			auto samplesOf = [ & ]( int i ) { return c.slots[ srcSlot( i ) ].pcmSamples; };
			WSP_CHECK( melBatchFromDevicePcm( c, nSrc, srcSlot, pcmOf, samplesOf ) );
			if( energy ) WSP_CHECK( energyFromDevicePcm( c, nSrc, srcSlot, pcmOf, samplesOf ) );
		}
		else
		{
			size_t total = 0;
			for( int b = 0; b < batch; b++ ) total += (size_t)nSamples[ b ];
			WSP_CHECK( ensurePcm( c, total ? total : 1 ) );
			std::vector<size_t> offs( (size_t)batch );
			size_t off = 0;
			for( int b = 0; b < batch; b++ )
			{
				if( nSamples[ b ] > 0 )
					WSP_CUDA( cudaMemcpyAsync( c.pcmDev + off, pcm[ b ], (size_t)nSamples[ b ] * 4, cudaMemcpyHostToDevice, s ) );
				offs[ (size_t)b ] = off;
				off += (size_t)nSamples[ b ];
			}
			auto pcmOf = [ & ]( int b ) { return (const float*)( c.pcmDev + offs[ (size_t)b ] ); };
			auto samplesOf = [ & ]( int b ) { return (int)nSamples[ b ]; };
			WSP_CHECK( melBatchFromDevicePcm( c, batch, srcSlot, pcmOf, samplesOf ) );
			if( energy ) WSP_CHECK( energyFromDevicePcm( c, batch, srcSlot, pcmOf, samplesOf ) );
		}
		WSP_CUDA( cudaEventRecord( c.ev[ 1 ], s ) );
		std::vector<int32_t> rowSlot( rows ? (size_t)batch : 0 ), rowSeek( rows ? (size_t)batch : 0 );
		for( size_t b = 0; b < rowSlot.size(); b++ ) { rowSlot[ b ] = rows[ b ].slot; rowSeek[ b ] = rows[ b ].seek; }
		WSP_CHECK( encodeAsync( c, rows ? rowSlot.data() : nullptr, rows ? rowSeek.data() : nullptr, batch ) );
		WSP_CUDA( cudaEventRecord( c.ev[ 2 ], s ) );
		// prompt step: same prompt for every chunk, first sample uses the initial-timestamp rules (whisper.cpp:2943); with the
		// language sentinel the tokens uploaded are the detection pass's [sot] per chunk, and langPick writes the prompts
		std::vector<int32_t> ptoks( detect ? (size_t)batch : (size_t)batch * nPrompt, c.e->tokSot );
		if( !detect )
			for( int b = 0; b < batch; b++ ) for( int i = 0; i < nPrompt; i++ ) ptoks[ (size_t)b * nPrompt + i ] = prompt[ i ];
		WSP_CUDA( cudaMemcpyAsync( c.tokensDev, ptoks.data(), ptoks.size() * 4, cudaMemcpyHostToDevice, s ) );
		WSP_CUDA( kern::setInts( c.dNPast, 0, 0, s ) );
		WSP_CUDA( kern::setInts( c.dFlags, 1, 1, s ) );
		WSP_CUDA( kern::setInts( c.dStep, 0, 0, s ) );
		launched( 3 );
		if( detect ) WSP_CHECK( enqueueLanguageDetection( c, batch, prompt, nPrompt, autoPos ) );
		int steps = nDecode;
		if( !untilEot && !window )
		{
			WSP_CHECK( decodeSubmit( c, nPrompt, batch, false, true ) );
			for( int i = 1; i < nDecode; i++ )
				WSP_CHECK( decodeSubmit( c, 1, batch, false, true ) );
		}
		else
		{
			// the sampler logs the step at which every chunk ends (its first EOT, or the window rule's end); the steps go out in blocks of
			// kEotLag, and block k is enqueued before the host waits for block k - 1 and reads how many chunks have ended, so the stream
			// never runs dry between blocks
			struct Arm { Context& c; Arm( Context& x ) : c( x ) { c.eotArmed = true; } ~Arm() { c.eotArmed = false; } } arm( c );
			*(volatile int*)c.nEndedHost = 0;
			if( !window )
			{
				WSP_CUDA( cudaMemsetAsync( c.endStep, 0, (size_t)batch * 4, s ) );
				WSP_CUDA( cudaMemsetAsync( c.nEnded, 0, 4, s ) );
				WSP_CUDA( cudaMemsetAsync( c.winCtl, 0, 4, s ) );
			}
			else
			{
				// a chunk too short for a window starts as ended (endStep -1) and counts as ended from the start
				std::vector<int32_t> ctl( 4 + (size_t)batch ), ends( (size_t)batch, 0 );
				std::vector<wsp::WindowState> st( (size_t)batch, wsp::windowStart() );
				ctl[ 0 ] = 1; ctl[ 1 ] = window->params.max_tokens; ctl[ 2 ] = window->params.single_segment != 0; ctl[ 3 ] = nDecode;
				int preEnded = 0;
				for( int b = 0; b < batch; b++ )
				{
					ctl[ 4 + (size_t)b ] = toEnd[ (size_t)b ];
					if( toEnd[ (size_t)b ] > 100 ) continue;
					st[ (size_t)b ] = wsp::WindowState{ 0, 0, 0, 0, 1 };
					ends[ (size_t)b ] = -1;
					preEnded++;
				}
				WSP_CUDA( cudaMemcpyAsync( c.winCtl, ctl.data(), ctl.size() * 4, cudaMemcpyHostToDevice, s ) );
				WSP_CUDA( cudaMemcpyAsync( c.winState, st.data(), st.size() * sizeof( wsp::WindowState ), cudaMemcpyHostToDevice, s ) );
				WSP_CUDA( cudaMemcpyAsync( c.endStep, ends.data(), ends.size() * 4, cudaMemcpyHostToDevice, s ) );
				WSP_CUDA( cudaMemcpyAsync( c.nEnded, &preEnded, 4, cudaMemcpyHostToDevice, s ) );
			}
			WSP_CHECK( decodeSubmit( c, nPrompt, batch, false, true ) );
			steps = 1;
			int waitOn = 0;
			WSP_CUDA( cudaEventRecord( c.blockEv[ waitOn ], s ) );
			while( steps < nDecode )
			{
				const int n = nDecode - steps < kEotLag ? nDecode - steps : kEotLag;
				for( int i = 0; i < n; i++ ) WSP_CHECK( decodeSubmit( c, 1, batch, false, true ) );
				steps += n;
				WSP_CUDA( cudaEventRecord( c.blockEv[ waitOn ^ 1 ], s ) );
				WSP_CUDA( cudaEventSynchronize( c.blockEv[ waitOn ] ) );
				waitOn ^= 1;
				if( *(volatile int*)c.nEndedHost >= batch ) break;
			}
		}
		c.nPastHost = nPrompt + steps - 1;
		WSP_CUDA( cudaEventRecord( c.ev[ 3 ], s ) );
		c.lastLogitRows = batch;
		// one D2H of the token log (and of the end-of-text steps) at the end: [batch][n_decode] int32
		std::vector<int32_t> hist( (size_t)batch * c.histCap ), ends( (size_t)batch );
		WSP_CUDA( cudaMemcpyAsync( hist.data(), c.history, hist.size() * 4, cudaMemcpyDeviceToHost, s ) );
		if( untilEot || window ) WSP_CUDA( cudaMemcpyAsync( ends.data(), c.endStep, ends.size() * 4, cudaMemcpyDeviceToHost, s ) );
		std::vector<wsp::WindowState> winSt( window ? (size_t)batch : 0 );
		std::vector<kern::TokenData> tdLog( window ? (size_t)batch * c.histCap : 0 );
		if( window )
		{
			WSP_CUDA( cudaMemcpyAsync( winSt.data(), c.winState, winSt.size() * sizeof( wsp::WindowState ), cudaMemcpyDeviceToHost, s ) );
			WSP_CUDA( cudaMemcpyAsync( tdLog.data(), c.tokenLog, tdLog.size() * sizeof( kern::TokenData ), cudaMemcpyDeviceToHost, s ) );
		}
		if( energy )
			for( const int slot : srcs )
				if( c.energyLen[ (size_t)slot ] > 0 )
					WSP_CUDA( cudaMemcpyAsync( c.energyHost + (size_t)slot * c.energyCap, c.energy + (size_t)slot * c.energyCap,
						(size_t)c.energyLen[ (size_t)slot ] * 4, cudaMemcpyDeviceToHost, s ) );
		std::vector<int32_t> langIds( detect ? (size_t)batch : 0 );
		std::vector<float> langProbs( detect ? (size_t)batch * c.e->nLangs : 0 );
		if( detect )
		{
			WSP_CUDA( cudaMemcpyAsync( langIds.data(), c.langIds, langIds.size() * 4, cudaMemcpyDeviceToHost, s ) );
			WSP_CUDA( cudaMemcpyAsync( langProbs.data(), c.langProbs, langProbs.size() * 4, cudaMemcpyDeviceToHost, s ) );
		}
		WSP_CUDA( cudaStreamSynchronize( s ) );
		c.lastLangIds.swap( langIds );
		c.lastLangProbs.swap( langProbs );
		if( energy )
		{
			c.windowEnergyBatch = batch;
			c.windowEnergyLen.swap( energyLen );
			c.windowRows.resize( (size_t)batch );
			for( int b = 0; b < batch; b++ ) c.windowRows[ (size_t)b ] = rows ? rows[ b ] : WindowRow{ b, 0, toEnd[ (size_t)b ] };
		}
		if( window )
			for( int b = 0; b < batch; b++ )
			{
				const wsp::WindowState& st = winSt[ (size_t)b ];
				const int n = ends[ (size_t)b ] > 0 ? ends[ (size_t)b ] : 0;
				window->results[ b ] = wsp_window_result{ n, st.resultLen, st.seekDelta, st.failed };
				if( window->tokens )
					for( int i = 0; i < n; i++ )
					{
						const kern::TokenData& t = tdLog[ (size_t)b * c.histCap + i ];
						window->tokens[ (size_t)b * window->cap + i ] = wsp_token_data{ t.id, t.tid, t.p, t.pt, t.ptsum };
					}
			}
		for( int b = 0; b < batch; b++ )
		{
			const int n = untilEot && ends[ (size_t)b ] > 0 ? ends[ (size_t)b ] : nDecode;
			if( nOut ) nOut[ b ] = n;
			if( tokensOut )
				for( int i = 0; i < n; i++ ) tokensOut[ (size_t)b * nDecode + i ] = hist[ (size_t)b * c.histCap + i ];
		}
		const float m0 = addStage( c, 0, c.ev[ 0 ], c.ev[ 1 ], 1 );
		const float m1 = addStage( c, 1, c.ev[ 1 ], c.ev[ 2 ], 1 );
		const float m2 = addStage( c, 2, c.ev[ 2 ], c.ev[ 3 ], steps );
		if( stageMs ) { stageMs[ 0 ] = m0; stageMs[ 1 ] = m1; stageMs[ 2 ] = m2; }
		return WSP_OK;
	}

	// whisper_full( clip of spans[b].slot, offset_ms, duration_ms )'s window bounds (whisper.cpp:2810-2811) for every row, then the
	// window call over them.  The seek arithmetic cannot overflow: offset_ms / 10, |duration_ms| / 10 and n_len = n_samples / 160 are
	// each below 2^31 / 10, so seek_end stays within int32.
	int ctxRunSpans( Context& c, const wsp_window_span* spans, int batch, const int32_t* prompt, int nPrompt, int nDecode, float* stageMs,
		const WindowOut& window )
	{
		if( batch < 1 || batch > c.maxB ) return fail( WSP_E_BOUNDS, "batch exceeds the context's max_batch" );
		std::vector<WindowRow> rows( (size_t)batch );
		for( int b = 0; b < batch; b++ )
		{
			const wsp_window_span& sp = spans[ b ];
			if( sp.slot < 0 || sp.slot >= c.maxB ) return fail( WSP_E_BOUNDS, "span slot outside max_batch" );
			if( !c.slots[ sp.slot ].pcm ) return fail( WSP_E_INVALIDARG, "no resident PCM in slot " + std::to_string( sp.slot ) + " (call wsp_upload_pcm)" );
			if( sp.offset_ms < 0 ) return fail( WSP_E_INVALIDARG, "negative offset_ms" );
			const int nLen = melFrames( c, c.slots[ sp.slot ].pcmSamples );
			const int seek = sp.offset_ms / 10;
			rows[ (size_t)b ] = WindowRow{ sp.slot, seek, seek + ( sp.duration_ms == 0 ? nLen : sp.duration_ms / 10 ) };
		}
		return ctxRunChunks( c, nullptr, nullptr, batch, prompt, nPrompt, nDecode, nullptr, nullptr, stageMs, true, &window, rows.data() );
	}
}

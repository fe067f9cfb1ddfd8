// TEST INFRASTRUCTURE — flat C helpers for tests/test_gpu_audio_ctx.py: iContext::runFull, runStreamed and runCapture with
// sFullParams::audio_ctx set, through the COM-style surface (include/whisper_b200_com.h) and nothing else, the way a client application
// calls it.  Built into tests/audio_ctx_shim/_build/libwsac_test.so and linked against libwhisper_b200.so.
#include "whisper_b200_com.h"
#include <atomic>
#include <chrono>
#include <string.h>
#include <string>
#include <thread>
#include <vector>
using namespace Whisper;

namespace
{
	struct Segment
	{
		int64_t t0, t1;   // 100 ns ticks
		std::vector<int> tokens;
	};
	struct Session
	{
		iModel* model = nullptr;
		iContext* context = nullptr;
		std::vector<Segment> segs;   // of the last run: getResults after runFull / runStreamed, new_segment_callback during runCapture
	};

	void append( Session* s, iTranscribeResult* res, uint32_t first )
	{
		sTranscribeLength len;
		res->getSize( len );
		for( uint32_t i = first; i < len.countSegments; i++ )
		{
			const sSegment& seg = res->getSegments()[ i ];
			Segment c{ (int64_t)seg.time.begin.ticks, (int64_t)seg.time.end.ticks, {} };
			for( uint32_t j = 0; j < seg.countTokens; j++ ) c.tokens.push_back( res->getTokens()[ seg.firstToken + j ].id );
			s->segs.push_back( std::move( c ) );
		}
	}
	HRESULT captureSegCallback( iContext* ctx, uint32_t nNew, void* pv ) noexcept
	{
		iTranscribeResult* res = nullptr;
		if( FAILED( ctx->getResults( (eResultFlags)( (uint32_t)eResultFlags::Tokens | (uint32_t)eResultFlags::Timestamps ), &res ) ) ) return E_FAIL;
		sTranscribeLength len;
		res->getSize( len );
		append( static_cast<Session*>( pv ), res, len.countSegments - nNew );
		res->Release();
		return S_OK;
	}
	// a live source played from an array in ragged blocks that never runs ahead of a transcription in flight (deterministic cuts)
	struct LiveSource
	{
		const float* pcm; uint32_t n, pos = 0, lcg = 4242u;
		std::atomic<uint8_t> status{ 0 };
		LiveSource( const float* p, uint32_t count ) : pcm( p ), n( count ) {}
		HRESULT read( float* mono, uint32_t capacity, uint32_t* written )
		{
			for( int waited = 0; ( status.load() & (uint8_t)eCaptureStatus::Transcribing ) && waited < 300000; waited++ )   // at most ~30 s
				std::this_thread::sleep_for( std::chrono::microseconds( 100 ) );
			lcg = lcg * 1664525u + 1013904223u;
			uint32_t want = 100 + ( lcg >> 8 ) % 900;
			if( want > capacity ) want = capacity;
			if( want > n - pos ) want = n - pos;
			if( want ) memcpy( mono, pcm + pos, (size_t)want * 4 );
			pos += want;
			*written = want;
			return S_OK;
		}
		bool finished() const { return pos >= n && !( status.load() & (uint8_t)eCaptureStatus::Transcribing ); }
	};
	// a file-like source for runStreamed: ragged blocks of 1..maxBlock samples
	struct BlockSource { const float* pcm; uint32_t n, pos, maxBlock, lcg; };

	HRESULT makeParams( Session* s, uint32_t flags, const char* language, int32_t maxTokens, int32_t cpuThreads, int32_t audioCtx, sFullParams& p )
	{
		const HRESULT hr = s->context->fullDefaultParams( eSamplingStrategy::Greedy, &p );
		if( FAILED( hr ) ) return hr;
		p.flags = (eFullParamsFlags)flags;
		p.language = ( language && strcmp( language, "auto" ) != 0 ) ? findLanguageKeyA( language ) : makeLanguageKey( "auto" );
		p.max_tokens = maxTokens;
		p.cpuThreads = cpuThreads;
		p.audio_ctx = audioCtx;
		return S_OK;
	}
}

extern "C" {

int32_t wsac_open( const char* modelPathUtf8, int32_t device, void** out )
{
	if( !modelPathUtf8 || !out ) return E_POINTER;
	std::wstring w;
	for( const char* p = modelPathUtf8; *p; p++ ) w.push_back( (wchar_t)(unsigned char)*p );   // test paths are ASCII
	std::wstring adapter = std::to_wstring( device );
	sModelSetup setup;
	setup.impl = eModelImplementation::B200;
	setup.adapter = adapter.c_str();
	Session* s = new Session();
	HRESULT hr = loadModel( w.c_str(), setup, nullptr, &s->model );
	if( SUCCEEDED( hr ) ) hr = s->model->createContext( &s->context );
	if( FAILED( hr ) )
	{
		if( s->model ) s->model->Release();
		delete s;
		return hr;
	}
	*out = s;
	return S_OK;
}
void wsac_close( void* h )
{
	Session* s = static_cast<Session*>( h );
	if( !s ) return;
	if( s->context ) s->context->Release();
	if( s->model ) s->model->Release();
	delete s;
}

// streamed = 0: runFull over an iAudioBuffer; 1: runStreamed over an iAudioReader handing out ragged blocks of 1..maxBlock samples
int32_t wsac_run( void* h, int32_t streamed, const float* pcm, int32_t nSamples, uint32_t flags, const char* language, int32_t maxTokens,
	int32_t cpuThreads, int32_t offsetMs, int32_t durationMs, int32_t audioCtx, int32_t maxBlock )
{
	Session* s = static_cast<Session*>( h );
	if( !s ) return E_POINTER;
	sFullParams p;
	HRESULT hr = makeParams( s, flags, language, maxTokens, cpuThreads, audioCtx, p );
	if( FAILED( hr ) ) return hr;
	p.offset_ms = offsetMs;
	p.duration_ms = durationMs;
	s->segs.clear();
	if( streamed )
	{
		BlockSource src{ pcm, (uint32_t)nSamples, 0, (uint32_t)( maxBlock > 0 ? maxBlock : 1 ), 12345u };
		auto readFn = []( float* mono, uint32_t capacity, uint32_t* written, void* pv ) noexcept -> HRESULT {
			BlockSource* k = static_cast<BlockSource*>( pv );
			k->lcg = k->lcg * 1664525u + 1013904223u;
			uint32_t want = 1 + ( k->lcg >> 8 ) % k->maxBlock;
			if( want > capacity ) want = capacity;
			if( want > k->n - k->pos ) want = k->n - k->pos;
			if( want ) memcpy( mono, k->pcm + k->pos, (size_t)want * 4 );
			k->pos += want;
			*written = want;
			return S_OK;
		};
		iAudioReader* reader = nullptr;
		hr = createAudioReader( readFn, &src, (int64_t)( (uint32_t)nSamples / 160 ) * 100000, &reader );
		if( FAILED( hr ) ) return hr;
		hr = s->context->runStreamed( p, sProgressSink{ nullptr, nullptr }, reader );
		reader->Release();
	}
	else
	{
		iAudioBuffer* buf = nullptr;
		hr = createAudioBuffer( pcm, (uint32_t)nSamples, &buf );
		if( FAILED( hr ) ) return hr;
		hr = s->context->runFull( p, buf );
		buf->Release();
	}
	if( FAILED( hr ) ) return hr;
	iTranscribeResult* res = nullptr;
	const HRESULT hr2 = s->context->getResults( (eResultFlags)( (uint32_t)eResultFlags::Tokens | (uint32_t)eResultFlags::Timestamps ), &res );
	if( FAILED( hr2 ) ) return hr2;
	append( s, res, 0 );
	res->Release();
	return hr;
}

// runCapture over an iAudioCapture made with createAudioCapture; the segments are those new_segment_callback delivered.
// info[0] = segments collected, [1] = samples the source handed out
int32_t wsac_run_capture( void* h, const float* pcm, int32_t nSamples, uint32_t flags, const char* language, int32_t cpuThreads,
	float minDuration, float maxDuration, int32_t audioCtx, int32_t* info )
{
	Session* s = static_cast<Session*>( h );
	if( !s ) return E_POINTER;
	sFullParams p;
	HRESULT hr = makeParams( s, flags, language, 0, cpuThreads, audioCtx, p );
	if( FAILED( hr ) ) return hr;
	p.new_segment_callback = &captureSegCallback;
	p.new_segment_callback_user_data = s;
	s->segs.clear();
	LiveSource src( pcm, (uint32_t)nSamples );
	sCaptureParams cp;
	cp.minDuration = minDuration;
	cp.maxDuration = maxDuration;
	iAudioCapture* cap = nullptr;
	hr = createAudioCapture( []( float* m, uint32_t c, uint32_t* w, void* pv ) noexcept -> HRESULT { return static_cast<LiveSource*>( pv )->read( m, c, w ); }, &src, cp, &cap );
	if( FAILED( hr ) ) return hr;
	sCaptureCallbacks cb;
	cb.pv = &src;
	cb.shouldCancel = []( void* pv ) noexcept -> HRESULT { return static_cast<LiveSource*>( pv )->finished() ? S_FALSE : S_OK; };
	cb.captureStatus = []( void* pv, eCaptureStatus st ) noexcept -> HRESULT { static_cast<LiveSource*>( pv )->status.store( (uint8_t)st ); return S_OK; };
	hr = s->context->runCapture( p, cb, cap );
	cap->Release();
	if( info ) { info[ 0 ] = (int32_t)s->segs.size(); info[ 1 ] = (int32_t)src.pos; }
	return hr;
}

int32_t wsac_n_segments( void* h ) { return (int32_t) static_cast<Session*>( h )->segs.size(); }
int64_t wsac_segment_t0( void* h, int32_t i ) { return static_cast<Session*>( h )->segs[ i ].t0; }
int64_t wsac_segment_t1( void* h, int32_t i ) { return static_cast<Session*>( h )->segs[ i ].t1; }
int32_t wsac_segment_n_tokens( void* h, int32_t i ) { return (int32_t) static_cast<Session*>( h )->segs[ i ].tokens.size(); }
int32_t wsac_token( void* h, int32_t i, int32_t j ) { return static_cast<Session*>( h )->segs[ i ].tokens[ j ]; }

} // extern "C"

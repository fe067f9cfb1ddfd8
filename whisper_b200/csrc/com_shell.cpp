// COM-style shell over the C ABI: iModel / iContext / iTranscribeResult / iAudioBuffer, the exported factory functions, and the
// transcription driver.
//
// The shell mirrors the reference's own wrapper around its CPU back-end (Whisper/whisperCom.cpp:67-212: class Context implements
// iContext + iModel over whisper_context) and the driver follows the oracle's whisper_full() (Whisper/source/whisper.cpp:2765-3125)
// step for step — windowing by the last timestamp token, prompt carry-over, the retry / skip-one-second rule, segment splitting —
// with whisper_encode -> wsp_encode and whisper_decode + whisper_sample_* -> wsp_decode (sampling happens on the GPU).
// The D3D back-end's driver (Whisper/Whisper/ContextImpl.cpp:452-794) differs slightly (it always skips 1 s on failure); the oracle wins.
#include "../../include/whisper_b200.h"
#include "../../include/whisper_b200_com.h"
#include "pcm_streamer.h"
#include "capture_loop.h"
#include "speaker.h"
#include "wav_reader.h"
#include "token_times.h"
#include "window_rule.h"
#include <algorithm>
#include <atomic>
#include <chrono>
#include <functional>
#include <math.h>
#include <map>

#include <memory>
#include <mutex>
#include <regex>
#include <stdarg.h>
#include <stdio.h>
#include <string>
#include <vector>

namespace
{
	using namespace Whisper;

	// ---------------------------------------------------------------------------------------------------------------
	// logger (Whisper/API/loggerApi.h, Whisper/Utils/Logger.cpp)
	std::mutex g_logMutex;
	sLoggerSetup g_logger = { nullptr, nullptr, eLogLevel::Warning, eLoggerFlags::UseStandardError };

	void logMessage( eLogLevel lvl, const char* fmt, ... )
	{
		sLoggerSetup ls;
		{
			std::lock_guard<std::mutex> lk( g_logMutex );
			ls = g_logger;
		}
		if( (uint8_t)lvl > (uint8_t)ls.level ) return;
		char buf[ 1024 ];
		va_list ap;
		va_start( ap, fmt );
		vsnprintf( buf, sizeof( buf ), fmt, ap );
		va_end( ap );
		if( ls.sink ) ls.sink( ls.context, lvl, buf );
		if( !ls.sink || ( (uint8_t)ls.flags & (uint8_t)eLoggerFlags::UseStandardError ) ) fprintf( stderr, "%s\n", buf );
	}

	HRESULT hrFromStatus( wsp_status s )
	{
		switch( s )
		{
		case WSP_OK: return S_OK;
		case WSP_S_FALSE: return S_FALSE;
		case WSP_E_INVALIDARG: return E_INVALIDARG;
		case WSP_E_POINTER: return E_POINTER;
		case WSP_E_OUTOFMEMORY: return E_OUTOFMEMORY;
		case WSP_E_BOUNDS: return E_BOUNDS;
		case WSP_E_NOTIMPL: return E_NOTIMPL;
		default: return E_FAIL;
		}
	}
	HRESULT check( wsp_status s, const char* what )
	{
		if( s >= 0 ) return hrFromStatus( s );
		logMessage( eLogLevel::Error, "%s failed: %s", what, wsp_last_error() );
		return hrFromStatus( s );
	}
#define HR( expr )                              \
	do {                                        \
		const HRESULT _hr = ( expr );           \
		if( FAILED( _hr ) ) return _hr;         \
	} while( 0 )

	// ---------------------------------------------------------------------------------------------------------------
	// ref-counted object base (ComLightLib/server/ObjectRoot.hpp equivalent)
	template<class I>
	class Object : public I
	{
		std::atomic<uint32_t> refs{ 1 };

	protected:
		virtual ~Object() = default;
		virtual bool queryExtra( REFIID, void** ) { return false; }

	public:
		HRESULT WSPCALL QueryInterface( REFIID riid, void** pp ) override
		{
			if( !pp ) return E_POINTER;
			if( riid == I::iid() || riid == ComLight::IUnknown::iid() )
			{
				*pp = static_cast<I*>( this );
				AddRef();
				return S_OK;
			}
			if( queryExtra( riid, pp ) ) return S_OK;
			*pp = nullptr;
			return E_NOINTERFACE;
		}
		uint32_t WSPCALL AddRef() override { return ++refs; }
		uint32_t WSPCALL Release() override
		{
			const uint32_t r = --refs;
			if( r == 0 ) delete this;
			return r;
		}
	};

	// ---------------------------------------------------------------------------------------------------------------
	// languages (table order = token order after <|startoftranscript|>; codes/names as in OpenAI Whisper, cf. whisper.cpp:33-133)
	const char* const kLanguages =
		"en:english zh:chinese de:german es:spanish ru:russian ko:korean fr:french ja:japanese pt:portuguese tr:turkish pl:polish ca:catalan nl:dutch "
		"ar:arabic sv:swedish it:italian id:indonesian hi:hindi fi:finnish vi:vietnamese iw:hebrew uk:ukrainian el:greek ms:malay cs:czech ro:romanian "
		"da:danish hu:hungarian ta:tamil no:norwegian th:thai ur:urdu hr:croatian bg:bulgarian lt:lithuanian la:latin mi:maori ml:malayalam cy:welsh "
		"sk:slovak te:telugu fa:persian lv:latvian bn:bengali sr:serbian az:azerbaijani sl:slovenian kn:kannada et:estonian mk:macedonian br:breton "
		"eu:basque is:icelandic hy:armenian ne:nepali mn:mongolian bs:bosnian kk:kazakh sq:albanian sw:swahili gl:galician mr:marathi pa:punjabi "
		"si:sinhala km:khmer sn:shona yo:yoruba so:somali af:afrikaans oc:occitan ka:georgian be:belarusian tg:tajik sd:sindhi gu:gujarati am:amharic "
		"yi:yiddish lo:lao uz:uzbek fo:faroese ht:haitian_creole ps:pashto tk:turkmen nn:nynorsk mt:maltese sa:sanskrit lb:luxembourgish my:myanmar "
		"bo:tibetan tl:tagalog mg:malagasy as:assamese tt:tatar haw:hawaiian ln:lingala ha:hausa ba:bashkir jw:javanese su:sundanese";

	struct LanguageTable
	{
		std::vector<std::string> codes, names;
		std::vector<sLanguageEntry> entries;
		LanguageTable()
		{
			std::string all( kLanguages );
			size_t pos = 0;
			while( pos < all.size() )
			{
				size_t sp = all.find( ' ', pos );
				if( sp == std::string::npos ) sp = all.size();
				const std::string item = all.substr( pos, sp - pos );
				const size_t colon = item.find( ':' );
				codes.push_back( item.substr( 0, colon ) );
				std::string nm = item.substr( colon + 1 );
				for( char& c : nm ) if( c == '_' ) c = ' ';
				names.push_back( nm );
				pos = sp + 1;
			}
			for( size_t i = 0; i < codes.size(); i++ )
				entries.push_back( sLanguageEntry{ makeLanguageKey( codes[ i ].c_str() ), (int)i, names[ i ].c_str() } );
		}
		int idFromKey( uint32_t key ) const
		{
			for( const auto& e : entries ) if( e.key == key ) return e.id;
			return -1;
		}
	};
	const LanguageTable& languages()
	{
		static const LanguageTable t;
		return t;
	}

	std::string utf8FromWide( const wchar_t* w )
	{
		std::string out;
		if( !w ) return out;
		for( ; *w; w++ )
		{
			uint32_t c = (uint32_t)*w;
			if( sizeof( wchar_t ) == 2 && c >= 0xD800 && c <= 0xDBFF && w[ 1 ] )
			{
				c = 0x10000 + ( ( c - 0xD800 ) << 10 ) + ( (uint32_t)w[ 1 ] - 0xDC00 );
				w++;
			}
			if( c < 0x80 ) out.push_back( (char)c );
			else if( c < 0x800 ) { out.push_back( (char)( 0xC0 | ( c >> 6 ) ) ); out.push_back( (char)( 0x80 | ( c & 0x3F ) ) ); }
			else if( c < 0x10000 ) { out.push_back( (char)( 0xE0 | ( c >> 12 ) ) ); out.push_back( (char)( 0x80 | ( ( c >> 6 ) & 0x3F ) ) ); out.push_back( (char)( 0x80 | ( c & 0x3F ) ) ); }
			else { out.push_back( (char)( 0xF0 | ( c >> 18 ) ) ); out.push_back( (char)( 0x80 | ( ( c >> 12 ) & 0x3F ) ) ); out.push_back( (char)( 0x80 | ( ( c >> 6 ) & 0x3F ) ) ); out.push_back( (char)( 0x80 | ( c & 0x3F ) ) ); }
		}
		return out;
	}

	// ---------------------------------------------------------------------------------------------------------------
	struct SharedEngine
	{
		wsp_model* model = nullptr;
		wsp_engine* engine = nullptr;
		int32_t hp[ 11 ] = {};
		int32_t special[ 8 ] = {};
		~SharedEngine()
		{
			if( engine ) wsp_engine_destroy( engine );
			if( model ) wsp_model_close( model );
		}
		int nVocab() const { return hp[ 0 ]; }
		int nTextCtx() const { return hp[ 5 ]; }
		int tokEot() const { return special[ 0 ]; }
		int tokSot() const { return special[ 1 ]; }
		int tokPrev() const { return special[ 2 ]; }
		int tokBeg() const { return special[ 5 ]; }
	};

	class AudioBufferObj : public Object<iAudioBuffer>
	{
		std::vector<float> pcm, stereo;

	public:
		AudioBufferObj( const float* p, uint32_t n ) : pcm( p, p + n ) {}
		AudioBufferObj( const float* p, const float* interleaved, uint32_t n ) : pcm( p, p + n ), stereo( interleaved, interleaved + 2 * (size_t)n ) {}
		uint32_t WSPCALL countSamples() const override { return (uint32_t)pcm.size(); }
		const float* WSPCALL getPcmMono() const override { return pcm.data(); }
		const float* WSPCALL getPcmStereo() const override { return stereo.empty() ? nullptr : stereo.data(); }
		HRESULT WSPCALL getTime( int64_t& rdi ) const override { rdi = 0; return S_OK; }
	};

	// iAudioReader over a pull callback (createAudioReader): the Linux replacement of iMediaFoundation::openAudioFile
	class CallbackSourceReader : public Object<IMFSourceReader>
	{
		pfnReadPcm pfn;
		void* pv;

	public:
		CallbackSourceReader( pfnReadPcm f, void* p ) : pfn( f ), pv( p ) {}
		HRESULT WSPCALL readPcm( float* mono, uint32_t capacity, uint32_t* written ) override
		{
			if( !mono || !written ) return E_POINTER;
			*written = 0;
			return pfn( mono, capacity, written, pv );
		}
	};
	class AudioReaderObj : public Object<iAudioReader>
	{
		CallbackSourceReader* source;
		int64_t duration;
		~AudioReaderObj() override { source->Release(); }

	public:
		AudioReaderObj( pfnReadPcm f, void* p, int64_t ticks ) : source( new CallbackSourceReader( f, p ) ), duration( ticks ) {}
		HRESULT WSPCALL getDuration( int64_t& rdi ) const override { rdi = duration; return S_OK; }
		HRESULT WSPCALL getReader( IMFSourceReader** pp ) const override
		{
			if( !pp ) return E_POINTER;
			source->AddRef();
			*pp = source;
			return S_OK;
		}
		HRESULT WSPCALL requestedStereo() const override { return S_FALSE; }
	};

	class AudioCaptureObj : public Object<iAudioCapture>
	{
		CallbackSourceReader* source;
		sCaptureParams params;
		~AudioCaptureObj() override { source->Release(); }

	public:
		AudioCaptureObj( pfnReadPcm f, void* p, const sCaptureParams& cp ) : source( new CallbackSourceReader( f, p ) ), params( cp ) {}
		HRESULT WSPCALL getReader( IMFSourceReader** pp ) const override
		{
			if( !pp ) return E_POINTER;
			source->AddRef();
			*pp = source;
			return S_OK;
		}
		const sCaptureParams& WSPCALL getParams() const override { return params; }
	};

	// ---------------------------------------------------------------------------------------------------------------
	// iMediaFoundation for Linux: RIFF/WAVE in place of Media Foundation (csrc/wav_reader.h)
	class WavSourceReader : public Object<IMFSourceReader>
	{
		std::unique_ptr<wsp::WavDecoder> wav;

	public:
		explicit WavSourceReader( std::unique_ptr<wsp::WavDecoder> w ) : wav( std::move( w ) ) {}
		HRESULT WSPCALL readPcm( float* mono, uint32_t capacity, uint32_t* written ) override
		{
			if( !mono || !written ) return E_POINTER;
			*written = (uint32_t)wav->read( mono, nullptr, capacity );
			if( *written == 0 && !wav->error.empty() )
			{
				logMessage( eLogLevel::Error, "audio reader: %s", wav->error.c_str() );
				return E_FAIL;
			}
			return S_OK;
		}
	};
	class WavReaderObj : public Object<iAudioReader>
	{
		WavSourceReader* source;
		int64_t duration;
		bool stereo;
		~WavReaderObj() override { source->Release(); }

	public:
		WavReaderObj( std::unique_ptr<wsp::WavDecoder> w, bool wantStereo ) : duration( (int64_t)w->outputFrames() * 625 ), stereo( wantStereo && w->channels >= 2 )
		{
			source = new WavSourceReader( std::move( w ) );
		}
		HRESULT WSPCALL getDuration( int64_t& rdi ) const override { rdi = duration; return S_OK; }   // 16 kHz samples * 10^7 / 16000
		HRESULT WSPCALL getReader( IMFSourceReader** pp ) const override
		{
			if( !pp ) return E_POINTER;
			source->AddRef();
			*pp = source;
			return S_OK;
		}
		HRESULT WSPCALL requestedStereo() const override { return stereo ? S_OK : S_FALSE; }
	};
	class MediaFoundationObj : public Object<iMediaFoundation>
	{
		static HRESULT open( std::unique_ptr<wsp::WavDecoder>& w, bool ok, const char* what )
		{
			if( ok ) return S_OK;
			logMessage( eLogLevel::Error, "%s: %s", what, w->error.c_str() );
			return w->error.compare( 0, 11, "cannot open" ) == 0 ? WSP_HR( 0x80070002 ) : E_INVALIDARG;   // HRESULT_FROM_WIN32( ERROR_FILE_NOT_FOUND )
		}

	public:
		HRESULT WSPCALL loadAudioFile( LPCTSTR path, bool stereo, iAudioBuffer** pp ) const override
		{
			// Whisper/MF/loadAudioFile.cpp: decode the whole file into an AudioBuffer (mono, and the stereo pairs when asked for and present)
			if( !path || !pp ) return E_POINTER;
			*pp = nullptr;
			auto w = std::make_unique<wsp::WavDecoder>();
			HR( open( w, w->openFile( path ), path ) );
			const uint64_t n = w->outputFrames();
			if( n > 0xFFFFFFFFull ) return E_INVALIDARG;
			const bool keepStereo = stereo && w->channels >= 2;
			std::vector<float> mono( (size_t)n ), pairs( keepStereo ? 2 * (size_t)n : 0 );
			size_t done = 0;
			while( done < n )
			{
				const size_t got = w->read( mono.data() + done, keepStereo ? pairs.data() + 2 * done : nullptr, (size_t)n - done );
				if( got == 0 ) break;
				done += got;
			}
			if( done != n )
			{
				logMessage( eLogLevel::Error, "%s: %s", path, w->error.empty() ? "truncated audio data" : w->error.c_str() );
				return E_FAIL;
			}
			*pp = keepStereo ? new AudioBufferObj( mono.data(), pairs.data(), (uint32_t)n ) : new AudioBufferObj( mono.data(), (uint32_t)n );
			return S_OK;
		}
		HRESULT WSPCALL openAudioFile( LPCTSTR path, bool stereo, iAudioReader** pp ) override
		{
			if( !path || !pp ) return E_POINTER;
			*pp = nullptr;
			auto w = std::make_unique<wsp::WavDecoder>();
			HR( open( w, w->openFile( path ), path ) );
			*pp = new WavReaderObj( std::move( w ), stereo );
			return S_OK;
		}
		HRESULT WSPCALL loadAudioFileData( const void* data, uint64_t size, bool stereo, iAudioReader** pp ) override
		{
			if( !data || !pp ) return E_POINTER;
			*pp = nullptr;
			auto w = std::make_unique<wsp::WavDecoder>();
			HR( open( w, w->openMemory( data, size ), "loadAudioFileData" ) );
			*pp = new WavReaderObj( std::move( w ), stereo );
			return S_OK;
		}
		HRESULT WSPCALL listCaptureDevices( pfnFoundCaptureDevices pfn, void* pv ) override
		{
			if( !pfn ) return E_POINTER;
			return pfn( 0, nullptr, pv );   // no capture devices are enumerated on this platform
		}
		HRESULT WSPCALL openCaptureDevice( LPCTSTR, const sCaptureParams&, iAudioCapture** pp ) override
		{
			if( pp ) *pp = nullptr;
			logMessage( eLogLevel::Error, "whisper_b200: no capture devices on this platform; wrap the live source with createAudioCapture" );
			return E_NOTIMPL;
		}
	};

	struct ResultData
	{
		// whisper_token_data (whisper.h:71-85): t0 / t1 stay -1 unless token-level timestamps were requested
		struct Tok { wsp_token_data d; int64_t t0 = -1, t1 = -1; float vlen = 0.0f; };
		struct Seg { int64_t t0, t1; std::string text; std::vector<Tok> tokens; };
		std::vector<Seg> segs;
		int64_t timeOffset = 0;   // 100 ns ticks: iAudioBuffer::getTime of the clip (ContextImpl::mediaTimeOffset, ContextImpl.misc.cpp:264-286, 364)
	};

	class ResultObj : public Object<iTranscribeResult>
	{
	public:
		std::vector<std::string> texts;
		std::vector<sSegment> segments;
		std::vector<sToken> tokens;
		std::shared_ptr<SharedEngine> eng;   // token text pointers live in the model

		void build( const ResultData& rd, const std::shared_ptr<SharedEngine>& e, bool makeTokens )
		{
			// Whisper/source.compat/convertThings.cpp:160-213 (makeNewResults): 10 ms units -> 100 ns ticks, Special = id >= eot
			eng = e;
			texts.clear(); segments.clear(); tokens.clear();
			texts.reserve( rd.segs.size() );
			for( const auto& s : rd.segs ) texts.push_back( s.text );
			for( size_t i = 0; i < rd.segs.size(); i++ )
			{
				const auto& s = rd.segs[ i ];
				sSegment seg;
				seg.text = texts[ i ].c_str();
				seg.time.begin.ticks = (uint64_t)( s.t0 * 100000 + rd.timeOffset );
				seg.time.end.ticks = (uint64_t)( s.t1 * 100000 + rd.timeOffset );
				seg.firstToken = (uint32_t)tokens.size();
				seg.countTokens = 0;
				if( makeTokens )
				{
					seg.countTokens = (uint32_t)s.tokens.size();
					for( const auto& tok : s.tokens )
					{
						const wsp_token_data& t = tok.d;
						sToken tk;
						tk.text = wsp_model_token_text( e->model, t.id );
						tk.time.begin.ticks = (uint64_t)( tok.t0 * 100000 + rd.timeOffset );   // -1 (not computed) converts like the reference's MFllMulDiv( -1, ... )
						tk.time.end.ticks = (uint64_t)( tok.t1 * 100000 + rd.timeOffset );
						tk.probability = t.p; tk.probabilityTimestamp = t.pt; tk.ptsum = t.ptsum; tk.vlen = tok.vlen;
						tk.id = t.id;
						tk.flags = t.id >= e->tokEot() ? eTokenFlags::Special : eTokenFlags::None;
						tokens.push_back( tk );
					}
				}
				segments.push_back( seg );
			}
		}
		HRESULT WSPCALL getSize( sTranscribeLength& rdi ) const override
		{
			rdi.countSegments = (uint32_t)segments.size();
			rdi.countTokens = (uint32_t)tokens.size();
			return S_OK;
		}
		const sSegment* WSPCALL getSegments() const override { return segments.empty() ? nullptr : segments.data(); }
		const sToken* WSPCALL getTokens() const override { return tokens.empty() ? nullptr : tokens.data(); }
	};

	class ModelObj;

	class ContextObj : public Object<iContext>
	{
		ModelObj* owner;                       // holds a reference (ContextImpl.h:16)
		std::shared_ptr<SharedEngine> eng;
		wsp_context* ctx = nullptr;
		std::vector<int32_t> promptPast;       // text context carried across windows and calls (whisper_context::prompt_past)
		ResultData results;
		mutable ResultObj* staticResult = nullptr;
		// token-level timestamps (whisper_context::energy / t_beg / t_last / tid_last, whisper.cpp:425-431); the energy is the device's
		std::vector<float> energy;
		wsp::TokenTimeState tokenTimeState;
		int tokenTimesAndWrap( const sFullParams& params );
		// what detectSpeaker looks at: the stereo samples of the clip being transcribed (ContextImpl::currentSpectrogram, ContextImpl.cpp:441-450)
		bool insideRun = false;
		const float* curStereo = nullptr;
		uint64_t curStereoFrames = 0;
		// host-timed blocks of timingsPrint: [0] whole run calls (eCpuBlock::RunComplete), [1] client callbacks (eCpuBlock::Callbacks)
		double hostMs[ 2 ] = { 0.0, 0.0 };
		int64_t hostCalls[ 2 ] = { 0, 0 };
		struct HostTimer
		{
			double& ms; int64_t& calls;
			std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now();
			HostTimer( ContextObj& c, int i ) : ms( c.hostMs[ i ] ), calls( c.hostCalls[ i ] ) {}
			~HostTimer() { ms += std::chrono::duration<double, std::milli>( std::chrono::steady_clock::now() - t0 ).count(); calls++; }
		};

		~ContextObj() override;

		HRESULT decode( const std::vector<int32_t>& tokens, int nPast, bool first, wsp_token_data& out )
		{
			const uint32_t flags = first ? ( WSP_DECODE_FORCE_TIMESTAMP | WSP_DECODE_INITIAL ) : 0u;
			return check( wsp_decode( ctx, tokens.data(), (int32_t)tokens.size(), nPast, 1, flags, &out ), "wsp_decode" );
		}
		HRESULT detectLanguage( int& langId );
		// where the loop's mel comes from: `prepare( seek )` makes the window that starts at frame `seek` available in slot 0 and returns
		// the frame offset to encode at (the iSpectrogram of Whisper/Whisper/iSpectrogram.h:11-23, with makeBuffer + upload folded into one)
		struct MelSource
		{
			int nLen = 0;
			std::function<HRESULT( int seek, int32_t& encodeAt )> prepare;
		};
		HRESULT checkParams( const sFullParams& params );
		HRESULT runImpl( const sFullParams& params, const sProgressSink& progress, const MelSource& mel, bool tokenTimestamps );

	public:
		ContextObj( ModelObj* m, const std::shared_ptr<SharedEngine>& e );
		HRESULT init() { return check( wsp_context_create( eng->engine, 1, &ctx ), "wsp_context_create" ); }

		HRESULT WSPCALL runFull( const sFullParams& params, const iAudioBuffer* buffer ) override;
		HRESULT WSPCALL runStreamed( const sFullParams& params, const sProgressSink& progress, const iAudioReader* reader ) override;
		HRESULT WSPCALL runCapture( const sFullParams& params, const sCaptureCallbacks& callbacks, const iAudioCapture* reader ) override;
		HRESULT WSPCALL getResults( eResultFlags flags, iTranscribeResult** pp ) const override
		{
			if( !pp ) return E_POINTER;
			const bool makeTokens = 0 != ( (uint32_t)flags & (uint32_t)eResultFlags::Tokens );
			if( (uint32_t)flags & (uint32_t)eResultFlags::NewObject )
			{
				ResultObj* r = new ResultObj();
				r->build( results, eng, makeTokens );
				*pp = r;
				return S_OK;
			}
			// context-owned object whose content is replaced by the next call (TranscribeStructs.h:110-114)
			if( !staticResult ) staticResult = new ResultObj();
			staticResult->build( results, eng, makeTokens );
			staticResult->AddRef();
			*pp = staticResult;
			return S_OK;
		}
		HRESULT WSPCALL detectSpeaker( const sTimeInterval& time, eSpeakerChannel& result ) const override
		{
			// ContextImpl::detectSpeaker (Whisper/Whisper/ContextImpl.diarize.cpp:75-112): sum of |sample| per channel over the interval,
			// a channel wins when it is more than 1.1 x the other.  Only meaningful while a run is in progress, i.e. from the callbacks.
			result = eSpeakerChannel::Unsure;
			if( !insideRun )
			{
				logMessage( eLogLevel::Error, "iContext.detectSpeaker() method only works when called from the callbacks" );
				return WSP_HR( 0x80040007 );   // OLE_E_BLANK
			}
			const int64_t begin = ( ( (int64_t)time.begin.ticks - results.timeOffset ) * 100 ) / 10000000;   // 10 ms chunks, :9-13
			const int64_t end = ( ( (int64_t)time.end.ticks - results.timeOffset ) * 100 ) / 10000000;
			// the rule (csrc/speaker.h) is the one wsp_chunk_speakers runs on the device
			const int r = wsp::speakerOfSegment( curStereo, curStereo ? (int64_t)curStereoFrames : 0, begin, end );
			if( r == WSP_SPEAKER_OUT_OF_RANGE ) return E_BOUNDS;   // Spectrogram::copyStereoPcm, Spectrogram.cpp:142-168
			result = (eSpeakerChannel)(uint8_t)r;
			return S_OK;
		}
		HRESULT WSPCALL getModel( iModel** pp ) override;
		HRESULT WSPCALL fullDefaultParams( eSamplingStrategy strategy, sFullParams* rdi ) override
		{
			if( !rdi ) return E_POINTER;
			// whisper_full_default_params (whisper.cpp:2596-2710) through makeNewParams (convertThings.cpp:7-60)
			memset( rdi, 0, sizeof( *rdi ) );
			rdi->strategy = strategy;
			rdi->cpuThreads = 4;
			rdi->n_max_text_ctx = 16384;
			rdi->flags = (eFullParamsFlags)( (uint32_t)eFullParamsFlags::PrintProgress | (uint32_t)eFullParamsFlags::PrintTimestamps );
			rdi->language = makeLanguageKey( "en" );
			rdi->thold_pt = 0.01f;
			rdi->thold_ptsum = 0.01f;
			if( strategy == eSamplingStrategy::BeamSearch ) { rdi->greedy.n_past = -1; rdi->beam_search.beam_width = 10; rdi->beam_search.n_best = 5; }
			else { rdi->beam_search.n_past = -1; rdi->beam_search.beam_width = -1; rdi->beam_search.n_best = -1; }
			return S_OK;
		}
		HRESULT WSPCALL timingsPrint() override
		{
			// the per-block table of ContextImpl::timingsPrint (ContextImpl.misc.cpp:170-182, ProfileCollection::print): host-timed blocks,
			// device-timed blocks (CUDA events on the context's stream), then the memory table
			float ms[ 4 ]; int32_t calls[ 4 ];
			HR( check( wsp_timings( ctx, ms, calls, 0 ), "wsp_timings" ) );
			auto line = []( const char* name, double msTotal, int64_t count ) {
				if( count <= 0 ) return;
				auto scaled = []( double v, const char*& unit ) { if( v >= 1000.0 ) { unit = "seconds"; return v / 1000.0; } if( v >= 1.0 ) { unit = "milliseconds"; return v; } unit = "microseconds"; return v * 1000.0; };
				const char* u1; const char* u2;
				const double total = scaled( msTotal, u1 );
				if( count == 1 ) logMessage( eLogLevel::Info, "%s\t%g %s", name, total, u1 );
				else
				{
					const double avg = scaled( msTotal / (double)count, u2 );
					logMessage( eLogLevel::Info, "%s\t%g %s, %lld calls, %g %s average", name, total, u1, (long long)count, avg, u2 );
				}
			};
			logMessage( eLogLevel::Info, "    CPU Tasks" );
			line( "RunComplete", hostMs[ 0 ], hostCalls[ 0 ] );
			line( "Callbacks", hostMs[ 1 ], hostCalls[ 1 ] );
			logMessage( eLogLevel::Info, "    GPU Tasks" );
			line( "Spectrogram", ms[ 0 ], calls[ 0 ] );
			line( "Encode", ms[ 1 ], calls[ 1 ] );
			line( "Decode", ms[ 2 ], calls[ 2 ] );
			line( "Sample", ms[ 3 ], calls[ 3 ] );
			auto mem = []( const char* what, uint64_t vram ) {
				const char* unit = "bytes"; double v = (double)vram;
				if( vram >= ( 1ull << 30 ) ) { v /= (double)( 1ull << 30 ); unit = "GB"; }
				else if( vram >= ( 1ull << 20 ) ) { v /= (double)( 1ull << 20 ); unit = "MB"; }
				else if( vram >= ( 1ull << 10 ) ) { v /= 1024.0; unit = "KB"; }
				logMessage( eLogLevel::Info, "%s\t0 bytes RAM, %g %s VRAM", what, v, unit );
			};
			logMessage( eLogLevel::Info, "    Memory Usage" );
			const uint64_t mModel = wsp_engine_weight_bytes( eng->engine ), mCtx = wsp_context_device_bytes( ctx );
			mem( "Model", mModel );
			mem( "Context", mCtx );
			mem( "Total", mModel + mCtx );
			return S_OK;
		}
		HRESULT WSPCALL timingsReset() override
		{
			float ms[ 4 ]; int32_t calls[ 4 ];
			hostMs[ 0 ] = hostMs[ 1 ] = 0.0; hostCalls[ 0 ] = hostCalls[ 1 ] = 0;
			return check( wsp_timings( ctx, ms, calls, 1 ), "wsp_timings" );
		}
		// not part of the COM surface: used by the flat test helpers below
		const ResultData& data() const { return results; }
		void clearPromptPast() { promptPast.clear(); }
	};

	class ModelObj : public Object<iModel>
	{
		std::shared_ptr<SharedEngine> eng;
		~ModelObj() override = default;

	public:
		explicit ModelObj( const std::shared_ptr<SharedEngine>& e ) : eng( e ) {}
		HRESULT WSPCALL createContext( iContext** pp ) override
		{
			if( !pp ) return E_POINTER;
			ContextObj* c = new ContextObj( this, eng );
			const HRESULT hr = c->init();
			if( FAILED( hr ) ) { c->Release(); return hr; }
			*pp = c;
			return S_OK;
		}
		HRESULT WSPCALL tokenize( const char* text, pfnDecodedTokens pfn, void* pv ) override
		{
			// whisper.cpp:2192-2245: GPT-2 style pre-split, then greedy longest match against the vocabulary
			if( !text || !pfn ) return E_POINTER;
			std::vector<int> out;
			try
			{
				static const std::regex re( R"('s|'t|'re|'ve|'m|'ll|'d| ?[[:alpha:]]+| ?[[:digit:]]+| ?[^\s[:alpha:][:digit:]]+|\s+(?!\S)|\s+)" );
				std::string str( text );
				std::vector<std::string> words;
				for( std::sregex_iterator it( str.begin(), str.end(), re ), end; it != end; ++it ) words.push_back( it->str() );
				const int nv = eng->nVocab();
				// reverse map built on first use
				static std::mutex mtx;
				std::lock_guard<std::mutex> lk( mtx );
				if( vocabMap.empty() )
					for( int i = 0; i < nv; i++ )
					{
						const char* t = wsp_model_token_text( eng->model, i );
						if( t ) vocabMap[ t ] = i;   // later duplicates win, like std::map assignment in the loader (whisper.cpp:569)
					}
				for( const auto& word : words )
				{
					const int n = (int)word.size();
					int i = 0;
					while( i < n )
					{
						int j = n;
						while( j > i )
						{
							auto f = vocabMap.find( word.substr( i, j - i ) );
							if( f != vocabMap.end() ) { out.push_back( f->second ); i = j; break; }
							--j;
						}
						if( i == n ) break;
						if( j == i )
						{
							// Reached both when nothing matched and right after a match that did not end the word (i was just set to j):
							// the reference then emits the next character on its own (whisper.cpp:2232-2241).  Kept, quirk included.
							auto f1 = vocabMap.find( word.substr( i, 1 ) );
							if( f1 != vocabMap.end() ) out.push_back( f1->second );
							else logMessage( eLogLevel::Warning, "tokenize: unknown token '%c'", word[ i ] );
							++i;
						}
					}
				}
			}
			catch( const std::exception& ) { return E_FAIL; }
			if( !out.empty() ) pfn( out.data(), (int)out.size(), pv );
			return S_OK;
		}
		HRESULT WSPCALL isMultilingual() override { return wsp_model_is_multilingual( eng->model ) ? S_OK : S_FALSE; }
		HRESULT WSPCALL getSpecialTokens( SpecialTokens& rdi ) override
		{
			const int32_t* s = eng->special;
			rdi = SpecialTokens{ s[ 0 ], s[ 1 ], s[ 2 ], s[ 3 ], s[ 4 ], s[ 5 ], s[ 6 ], s[ 7 ] };
			return S_OK;
		}
		const char* WSPCALL stringFromToken( whisper_token token ) override { return wsp_model_token_text( eng->model, token ); }
		HRESULT WSPCALL clone( iModel** rdi ) override
		{
			// the reference needs a second D3D device sharing the weight buffers (ModelImpl.cpp:40-60); here the engine is immutable and
			// every context has its own stream and state, so a clone is simply another handle on the same weights
			if( !rdi ) return E_POINTER;
			*rdi = new ModelObj( eng );
			return S_OK;
		}

	private:
		std::map<std::string, int> vocabMap;
	};

	ContextObj::ContextObj( ModelObj* m, const std::shared_ptr<SharedEngine>& e ) : owner( m ), eng( e ) { owner->AddRef(); }
	ContextObj::~ContextObj()
	{
		if( staticResult ) staticResult->Release();
		if( ctx ) wsp_context_destroy( ctx );
		owner->Release();
	}
	HRESULT WSPCALL ContextObj::getModel( iModel** pp )
	{
		if( !pp ) return E_POINTER;
		owner->AddRef();
		*pp = owner;
		return S_OK;
	}

	// ---- token-level timestamps and segment wrapping (csrc/token_times.h) -------------------------------------------------------
	// whisper_exp_compute_token_level_timestamps (whisper.cpp:3374-3600) over the last segment, then, with max_len, whisper_wrap_segment
	// (:2713-2763) of it; returns the number of segments the last one became
	int ContextObj::tokenTimesAndWrap( const sFullParams& params )
	{
		ResultData::Seg& seg = results.segs.back();
		const int n = (int)seg.tokens.size();
		const int tokEot = eng->tokEot();
		std::vector<wsp_token_data> td( (size_t)n );
		std::vector<wsp_token_time> tt( (size_t)n );
		std::vector<float> vlen( (size_t)n );
		std::vector<int> textLen( (size_t)n );
		for( int j = 0; j < n; j++ )
		{
			const ResultData::Tok& tk = seg.tokens[ (size_t)j ];
			const char* text = wsp_model_token_text( eng->model, tk.d.id );
			td[ (size_t)j ] = tk.d;
			tt[ (size_t)j ] = wsp_token_time{ tk.t0, tk.t1, tk.vlen };
			vlen[ (size_t)j ] = wsp::voiceLength( text );
			textLen[ (size_t)j ] = text ? (int)strlen( text ) : 0;
		}
		if( wsp::computeTokenTimes( td.data(), vlen.data(), tt.data(), n, seg.t0, seg.t1, eng->tokBeg(), tokEot, energy.data(), (int)energy.size(),
				params.thold_pt, params.thold_ptsum, tokenTimeState ) )
			for( int j = 0; j < n; j++ )
			{
				ResultData::Tok& tk = seg.tokens[ (size_t)j ];
				tk.t0 = tt[ (size_t)j ].t0; tk.t1 = tt[ (size_t)j ].t1; tk.vlen = tt[ (size_t)j ].vlen;
			}
		else logMessage( eLogLevel::Warning, "computeTokenTimestamps: no signal data available" );
		if( params.max_len <= 0 ) return 1;
		std::vector<wsp_segment> pieces( (size_t)n + 1 );
		const int nNew = wsp::wrapSegment( td.data(), tt.data(), textLen.data(), 0, n, seg.t0, seg.t1, tokEot, params.max_len, pieces.data(), n + 1 );
		ResultData::Seg whole = std::move( seg );
		results.segs.pop_back();
		for( int k = 0; k < nNew; k++ )
		{
			const wsp_segment& pc = pieces[ (size_t)k ];
			ResultData::Seg s;
			s.t0 = pc.t0; s.t1 = pc.t1;
			s.tokens.assign( whole.tokens.begin() + pc.i0, whole.tokens.begin() + pc.i1 );
			for( const auto& tk : s.tokens )                   // a wrapped segment's text is that of its non-special tokens (:2724-2727)
			{
				const char* text = tk.d.id < tokEot ? wsp_model_token_text( eng->model, tk.d.id ) : nullptr;
				if( text ) s.text += text;
			}
			results.segs.push_back( std::move( s ) );
		}
		return nNew;
	}

	// whisper_lang_auto_detect (whisper.cpp:2428-2495): encode at offset 0, decode [sot], most probable language token
	HRESULT ContextObj::detectLanguage( int& langId )
	{
		int32_t id = 0;
		HR( check( wsp_detect_language( ctx, 0, (int32_t)languages().codes.size(), nullptr, &id ), "wsp_detect_language" ) );
		langId = id;
		return S_OK;
	}

	HRESULT ContextObj::checkParams( const sFullParams& params )
	{
		if( params.flag( eFullParamsFlags::SpeedupAudio ) )
		{
			// the reference's GPU back-end answers the same (ContextImpl.cpp:459-463); only its CPU back-end has the phase vocoder
			logMessage( eLogLevel::Error, "whisper_b200: the SpeedupAudio flag is not implemented (nor is it by the reference's GPU model)" );
			return E_NOTIMPL;
		}
		// audio_ctx <= 0 selects the model's n_audio_ctx, as in the reference; above it the reference would read past its positional
		// embedding and cross-KV memories (whisper.cpp:1160-1167, 1479-1480), so it is refused here
		const int nAudioCtx = eng->hp[ 1 ];
		if( params.audio_ctx > nAudioCtx )
		{
			logMessage( eLogLevel::Error, "whisper_b200: audio_ctx %d exceeds the model's n_audio_ctx %d", params.audio_ctx, nAudioCtx );
			return E_INVALIDARG;
		}
		// the reference's decoder arithmetic depends on its thread count (DESIGN.md §2); follow the caller's cpuThreads
		const int threads = params.cpuThreads < 1 ? 1 : ( params.cpuThreads > 16 ? 16 : params.cpuThreads );
		return check( wsp_set_reference_threads( ctx, threads ), "wsp_set_reference_threads" );
	}

	HRESULT WSPCALL ContextObj::runFull( const sFullParams& params, const iAudioBuffer* buffer )
	{
		if( !buffer ) return E_POINTER;
		HR( checkParams( params ) );
		results.segs.clear();                                                                     // whisper.cpp:2771-2773
		results.timeOffset = 0;
		HR( buffer->getTime( results.timeOffset ) );                                              // ContextImpl.misc.cpp:364
		const float* pcm = buffer->getPcmMono();
		const int nSamples = (int)buffer->countSamples();
		if( !pcm && nSamples > 0 ) return E_POINTER;
		// with token timestamps the clip's signal energy (get_signal_energy, :2803-2808) is computed on the device with its log-mel
		const bool tokenTimestamps = params.flag( eFullParamsFlags::TokenTimestamps );
		HR( check( wsp_set_token_timestamps( ctx, tokenTimestamps ? 1 : 0 ), "wsp_set_token_timestamps" ) );
		HR( check( wsp_pcm_to_mel( ctx, 0, pcm, nSamples ), "wsp_pcm_to_mel" ) );                 // :2782
		if( tokenTimestamps )                                                                      // :2803-2808
		{
			tokenTimeState = wsp::TokenTimeState();
			size_t n = 0;
			HR( check( wsp_get_tensor( ctx, "energy", 0, nullptr, 0, &n ), "wsp_get_tensor" ) );
			energy.resize( n );
			if( n ) HR( check( wsp_get_tensor( ctx, "energy", 0, energy.data(), n, &n ), "wsp_get_tensor" ) );
		}
		MelSource mel;
		mel.nLen = wsp_mel_len( ctx, 0 );
		mel.prepare = []( int seek, int32_t& encodeAt ) -> HRESULT { encodeAt = seek; return S_OK; };   // the whole clip's mel is resident
		curStereo = buffer->getPcmStereo();
		curStereoFrames = curStereo ? (uint64_t)nSamples : 0;
		return runImpl( params, sProgressSink{ nullptr, nullptr }, mel, tokenTimestamps );
	}

	// iContext::runStreamed (Whisper/Whisper/ContextImpl.misc.cpp:391-419): the same loop, fed window by window from a source that
	// delivers PCM in stream order.  What differs from runFull, as in the reference: every window's log-mel is normalised by ITS OWN
	// maximum (MelStreamer::makeTransposedBuffer, MelStreamer.cpp:128-170) — the clip's global maximum is not known while streaming —
	// and token-level timestamps are refused (they need the whole signal's energy).
	HRESULT WSPCALL ContextObj::runStreamed( const sFullParams& params, const sProgressSink& progress, const iAudioReader* reader )
	{
		if( !reader ) return E_POINTER;
		if( params.flag( eFullParamsFlags::TokenTimestamps ) )
		{
			logMessage( eLogLevel::Error, "eFullParamsFlags.TokenTimestamps flag is not supported in streaming mode" );
			return E_NOTIMPL;
		}
		HR( checkParams( params ) );
		results.segs.clear();
		results.timeOffset = 0;                                                                   // ContextImpl.misc.cpp:399
		int64_t ticks = 0;
		HR( reader->getDuration( ticks ) );
		if( ticks < 0 ) return E_INVALIDARG;
		IMFSourceReader* src = nullptr;
		HR( reader->getReader( &src ) );
		if( !src ) return E_POINTER;
		struct Releaser { IMFSourceReader* p; ~Releaser() { p->Release(); } } releaser{ src };
		const int64_t frames = ticks / 100000;                                                     // PcmReader.cpp:265-270
		if( frames > 0x7FFFFFFF - 3000 ) return E_INVALIDARG;
		// cpuThreads >= 2 reads the source ahead on a background thread, like MelStreamerThread (ContextImpl.misc.cpp:404-413)
		wsp::PcmStreamer streamer( [ src ]( float* dst, uint32_t cap, uint32_t* got ) -> int32_t { return src->readPcm( dst, cap, got ); },
			(size_t)frames, params.cpuThreads > 1 );
		size_t lastBufferEnd = ~(size_t)0;
		float lastBufferMax = 0.0f;
		MelSource mel;
		mel.nLen = (int)frames;
		mel.prepare = [ & ]( int seek, int32_t& encodeAt ) -> HRESULT {
			// MelInputTensor.cpp:36-52: frames [ i0, i1 ) of the stream, the rest of the 3000-frame window stays zero
			const size_t nLen = streamer.length();
			const size_t i0 = std::min( (size_t)seek, nLen );
			const size_t i1 = std::min( (size_t)seek + 3000, nLen );
			const float* pcm = nullptr;
			size_t nSamples = 0;
			const int32_t hr = streamer.window( i0, i1 - i0, &pcm, &nSamples );
			if( hr < 0 )
			{
				logMessage( eLogLevel::Error, hr == E_UNEXPECTED ? "MelStreamer doesn't support backwards seeks" : "runStreamed: the audio reader failed" );
				return hr;
			}
			// MelStreamer.cpp:152-166: a window that ends where the previous one ended (the tail of the stream) keeps that window's maximum
			const size_t bufferEnd = i1;
			float found = 0.0f;
			const bool reuse = lastBufferEnd == bufferEnd;
			HR( check( wsp_pcm_to_mel_window( ctx, 0, pcm, (int32_t)nSamples, (int32_t)( i1 - i0 ), reuse ? &lastBufferMax : nullptr, &found ), "wsp_pcm_to_mel_window" ) );
			if( !reuse ) { lastBufferEnd = bufferEnd; lastBufferMax = found; }
			encodeAt = 0;
			return S_OK;
		};
		return runImpl( params, progress, mel, false );
	}

	// iContext::runCapture (Whisper/Whisper/ContextImpl.capture.cpp:392-429): listen to a live source until the client's shouldCancel
	// says stop; the voice activity detector cuts the audio into utterances and each one goes through runFull on a background thread
	// while listening continues (csrc/capture_loop.h).  Results reach the client through sFullParams::new_segment_callback — on that
	// background thread, as in the reference — with times offset by the utterance's position in the stream (iAudioBuffer::getTime).
	HRESULT WSPCALL ContextObj::runCapture( const sFullParams& params, const sCaptureCallbacks& callbacks, const iAudioCapture* reader )
	{
		if( !reader ) return E_POINTER;
		const sCaptureParams& cp = reader->getParams();
		if( !( cp.minDuration >= 0.125f && cp.minDuration <= 30.0f ) )
		{
			logMessage( eLogLevel::Error, "%s parameter %g is out of range", "minDuration", cp.minDuration );
			return E_INVALIDARG;
		}
		if( !( cp.maxDuration >= 0.125f && cp.maxDuration <= 30.0f ) )
		{
			logMessage( eLogLevel::Error, "%s parameter %g is out of range", "maxDuration", cp.maxDuration );
			return E_INVALIDARG;
		}
		IMFSourceReader* src = nullptr;
		HR( reader->getReader( &src ) );
		if( !src ) return E_POINTER;
		struct Releaser { IMFSourceReader* p; ~Releaser() { p->Release(); } } releaser{ src };

		// the utterance handed to runFull: a stack object, never reference-counted away (TranscribeBufferObj, ContextImpl.capture.cpp:15-53)
		struct Utterance : public iAudioBuffer
		{
			const std::vector<float>& pcm;
			int64_t firstSample;
			Utterance( const std::vector<float>& p, int64_t f ) : pcm( p ), firstSample( f ) {}
			HRESULT WSPCALL QueryInterface( REFIID, void** ) override { return E_NOINTERFACE; }
			uint32_t WSPCALL AddRef() override { return 1; }
			uint32_t WSPCALL Release() override { return 1; }
			uint32_t WSPCALL countSamples() const override { return (uint32_t)pcm.size(); }
			const float* WSPCALL getPcmMono() const override { return pcm.empty() ? nullptr : pcm.data(); }
			const float* WSPCALL getPcmStereo() const override { return nullptr; }
			HRESULT WSPCALL getTime( int64_t& rdi ) const override { rdi = firstSample * 10000000 / 16000; return S_OK; }
		};
		wsp::CaptureLoop::StatusFn status;
		if( callbacks.captureStatus )
			status = [ &callbacks ]( uint8_t bits ) -> int32_t { return callbacks.captureStatus( callbacks.pv, (eCaptureStatus)bits ); };
		wsp::CaptureLoop loop(
			[ src ]( float* dst, uint32_t cap, uint32_t* got ) -> int32_t { return src->readPcm( dst, cap, got ); },
			status,
			[ this, &params ]( const std::vector<float>& pcm, int64_t firstSample ) -> int32_t {
				Utterance u( pcm, firstSample );
				return runFull( params, &u );
			},
			wsp::CaptureLoop::settingsFromSeconds( cp.minDuration, cp.maxDuration, cp.dropStartSilence, cp.pauseDuration ) );
		HR( loop.startup() );
		while( true )
		{
			const HRESULT cancel = callbacks.shouldCancel ? callbacks.shouldCancel( callbacks.pv ) : S_OK;
			if( FAILED( cancel ) ) return cancel;
			if( cancel != S_OK ) return S_OK;      // the loop's destructor lets a transcription in flight finish
			HR( loop.step() );
		}
	}

	HRESULT ContextObj::runImpl( const sFullParams& params, const sProgressSink& progress, const MelSource& mel, const bool tokenTimestamps )
	{
		HostTimer runComplete( *this, 0 );
		struct RunScope
		{
			ContextObj& c;
			RunScope( ContextObj& o ) : c( o ) { c.insideRun = true; }
			~RunScope() { c.insideRun = false; c.curStereo = nullptr; c.curStereoFrames = 0; }
		} runScope( *this );
		const int nLen = mel.nLen;

		const int tokEot = eng->tokEot(), tokSot = eng->tokSot(), tokPrev = eng->tokPrev(), tokBeg = eng->tokBeg();
		const int nTextCtx = eng->nTextCtx();
		const bool multilingual = wsp_model_is_multilingual( eng->model ) != 0;

		int langId = languages().idFromKey( params.language );
		if( params.language == 0 || params.language == makeLanguageKey( "auto" ) )              // :2789-2801
		{
			if( nLen < 1 ) return S_OK;
			int32_t at = 0;
			HR( mel.prepare( 0, at ) );
			HR( detectLanguage( langId ) );
			logMessage( eLogLevel::Info, "whisper_b200: auto-detected language: %s", languages().codes[ langId ].c_str() );
		}
		if( langId < 0 )
		{
			logMessage( eLogLevel::Error, "whisper_b200: unknown language key 0x%x", params.language );
			return E_INVALIDARG;
		}

		const int seekStart = params.offset_ms / 10;                                               // :2810-2818
		const int seekEnd = seekStart + ( params.duration_ms == 0 ? nLen : params.duration_ms / 10 );
		if( seekEnd < 100 + seekStart ) return S_OK;

		if( params.flag( eFullParamsFlags::NoContext ) ) promptPast.clear();                      // :2821-2824
		if( params.prompt_tokens && params.prompt_n_tokens > 0 )                                   // :2827-2833
		{
			promptPast.insert( promptPast.begin(), params.prompt_tokens, params.prompt_tokens + params.prompt_n_tokens );
		}
		// audio_ctx is context state that whisper_full overwrites only here (:2836): AFTER language auto-detection, which therefore
		// still encodes with the previous call's value, and not at all when the clip is shorter than 1 s (the return above)
		HR( check( wsp_set_audio_ctx( ctx, params.audio_ctx ), "wsp_set_audio_ctx" ) );

		std::vector<int32_t> promptInit = { tokSot };                                              // :2839-2848
		if( multilingual )
		{
			promptInit.push_back( tokSot + 1 + langId );
			promptInit.push_back( params.flag( eFullParamsFlags::Translate ) ? eng->special[ 6 ] : eng->special[ 7 ] );
		}

		int progressPrev = 0;
		std::vector<wsp_token_data> tokensCur;
		std::vector<int32_t> prompt;
		const bool singleSegment = params.flag( eFullParamsFlags::SingleSegment );
		const bool printSpecial = params.flag( eFullParamsFlags::PrintSpecial );

		int seek = seekStart;
		bool stoppedPrematurely = false;
		while( true )                                                                              // :2861
		{
			const int progressCur = ( 100 * ( seek - seekStart ) ) / ( seekEnd - seekStart );
			while( progressCur >= progressPrev + 5 )
			{
				progressPrev += 5;
				if( params.flag( eFullParamsFlags::PrintProgress ) ) logMessage( eLogLevel::Info, "runFull: progress = %3d%%", progressPrev );
			}
			if( progress.pfn )                                                                     // ContextImpl.cpp:533-540
			{
				HostTimer cb( *this, 1 );
				const HRESULT hr = progress.pfn( (double)( seek - seekStart ) / (double)( seekEnd - seekStart ), this, progress.pv );
				if( FAILED( hr ) ) return hr;
			}
			if( seek + 100 >= seekEnd ) break;                                                    // :2871
			if( seek > seekStart && seek + 500 >= seekEnd ) promptPast.clear();                    // :2877
			if( params.encoder_begin_callback )                                                    // :2881-2886 (HRESULT flavour: sFullParams.h:18-19)
			{
				HostTimer cb( *this, 1 );
				const HRESULT hr = params.encoder_begin_callback( this, params.encoder_begin_callback_user_data );
				if( FAILED( hr ) ) return hr;
				if( hr != S_OK ) { stoppedPrematurely = true; break; }
			}
			int32_t seek32 = seek;
			HR( mel.prepare( seek, seek32 ) );
			HR( check( wsp_encode( ctx, &seek32, 1 ), "wsp_encode" ) );                            // :2889

			int nPast = 0;
			prompt.clear();
			if( !promptPast.empty() )                                                              // :2898-2906
			{
				int nTake = params.n_max_text_ctx < nTextCtx / 2 ? params.n_max_text_ctx : nTextCtx / 2;
				if( nTake > (int)promptPast.size() ) nTake = (int)promptPast.size();
				prompt.push_back( tokPrev );
				prompt.insert( prompt.end(), promptPast.end() - nTake, promptPast.end() );
				promptPast.assign( prompt.begin() + 1, prompt.end() );
			}
			prompt.insert( prompt.end(), promptInit.begin(), promptInit.end() );

			tokensCur.clear();
			const wsp::WindowRule rule{ tokEot, tokBeg, params.max_tokens, singleSegment ? 1 : 0, nTextCtx / 2 - 4 };   // :2926
			wsp::WindowState win = wsp::windowStart();
			for( int i = 0; i < rule.nMax && !win.ended; i++ )
			{
				wsp_token_data token;
				HR( decode( prompt, nPast, i == 0, token ) );                                      // :2927-2943 decode + sample
				nPast += (int)prompt.size();
				prompt.clear();
				prompt.push_back( token.id );
				tokensCur.push_back( token );   // a token that goes back in time ends the window past its result: the resize drops it
				wsp::windowStep( win, rule, seek, seekEnd, i, token.id );                           // :2946-3003
			}
			const int seekDelta = win.seekDelta, resultLen = win.resultLen;
			const wsp_window_result result{ (int32_t)tokensCur.size(), resultLen, seekDelta, win.failed };

			if( win.failed )                                                                       // :3006-3016
			{
				if( !promptPast.empty() ) promptPast.clear();
				else
				{
					logMessage( eLogLevel::Warning, "runFull: failed to generate timestamp token - skipping one second" );
					seek += 100;
				}
				continue;
			}

			tokensCur.resize( (size_t)resultLen );                                                 // :3019
			for( const auto& r : tokensCur ) promptPast.push_back( r.id );

			auto emit = [ & ]( int64_t t0, int64_t t1, const std::string& text, int i0, int i1 ) -> HRESULT {
				ResultData::Seg s;
				s.t0 = t0; s.t1 = t1; s.text = text;
				for( int k = i0; k < i1; k++ ) { ResultData::Tok tk; tk.d = tokensCur[ k ]; s.tokens.push_back( tk ); }
				results.segs.push_back( std::move( s ) );
				int nNew = 1;
				if( tokenTimestamps )                                                              // :3063-3070, 3107-3114
				{
					nNew = tokenTimesAndWrap( params );
				}
				if( params.new_segment_callback )
				{
					HostTimer cb( *this, 1 );
					const HRESULT hr = params.new_segment_callback( this, (uint32_t)nNew, params.new_segment_callback_user_data );
					if( FAILED( hr ) ) return hr;
				}
				return S_OK;
			};

			// :3026-3119
			std::vector<wsp_segment> segs( tokensCur.size() + 1 );
			int32_t nSegs = 0;
			const uint32_t segFlags = ( singleSegment ? WSP_SEGMENT_SINGLE : 0 ) | ( printSpecial ? WSP_SEGMENT_PRINT_SPECIAL : 0 );
			HR( check( wsp_window_segments( eng->model, tokensCur.data(), &result, seek, segFlags, segs.data(), (int32_t)segs.size(), &nSegs ), "wsp_window_segments" ) );
			for( int k = 0; k < nSegs; k++ )
			{
				std::string text;
				for( int i = segs[ k ].i0; i < segs[ k ].i1; i++ )
				{
					const int id = tokensCur[ i ].id;
					const char* t = printSpecial || id < tokEot ? wsp_model_token_text( eng->model, id ) : nullptr;
					if( t ) text += t;
				}
				HR( emit( segs[ k ].t0, segs[ k ].t1, text, segs[ k ].i0, segs[ k ].i1 ) );
			}
			seek += seekDelta;                                                                     // :3121
		}
		if( progress.pfn && !stoppedPrematurely )                                                  // ContextImpl.cpp:788-792
		{
			const HRESULT hr = progress.pfn( 1.0, this, progress.pv );
			if( FAILED( hr ) ) return hr;
		}
		return S_OK;
	}

	const std::vector<std::string>& deviceNames()
	{
		static std::vector<std::string> names;
		if( names.empty() )
		{
			const int n = wsp_device_count();
			for( int i = 0; i < n; i++ )
			{
				char buf[ 256 ] = {};
				if( wsp_device_name( i, buf, sizeof( buf ) ) == WSP_OK ) names.push_back( buf );
			}
		}
		return names;
	}
}



// ===================================================================================================================
// exported functions (Whisper/whisper.def:1-8)
// ===================================================================================================================
namespace Whisper
{
	HRESULT WSPCALL setupLogger( const sLoggerSetup& setup )
	{
		std::lock_guard<std::mutex> lk( g_logMutex );
		g_logger = setup;
		return S_OK;
	}

	HRESULT WSPCALL loadModel( const wchar_t* path, const sModelSetup& setup, const sLoadModelCallbacks* callbacks, iModel** pp )
	{
		if( !path || !pp ) return E_POINTER;
		*pp = nullptr;
		if( setup.impl != eModelImplementation::GPU && setup.impl != eModelImplementation::B200 )
		{
			// the published reference DLL answers the same for its compiled-out back-ends (modelFactory.cpp:15-19, stdafx.h:30-34)
			logMessage( eLogLevel::Error, "whisper_b200: model implementation %u is not available in this build", (unsigned)setup.impl );
			return E_NOTIMPL;
		}
		int device = 0;
		if( setup.adapter && *setup.adapter )
		{
			// adapter = the name listGPUs reported, or a plain device index
			const std::string want = utf8FromWide( setup.adapter );
			const auto& names = deviceNames();
			bool found = false;
			for( size_t i = 0; i < names.size(); i++ ) if( names[ i ] == want ) { device = (int)i; found = true; }
			if( !found )
			{
				char* end = nullptr;
				const long v = strtol( want.c_str(), &end, 10 );
				if( end && *end == 0 && v >= 0 ) device = (int)v;
				else
				{
					logMessage( eLogLevel::Error, "whisper_b200: no such GPU: %s", want.c_str() );
					return E_INVALIDARG;
				}
			}
		}
		auto eng = std::make_shared<SharedEngine>();
		const std::string p8 = utf8FromWide( path );
		HR( check( wsp_model_open( p8.c_str(), &eng->model ), "wsp_model_open" ) );
		wsp_model_hparams( eng->model, eng->hp );
		wsp_model_special_tokens( eng->model, eng->special );
		if( callbacks && callbacks->cancel )
		{
			const HRESULT hr = callbacks->cancel( callbacks->pv );
			if( FAILED( hr ) ) return hr;
			if( hr != S_OK ) return E_ABORT;
		}
		if( callbacks && callbacks->progress ) callbacks->progress( 0.1, callbacks->pv );
		HR( check( wsp_engine_create( eng->model, device, &eng->engine ), "wsp_engine_create" ) );
		if( callbacks && callbacks->progress ) callbacks->progress( 1.0, callbacks->pv );
		logMessage( eLogLevel::Debug, "whisper_b200: loaded %s, %.1f MB of weights on device %d", p8.c_str(), wsp_engine_weight_bytes( eng->engine ) / 1e6, device );
		*pp = new ModelObj( eng );
		return S_OK;
	}

	uint32_t WSPCALL findLanguageKeyA( const char* lang )
	{
		if( !lang ) return UINT32_MAX;
		std::string s( lang );
		for( char& c : s ) c = (char)tolower( (unsigned char)c );
		const auto& t = languages();
		for( size_t i = 0; i < t.codes.size(); i++ )
			if( t.codes[ i ] == s || t.names[ i ] == s ) return t.entries[ i ].key;
		return UINT32_MAX;
	}
	uint32_t WSPCALL findLanguageKeyW( const wchar_t* lang )
	{
		if( !lang ) return UINT32_MAX;
		return findLanguageKeyA( utf8FromWide( lang ).c_str() );
	}
	HRESULT WSPCALL getSupportedLanguages( sLanguageList& rdi )
	{
		const auto& t = languages();
		rdi.length = (uint32_t)t.entries.size();
		rdi.pointer = t.entries.data();
		return S_OK;
	}
	HRESULT WSPCALL listGPUs( pfnListAdapters pfn, void* pv )
	{
		if( !pfn ) return E_POINTER;
		for( const auto& n : deviceNames() )
		{
			std::wstring w( n.begin(), n.end() );
			pfn( w.c_str(), pv );
		}
		return S_OK;
	}
	HRESULT WSPCALL initMediaFoundation( iMediaFoundation** pp )
	{
		if( !pp ) return E_POINTER;
		*pp = new MediaFoundationObj();
		return S_OK;
	}
	HRESULT WSPCALL createAudioReader( pfnReadPcm pfn, void* pv, int64_t durationTicks, iAudioReader** pp )
	{
		if( !pp || !pfn ) return E_POINTER;
		if( durationTicks < 0 ) return E_INVALIDARG;
		*pp = new AudioReaderObj( pfn, pv, durationTicks );
		return S_OK;
	}
	HRESULT WSPCALL createAudioCapture( pfnReadPcm pfn, void* pv, const sCaptureParams& captureParams, iAudioCapture** pp )
	{
		if( !pp || !pfn ) return E_POINTER;
		*pp = new AudioCaptureObj( pfn, pv, captureParams );
		return S_OK;
	}
	HRESULT WSPCALL createAudioBufferStereo( const float* pcmMono, const float* pcmStereo, uint32_t countSamples, iAudioBuffer** pp )
	{
		if( !pp || ( ( !pcmMono || !pcmStereo ) && countSamples ) ) return E_POINTER;
		*pp = new AudioBufferObj( pcmMono, pcmStereo, countSamples );
		return S_OK;
	}
	HRESULT WSPCALL createAudioBuffer( const float* pcmMono, uint32_t countSamples, iAudioBuffer** pp )
	{
		if( !pp || ( !pcmMono && countSamples ) ) return E_POINTER;
		*pp = new AudioBufferObj( pcmMono, countSamples );
		return S_OK;
	}
}

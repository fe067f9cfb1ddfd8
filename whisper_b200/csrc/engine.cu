// Engine: weight upload / packing.  Context: workspaces, tensor maps, encode and decode orchestration.
#include "engine.h"
#include <math.h>
#include <memory>
#include <string.h>

namespace wsp
{
	thread_local std::string g_lastError;
	std::atomic<uint64_t> g_launchCount{ 0 };

	int fail( int status, const std::string& what )
	{
		g_lastError = what;
		return status;
	}
	int cudaFail( cudaError_t e, const char* what )
	{
		g_lastError = std::string( what ) + ": " + cudaGetErrorName( e ) + " (" + cudaGetErrorString( e ) + ")";
		return e == cudaErrorMemoryAllocation ? WSP_E_OUTOFMEMORY : WSP_E_CUDA;
	}

	// ===============================================================================================================
	// Engine
	// ===============================================================================================================
	Engine::~Engine()
	{
		if( arena ) cudaFree( arena );
	}

	namespace
	{
		struct Uploader
		{
			const ModelFile& m;
			Engine& e;
			const uint8_t* devImage;
			std::vector<uint8_t> hostTmp;

			template<class T> T* alloc( size_t count )
			{
				const size_t bytes = ( count * sizeof( T ) + 255 ) & ~(size_t)255;
				if( e.arenaUsed + bytes > e.arenaSize ) return nullptr;
				T* p = reinterpret_cast<T*>( e.arena + e.arenaUsed );
				e.arenaUsed += bytes;
				return p;
			}
			// host view of a tensor's bytes (mapped file, or staged back from the device image)
			const uint8_t* hostBytes( const TensorInfo& t )
			{
				if( m.image ) return m.image + t.offset;
				hostTmp.resize( t.nbytes );
				if( cudaMemcpy( hostTmp.data(), devImage + t.offset, t.nbytes, cudaMemcpyDeviceToHost ) != cudaSuccess ) return nullptr;
				return hostTmp.data();
			}
			// raw copy of an f16 (or f32) tensor into device memory, converting f32 -> f16 when the file stores f32 matrices
			int copyF16( const std::string& name, __half* dst )
			{
				const TensorInfo* t = m.find( name );
				if( !t ) return fail( WSP_E_FORMAT, "missing tensor " + name );
				if( t->ftype != 0 )
				{
					if( devImage ) WSP_CUDA( cudaMemcpy( dst, devImage + t->offset, t->nbytes, cudaMemcpyDeviceToDevice ) );
					else WSP_CUDA( cudaMemcpy( dst, m.image + t->offset, t->nbytes, cudaMemcpyHostToDevice ) );
					return WSP_OK;
				}
				const uint8_t* src = hostBytes( *t );
				if( !src ) return fail( WSP_E_CUDA, "staging " + name );
				std::vector<__half> tmp( (size_t)t->elements() );
				const float* f = reinterpret_cast<const float*>( src );
				for( size_t i = 0; i < tmp.size(); i++ ) tmp[ i ] = __float2half_rn( f[ i ] );
				WSP_CUDA( cudaMemcpy( dst, tmp.data(), tmp.size() * 2, cudaMemcpyHostToDevice ) );
				return WSP_OK;
			}
			int copyF32( const std::string& name, float* dst )
			{
				const TensorInfo* t = m.find( name );
				if( !t ) return fail( WSP_E_FORMAT, "missing tensor " + name );
				if( t->ftype == 0 )
				{
					if( devImage ) WSP_CUDA( cudaMemcpy( dst, devImage + t->offset, t->nbytes, cudaMemcpyDeviceToDevice ) );
					else WSP_CUDA( cudaMemcpy( dst, m.image + t->offset, t->nbytes, cudaMemcpyHostToDevice ) );
					return WSP_OK;
				}
				const uint8_t* src = hostBytes( *t );
				if( !src ) return fail( WSP_E_CUDA, "staging " + name );
				std::vector<float> tmp( (size_t)t->elements() );
				const __half* hsrc = reinterpret_cast<const __half*>( src );
				for( size_t i = 0; i < tmp.size(); i++ ) tmp[ i ] = __half2float( hsrc[ i ] );
				WSP_CUDA( cudaMemcpy( dst, tmp.data(), tmp.size() * 4, cudaMemcpyHostToDevice ) );
				return WSP_OK;
			}
			// host f32 copy of any tensor
			int hostF32( const std::string& name, std::vector<float>& out )
			{
				const TensorInfo* t = m.find( name );
				if( !t ) return fail( WSP_E_FORMAT, "missing tensor " + name );
				const uint8_t* src = hostBytes( *t );
				if( !src ) return fail( WSP_E_CUDA, "staging " + name );
				out.resize( (size_t)t->elements() );
				if( t->ftype == 0 ) memcpy( out.data(), src, out.size() * 4 );
				else
				{
					const __half* hsrc = reinterpret_cast<const __half*>( src );
					for( size_t i = 0; i < out.size(); i++ ) out[ i ] = __half2float( hsrc[ i ] );
				}
				return WSP_OK;
			}
			int ln( const std::string& prefix, LnW& w, int d )
			{
				w.g = alloc<float>( d );
				w.b = alloc<float>( d );
				if( !w.g || !w.b ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
				WSP_CHECK( copyF32( prefix + ".weight", w.g ) );
				return copyF32( prefix + ".bias", w.b );
			}
			int matrix( const std::string& name, __half*& w, size_t count )
			{
				w = alloc<__half>( count );
				if( !w ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
				return copyF16( name, w );
			}
			int vec( const std::string& name, float*& b, size_t count )
			{
				b = alloc<float>( count );
				if( !b ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
				return copyF32( name, b );
			}
			// stacked (q | k | v) weights [3d][d] and bias (q.b | 0 | v.b)
			int qkv( const std::string& p, __half*& w, float*& b, int d )
			{
				const size_t dd = (size_t)d * d;
				w = alloc<__half>( 3 * dd );
				b = alloc<float>( 3 * (size_t)d );
				if( !w || !b ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
				WSP_CHECK( copyF16( p + "attn.query.weight", w ) );
				WSP_CHECK( copyF16( p + "attn.key.weight", w + dd ) );
				WSP_CHECK( copyF16( p + "attn.value.weight", w + 2 * dd ) );
				WSP_CUDA( cudaMemset( b, 0, 3 * (size_t)d * 4 ) );
				WSP_CHECK( copyF32( p + "attn.query.bias", b ) );
				return copyF32( p + "attn.value.bias", b + 2 * d );
			}
		};
	}

	int createEngine( const ModelFile& m, int device, const void* devImage, uint64_t imageSize, Engine** out )
	{
		if( !m.image && !devImage ) return fail( WSP_E_INVALIDARG, "no tensor data: model has no file image and no device image was given" );
		if( devImage && imageSize < m.imageSize ) return fail( WSP_E_INVALIDARG, "device image smaller than the model file" );
		int count = 0;
		WSP_CUDA( cudaGetDeviceCount( &count ) );
		if( device < 0 || device >= count ) return fail( WSP_E_INVALIDARG, "no such CUDA device" );
		WSP_CUDA( cudaSetDevice( device ) );
		cudaDeviceProp prop;
		WSP_CUDA( cudaGetDeviceProperties( &prop, device ) );
		if( prop.major != 9 || prop.minor != 0 )
			return fail( WSP_E_CUDA, std::string( "whisper_b200 needs an sm_90a device (wgmma/TMA); found " ) + prop.name + " sm_" + std::to_string( prop.major ) + std::to_string( prop.minor ) );

		std::unique_ptr<Engine> e( new Engine() );
		e->device = device;
		e->numSMs = prop.multiProcessorCount;
		e->hp = m.hp;
		e->tokEot = m.vocab.token_eot; e->tokSot = m.vocab.token_sot; e->tokPrev = m.vocab.token_prev;
		e->tokSolm = m.vocab.token_solm; e->tokNot = m.vocab.token_not; e->tokBeg = m.vocab.token_beg;
		// the reference's g_lang: language l is token sot + 1 + l, up to the task tokens (whisper.cpp:2466-2468)
		e->nLangs = m.vocab.multilingual() ? Vocab::token_translate - m.vocab.token_sot - 1 : 0;
		e->tokenText = m.vocab.id_to_token;
		const HParams& h = m.hp;
		const int d = h.n_audio_state;
		const size_t dd = (size_t)d * d;

		// arena size: every tensor as f16/f32 + padding + packed extras
		size_t need = 0;
		for( const auto& t : m.tensors ) need += (size_t)t.elements() * 4 + 512;
		need += (size_t)d * 3 * kConv1KTap * 2 + ( 1u << 20 );
		need += (size_t)( h.n_audio_layer + h.n_text_layer ) * 3 * d * 4 + (size_t)h.n_text_layer * 2 * d * 4 + ( 1u << 20 );
		e->arenaSize = need;
		WSP_CUDA( cudaMalloc( &e->arena, e->arenaSize ) );
		Uploader up{ m, *e, static_cast<const uint8_t*>( devImage ) };

		// ---- encoder front: conv weights repacked to [out][tap][cin] (cin padded to 128 for conv1) ----
		{
			std::vector<float> w;
			WSP_CHECK( up.hostF32( "encoder.conv1.weight", w ) );   // [o][c][k], k fastest (ne = 3, 80, d)
			std::vector<__half> p( (size_t)d * 3 * kConv1KTap, __float2half_rn( 0.0f ) );
			for( int o = 0; o < d; o++ )
				for( int c = 0; c < h.n_mels; c++ )
					for( int k = 0; k < 3; k++ )
						p[ ( (size_t)o * 3 + k ) * kConv1KTap + c ] = __float2half_rn( w[ ( (size_t)o * h.n_mels + c ) * 3 + k ] );
			e->conv1w = up.alloc<__half>( p.size() );
			if( !e->conv1w ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
			WSP_CUDA( cudaMemcpy( e->conv1w, p.data(), p.size() * 2, cudaMemcpyHostToDevice ) );
			WSP_CHECK( up.hostF32( "encoder.conv2.weight", w ) );   // [o][c][k] (ne = 3, d, d)
			p.assign( (size_t)d * 3 * d, __float2half_rn( 0.0f ) );
			for( int o = 0; o < d; o++ )
				for( int c = 0; c < d; c++ )
					for( int k = 0; k < 3; k++ )
						p[ ( (size_t)o * 3 + k ) * d + c ] = __float2half_rn( w[ ( (size_t)o * d + c ) * 3 + k ] );
			e->conv2w = up.alloc<__half>( p.size() );
			if( !e->conv2w ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
			WSP_CUDA( cudaMemcpy( e->conv2w, p.data(), p.size() * 2, cudaMemcpyHostToDevice ) );
		}
		WSP_CHECK( up.vec( "encoder.conv1.bias", e->conv1b, d ) );
		WSP_CHECK( up.vec( "encoder.conv2.bias", e->conv2b, d ) );
		WSP_CHECK( up.vec( "encoder.positional_embedding", e->encPos, (size_t)d * h.n_audio_ctx ) );
		WSP_CHECK( up.ln( "encoder.ln_post", e->encLnPost, d ) );

		e->enc.resize( h.n_audio_layer );
		for( int i = 0; i < h.n_audio_layer; i++ )
		{
			const std::string p = "encoder.blocks." + std::to_string( i ) + ".";
			EncLayerW& L = e->enc[ i ];
			WSP_CHECK( up.ln( p + "attn_ln", L.ln1, d ) );
			WSP_CHECK( up.ln( p + "mlp_ln", L.ln2, d ) );
			WSP_CHECK( up.qkv( p, L.wqkv, L.bqkv, d ) );
			WSP_CHECK( up.matrix( p + "attn.out.weight", L.wo, dd ) );
			WSP_CHECK( up.vec( p + "attn.out.bias", L.bo, d ) );
			WSP_CHECK( up.matrix( p + "mlp.0.weight", L.w1, 4 * dd ) );
			WSP_CHECK( up.vec( p + "mlp.0.bias", L.b1, 4 * (size_t)d ) );
			WSP_CHECK( up.matrix( p + "mlp.2.weight", L.w2, 4 * dd ) );
			WSP_CHECK( up.vec( p + "mlp.2.bias", L.b2, d ) );
		}

		// ---- decoder ----
		WSP_CHECK( up.vec( "decoder.positional_embedding", e->decPos, (size_t)d * h.n_text_ctx ) );
		WSP_CHECK( up.matrix( "decoder.token_embedding.weight", e->tokEmb, (size_t)d * h.n_vocab ) );
		WSP_CHECK( up.ln( "decoder.ln", e->decLn, d ) );
		e->dec.resize( h.n_text_layer );
		e->crossW = up.alloc<__half>( (size_t)h.n_text_layer * 2 * dd );
		e->crossB = up.alloc<float>( (size_t)h.n_text_layer * 2 * d );
		if( !e->crossW || !e->crossB ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
		WSP_CUDA( cudaMemset( e->crossB, 0, (size_t)h.n_text_layer * 2 * d * 4 ) );
		for( int i = 0; i < h.n_text_layer; i++ )
		{
			const std::string p = "decoder.blocks." + std::to_string( i ) + ".";
			DecLayerW& L = e->dec[ i ];
			WSP_CHECK( up.ln( p + "attn_ln", L.ln1, d ) );
			WSP_CHECK( up.ln( p + "cross_attn_ln", L.lnc, d ) );
			WSP_CHECK( up.ln( p + "mlp_ln", L.ln3, d ) );
			WSP_CHECK( up.qkv( p, L.wqkv, L.bqkv, d ) );
			WSP_CHECK( up.matrix( p + "attn.out.weight", L.wo, dd ) );
			WSP_CHECK( up.vec( p + "attn.out.bias", L.bo, d ) );
			WSP_CHECK( up.matrix( p + "cross_attn.query.weight", L.wcq, dd ) );
			WSP_CHECK( up.vec( p + "cross_attn.query.bias", L.bcq, d ) );
			WSP_CHECK( up.matrix( p + "cross_attn.out.weight", L.wco, dd ) );
			WSP_CHECK( up.vec( p + "cross_attn.out.bias", L.bco, d ) );
			WSP_CHECK( up.matrix( p + "mlp.0.weight", L.w1, 4 * dd ) );
			WSP_CHECK( up.vec( p + "mlp.0.bias", L.b1, 4 * (size_t)d ) );
			WSP_CHECK( up.matrix( p + "mlp.2.weight", L.w2, 4 * dd ) );
			WSP_CHECK( up.vec( p + "mlp.2.bias", L.b2, d ) );
			// cross-attention K/V projections of all layers stacked into one [L*2d][d] GEMM operand
			WSP_CHECK( up.copyF16( p + "cross_attn.key.weight", e->crossW + (size_t)i * 2 * dd ) );
			WSP_CHECK( up.copyF16( p + "cross_attn.value.weight", e->crossW + (size_t)i * 2 * dd + dd ) );
			WSP_CHECK( up.copyF32( p + "cross_attn.value.bias", e->crossB + (size_t)i * 2 * d + d ) );
		}

		// ---- mel tables (whisper.cpp:2076 Hann in double -> f32; twiddles in double) ----
		{
			std::vector<float> hann( 400 );
			std::vector<double> ct( 400 ), st( 400 );
			for( int i = 0; i < 400; i++ )
			{
				hann[ i ] = (float)( 0.5 * ( 1.0 - cos( ( 2.0 * M_PI * i ) / 400.0 ) ) );
				ct[ i ] = cos( 2.0 * M_PI * i / 400.0 );
				st[ i ] = sin( 2.0 * M_PI * i / 400.0 );
			}
			float* dh = up.alloc<float>( 400 );
			double* dc = up.alloc<double>( 400 );
			double* ds = up.alloc<double>( 400 );
			float* df = up.alloc<float>( m.filters.size() );
			double2* dt = up.alloc<double2>( 400 );
			short2* db = up.alloc<short2>( 80 );
			if( !dh || !dc || !ds || !df || !dt || !db ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
			std::vector<double2> tw( 400 );
			for( int i = 0; i < 400; i++ ) tw[ i ] = make_double2( ct[ i ], st[ i ] );
			// the bins a band actually weighs: skipping the exact zeros of a filter row leaves the double sum bit-identical (x + 0.0 == x)
			std::vector<short2> bands( 80, make_short2( 0, 201 ) );
			if( m.filters.size() == (size_t)80 * 201 )
				for( int j = 0; j < 80; j++ )
				{
					int lo = 201, hi = 0;
					for( int k = 0; k < 201; k++ )
						if( m.filters[ (size_t)j * 201 + k ] != 0.0f ) { lo = k < lo ? k : lo; hi = k + 1; }
					bands[ (size_t)j ] = lo < hi ? make_short2( (short)lo, (short)hi ) : make_short2( 0, 0 );
				}
			WSP_CUDA( cudaMemcpy( dt, tw.data(), 400 * sizeof( double2 ), cudaMemcpyHostToDevice ) );
			WSP_CUDA( cudaMemcpy( db, bands.data(), 80 * sizeof( short2 ), cudaMemcpyHostToDevice ) );
			e->mel.twiddle = dt; e->mel.band = db;
			WSP_CUDA( cudaMemcpy( dh, hann.data(), 400 * 4, cudaMemcpyHostToDevice ) );
			WSP_CUDA( cudaMemcpy( dc, ct.data(), 400 * 8, cudaMemcpyHostToDevice ) );
			WSP_CUDA( cudaMemcpy( ds, st.data(), 400 * 8, cudaMemcpyHostToDevice ) );
			WSP_CUDA( cudaMemcpy( df, m.filters.data(), m.filters.size() * 4, cudaMemcpyHostToDevice ) );
			e->mel.hann = dh; e->mel.cosT = dc; e->mel.sinT = ds; e->mel.filters = df;
		}
		// ---- the phase vocoder's 800-point window and twiddles (speed-up: log_mel_spectrogram with fft_size 800, whisper.cpp:2076, 2303) ----
		{
			std::vector<float> hann( 800 );
			std::vector<double2> tw( 800 );
			for( int i = 0; i < 800; i++ )
			{
				hann[ i ] = (float)( 0.5 * ( 1.0 - cos( ( 2.0 * M_PI * i ) / 800.0 ) ) );
				tw[ i ] = make_double2( cos( 2.0 * M_PI * i / 800.0 ), sin( 2.0 * M_PI * i / 800.0 ) );
			}
			float* dh = up.alloc<float>( 800 );
			double2* dt = up.alloc<double2>( 800 );
			if( !dh || !dt ) return fail( WSP_E_OUTOFMEMORY, "weight arena" );
			WSP_CUDA( cudaMemcpy( dh, hann.data(), 800 * 4, cudaMemcpyHostToDevice ) );
			WSP_CUDA( cudaMemcpy( dt, tw.data(), 800 * sizeof( double2 ), cudaMemcpyHostToDevice ) );
			e->melVocoder = e->mel;
			e->melVocoder.hann = dh; e->melVocoder.twiddle = dt;
			e->melVocoder.cosT = e->melVocoder.sinT = nullptr;
		}
		WSP_CUDA( cudaDeviceSynchronize() );
		*out = e.release();
		return WSP_OK;
	}
}

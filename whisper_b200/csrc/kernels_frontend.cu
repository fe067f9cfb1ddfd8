// Front-end + normalisation kernels (HBM/latency-bound, no tensor cores): log-mel spectrogram, window gather, LayerNorm, embedding.
#include "kernels.cuh"
#include "ptx.cuh"
#include "speaker.h"
#include <math.h>

namespace kern
{
	// float <-> order-preserving int, for atomicMax on floats of any sign
	__device__ __forceinline__ int orderedFromFloat( float f )
	{
		const int i = __float_as_int( f );
		return i >= 0 ? i : i ^ 0x7FFFFFFF;
	}
	__device__ __forceinline__ float floatFromOrdered( int i ) { return __int_as_float( i >= 0 ? i : i ^ 0x7FFFFFFF ); }

	// ---------------------------------------------------------------------------------------------------------------
	// log-mel: one CTA per frame.  Oracle: log_mel_spectrogram (Whisper/source/whisper.cpp:2060-2181):
	//   frame i = hann .* pcm[160*i .. +400) (zero past the end) ; 400-point DFT ; power ; fold bin j with 400-j ;
	//   mel[j] = sum_k folded[k]*filters[j][k] in double ; log10(max(., 1e-10)) -> float.
	// The oracle's recursive f32 FFT (:2009-2056) is replaced by a direct 201-bin DFT with f64 accumulation: exact to f32
	// rounding, so the only difference to the oracle is the oracle's own f32 FFT round-off.
	// FFT = 800 is the phase vocoder of whisper_pcm_to_mel_phase_vocoder (:2299-2311, speed_up = true): hop 320, an 800-point
	// Hann window and DFT, the same fold over bins 1..399 (bin 400 single, bin 401 = |X399|^2 left unfolded because the loop stops
	// at 399), then adjacent bins averaged onto the model's 201: P'[j] = 0.5 * (P[2j] + P[2j+1]) (:2130-2135).
	constexpr int MEL_BINS = 201;
	constexpr int MEL_BANDS = 80;
	template<int FFT> struct MelGeom;
	template<> struct MelGeom<400> { static constexpr int HOP = 160, THREADS = 256; };
	template<> struct MelGeom<800> { static constexpr int HOP = 320, THREADS = 512; };

	template<int FFT>
	__device__ __forceinline__ void melFrame( const MelTables& tb, const float* __restrict__ pcm, int nSamples, int nLen, float* __restrict__ melRaw, int* maxSlot, const int frame )
	{
		constexpr int NBINS = FFT / 2 + 1;         // DFT bins computed: 201 | 401
		constexpr int NWARPS = MelGeom<FFT>::THREADS / 32;
		__shared__ float sx[ FFT ];
		__shared__ double2 stw[ FFT ];          // { cos, sin }( 2 pi m / FFT )
		__shared__ double sA[ 2 ][ FFT / 4 ];   // [k parity][n]: cosine-side combinations
		__shared__ double sB[ 2 ][ FFT / 4 ];   //                 sine-side combinations
		__shared__ float sp[ NBINS + 7 ];
		__shared__ float smax[ NWARPS ];
		const int tid = threadIdx.x;
		const int offset = frame * MelGeom<FFT>::HOP;
		for( int n = tid; n < FFT; n += blockDim.x )
		{
			const int idx = offset + n;
			sx[ n ] = idx < nSamples ? tb.hann[ n ] * pcm[ idx ] : 0.0f;
			stw[ n ] = tb.twiddle[ n ];
		}
		__syncthreads();
		// Real FFT-point DFT in a quarter of the multiply-adds (Q = FFT / 4).  With w = exp(-2 pi i k / FFT):
		//   X[k] = sum_{n<2Q} y[n] w^n,  y[n] = x[n] + (-1)^k x[n+2Q]           (w^2Q = (-1)^k)
		//        = y[0] + y[Q] (-i)^k + sum_{n=1..Q-1} ( y[n] w^n + (-1)^k y[2Q-n] conj(w^n) )
		//   Re = y[0] + Re(y[Q] (-i)^k) + sum cos(t_n) A[n],   A[n] = y[n] + (-1)^k y[2Q-n]
		//   Im =        Im(y[Q] (-i)^k) - sum sin(t_n) B[n],   B[n] = y[n] - (-1)^k y[2Q-n]
		// (f64 accumulation as before; only the summation order differs from the plain FFT-term sum)
		constexpr int Q = FFT / 4;   // 100 | 200
		if( tid < 2 * Q )
		{
			const int par = tid / Q, n = tid - par * Q;
			const double sg = par ? -1.0 : 1.0;
			const double yn = (double)sx[ n ] + sg * (double)sx[ n + 2 * Q ];
			const double ym = n == 0 ? 0.0 : (double)sx[ 2 * Q - n ] + sg * (double)sx[ 4 * Q - n ];   // y[2Q-n]
			sA[ par ][ n ] = yn + sg * ym;
			sB[ par ][ n ] = yn - sg * ym;
		}
		__syncthreads();
		if( tid < NBINS )
		{
			const int k = tid;
			const int par = k & 1;
			const double sg = par ? -1.0 : 1.0;
			const double y0 = (double)sx[ 0 ] + sg * (double)sx[ 2 * Q ];
			const double yQ = (double)sx[ Q ] + sg * (double)sx[ 3 * Q ];
			double re = y0, im = 0.0;
			switch( k & 3 )   // y[Q] * (-i)^k
			{
			case 0: re += yQ; break;
			case 1: im -= yQ; break;
			case 2: re -= yQ; break;
			default: im += yQ; break;
			}
			const double* A = sA[ par ];
			const double* Bv = sB[ par ];
			int idx = k;
#pragma unroll 4
			for( int n = 1; n < Q; n++ )
			{
				const double2 w = stw[ idx ];
				re += A[ n ] * w.x;
				im -= Bv[ n ] * w.y;
				idx += k;
				if( idx >= FFT ) idx -= FFT;
			}
			const float fr = (float)re, fi = (float)im;
			float pw = fr * fr + fi * fi;
			if constexpr( FFT == 800 )
				if( k == FFT / 2 - 1 ) sp[ FFT / 2 + 1 ] = pw;   // bin 401 = |X401|^2 = |X399|^2, not folded
			if( k > 0 && k < FFT / 2 ) pw = pw + pw;   // fft_out[j] += fft_out[FFT - j]  (whisper.cpp:2118-2123)
			sp[ k ] = pw;
		}
		__syncthreads();
		float v = -INFINITY;
		if( tid < MEL_BANDS )
		{
			const float* f = tb.filters + tid * MEL_BINS;
			const short2 range = tb.band[ tid ];   // outside it the filter row is exactly zero: those terms add +0.0
			double sum = 0.0;
			for( int k = range.x; k < range.y; k++ )
			{
				float p = sp[ k ];
				if constexpr( FFT == 800 )
					p = (float)( 0.5 * (double)( sp[ 2 * k ] + sp[ 2 * k + 1 ] ) );   // whisper.cpp:2133, f32 sum, double half
				sum += (double)( p * f[ k ] );   // float product, double accumulate (whisper.cpp:2139-2143)
			}
			if( sum < 1e-10 ) sum = 1e-10;
			v = (float)log10( sum );
			melRaw[ (size_t)tid * nLen + frame ] = v;
		}
		// block max -> one atomic
		v = ptx::warp_max( v );
		if( ( tid & 31 ) == 0 ) smax[ tid >> 5 ] = v;
		__syncthreads();
		if( tid == 0 )
		{
			float m = smax[ 0 ];
			for( int w = 1; w < 3; w++ ) m = fmaxf( m, smax[ w ] );   // bands live in warps 0..2
			atomicMax( maxSlot, orderedFromFloat( m ) );
		}
	}

	// up to MEL_BATCH chunks in one launch: blockIdx.y = chunk (the driver loop of BASELINE.md §2 transforms B chunks per step)
	template<int FFT>
	__global__ void __launch_bounds__( MelGeom<FFT>::THREADS )
		mel_power_batch_kernel( MelTables tb, MelBatch mb )
	{
		const int b = blockIdx.y;
		if( (int)blockIdx.x >= mb.nLen[ b ] ) return;
		melFrame<FFT>( tb, mb.pcm[ b ], mb.nSamples[ b ], mb.nLen[ b ], mb.mel[ b ], mb.maxSlots + b, blockIdx.x );
	}

	__device__ __forceinline__ void melNormOne( float* mel, int i, const int* maxSlot )
	{
		// whisper.cpp:2161-2177: mmax (double) -= 8.0; clamp; (x + 4.0) / 4.0 in double, stored as float
		const double mmax = (double)floatFromOrdered( *maxSlot ) - 8.0;
		float v = mel[ i ];
		if( (double)v < mmax ) v = (float)mmax;
		mel[ i ] = (float)( ( (double)v + 4.0 ) / 4.0 );
	}
	__global__ void mel_norm_batch_kernel( MelBatch mb )
	{
		const int b = blockIdx.y;
		const int i = blockIdx.x * blockDim.x + threadIdx.x;
		if( i >= MEL_BANDS * mb.nLen[ b ] ) return;
		melNormOne( mb.mel[ b ], i, mb.maxSlots + b );
	}

	__global__ void init_max_kernel( int* maxSlot ) { maxSlot[ threadIdx.x ] = orderedFromFloat( -1e20f ); }

	// the longest chunk's frame count (the grid's x extent), or -1 for a batch size outside 1..MEL_BATCH
	static int melBatchFrames( const MelBatch& mb )
	{
		if( mb.count < 1 || mb.count > MEL_BATCH ) return -1;
		int maxLen = 0;
		for( int b = 0; b < mb.count; b++ ) maxLen = mb.nLen[ b ] > maxLen ? mb.nLen[ b ] : maxLen;
		return maxLen;
	}
	cudaError_t melBatchPower( const MelTables& tb, const MelBatch& mb, bool speedUp, cudaStream_t s )
	{
		const int maxLen = melBatchFrames( mb );
		if( maxLen < 0 ) return cudaErrorInvalidValue;
		init_max_kernel<<<1, mb.count, 0, s>>>( mb.maxSlots );
		if( maxLen > 0 )
		{
			if( speedUp )
				mel_power_batch_kernel<800><<<dim3( maxLen, mb.count ), MelGeom<800>::THREADS, 0, s>>>( tb, mb );
			else
				mel_power_batch_kernel<400><<<dim3( maxLen, mb.count ), MelGeom<400>::THREADS, 0, s>>>( tb, mb );
		}
		return cudaGetLastError();
	}
	cudaError_t melBatchNormalize( const MelBatch& mb, cudaStream_t s )
	{
		const int maxLen = melBatchFrames( mb );
		if( maxLen < 0 ) return cudaErrorInvalidValue;
		if( maxLen > 0 )
			mel_norm_batch_kernel<<<dim3( ( MEL_BANDS * maxLen + 255 ) / 256, mb.count ), 256, 0, s>>>( mb );
		return cudaGetLastError();
	}

	// ---------------------------------------------------------------------------------------------------------------
	// window gather: mel[80][nLen] (band-major) -> f16 [1 + frames + 1][80] (time-major) at `offset`, zero beyond nLen
	// (whisper.cpp:1104-1120 copies the slice and zero-pads; the f16 rounding is ggml's conv input conversion, ggml.c:5275-5283).
	// Row r holds frame r - 1; rows 0 and frames + 1 are conv1's zero padding and are written here too: where they lie depends on
	// the window length (2 * audio_ctx frames), which may change from one encode to the next.
	__global__ void __launch_bounds__( 256 )
		mel_window_kernel( const float* __restrict__ mel, int nLen, int offset, __half* __restrict__ dst, int frames )
	{
		__shared__ float tile[ MEL_BANDS ][ 33 ];
		const int r0 = blockIdx.x * 32;
		for( int i = threadIdx.x; i < MEL_BANDS * 32; i += blockDim.x )
		{
			const int c = i >> 5, tt = i & 31;
			const int t = r0 + tt - 1;
			const int src = offset + t;
			tile[ c ][ tt ] = ( t >= 0 && t < frames && src < nLen ) ? mel[ (size_t)c * nLen + src ] : 0.0f;
		}
		__syncthreads();
		for( int i = threadIdx.x; i < MEL_BANDS * 32; i += blockDim.x )
		{
			const int tt = i / MEL_BANDS, c = i - tt * MEL_BANDS;
			const int r = r0 + tt;
			if( r < frames + 2 )
				dst[ (size_t)r * MEL_BANDS + c ] = __float2half_rn( tile[ c ][ tt ] );
		}
	}
	cudaError_t melWindow( const float* mel, int nLen, int offset, __half* dst, int frames, cudaStream_t s )
	{
		mel_window_kernel<<<( frames + 2 + 31 ) / 32, 256, 0, s>>>( mel, nLen, offset, dst, frames );
		return cudaGetLastError();
	}

	// ---------------------------------------------------------------------------------------------------------------
	// signal energy (get_signal_energy, whisper.cpp:3356-3372): one CTA per ENERGY_TILE samples of one chunk (blockIdx.y).  The CTA
	// stages |x| of its tile and the 32-sample halo on each side in shared memory, zero outside the clip, and each thread adds its
	// sample's 65 terms in the reference's order: a +0.0f in place of a skipped term leaves an f32 sum unchanged, so the result is the
	// reference's bit for bit.  The division is IEEE (no fast math in this build).
	constexpr int ENERGY_TILE = 512;
	static_assert( sizeof( EnergyBatch ) <= 4096, "EnergyBatch is passed by value as a kernel parameter" );
	__global__ void __launch_bounds__( ENERGY_TILE )
		signal_energy_kernel( const EnergyBatch eb )
	{
		__shared__ float sx[ ENERGY_TILE + 2 * ENERGY_HW ];
		const int b = blockIdx.y;
		const int n = eb.nSamples[ b ];
		const int i0 = blockIdx.x * ENERGY_TILE;
		if( i0 >= n ) return;
		const float* __restrict__ x = eb.pcm[ b ];
		for( int k = threadIdx.x; k < ENERGY_TILE + 2 * ENERGY_HW; k += ENERGY_TILE )
		{
			const int idx = i0 - ENERGY_HW + k;
			sx[ k ] = idx >= 0 && idx < n ? fabsf( x[ idx ] ) : 0.0f;
		}
		__syncthreads();
		const int i = i0 + threadIdx.x;
		if( i >= n ) return;
		float sum = 0.0f;
#pragma unroll
		for( int j = 0; j <= 2 * ENERGY_HW; j++ ) sum += sx[ threadIdx.x + j ];
		eb.out[ eb.row[ b ] * eb.stride + i ] = sum / (float)( 2 * ENERGY_HW + 1 );
	}
	cudaError_t signalEnergy( const EnergyBatch& eb, cudaStream_t s )
	{
		if( eb.count < 1 || eb.count > ENERGY_BATCH ) return cudaErrorInvalidValue;
		int maxN = 0;
		for( int b = 0; b < eb.count; b++ ) maxN = eb.nSamples[ b ] > maxN ? eb.nSamples[ b ] : maxN;
		const int tiles = ( maxN + ENERGY_TILE - 1 ) / ENERGY_TILE;   // one launch even for a batch of empty clips
		signal_energy_kernel<<<dim3( tiles > 0 ? tiles : 1, eb.count ), ENERGY_TILE, 0, s>>>( eb );
		return cudaGetLastError();
	}

	// ---------------------------------------------------------------------------------------------------------------
	// stereo -> mono (AudioBuffer::appendDownmixedStereo, Whisper/MF/AudioBuffer.cpp:57-93): (l + r) * 0.5f per frame, two frames per
	// thread and step.  An add then a multiply cannot contract into an FMA, so every sample is the reference's bit for bit.
	constexpr int DOWNMIX_THREADS = 256;
	__global__ void __launch_bounds__( DOWNMIX_THREADS )
		downmix_stereo_kernel( const float* __restrict__ lr, float* __restrict__ mono, int nFrames )
	{
		const float4* in = reinterpret_cast<const float4*>( lr );
		float2* out = reinterpret_cast<float2*>( mono );
		for( int i = blockIdx.x * blockDim.x + threadIdx.x; i < nFrames / 2; i += gridDim.x * blockDim.x )
		{
			const float4 v = in[ i ];
			out[ i ] = make_float2( ( v.x + v.y ) * 0.5f, ( v.z + v.w ) * 0.5f );
		}
		if( ( nFrames & 1 ) && blockIdx.x == 0 && threadIdx.x == 0 ) mono[ nFrames - 1 ] = ( lr[ 2 * nFrames - 2 ] + lr[ 2 * nFrames - 1 ] ) * 0.5f;
	}
	cudaError_t downmixStereo( const float* lr, float* mono, int nFrames, cudaStream_t s )
	{
		const int blocks = ( nFrames / 2 + DOWNMIX_THREADS - 1 ) / DOWNMIX_THREADS;
		downmix_stereo_kernel<<<blocks > 0 ? blocks : 1, DOWNMIX_THREADS, 0, s>>>( lr, mono, nFrames );
		return cudaGetLastError();
	}

	// ---------------------------------------------------------------------------------------------------------------
	// detectSpeaker's channel sums (ContextImpl.diarize.cpp:17-52): one warp per segment.  The reference keeps four f32 chains, one per
	// SSE lane { |L even|, |R even|, |L odd|, |R odd| }, each added in frame order; a tree would round differently and move decisions
	// whose ratio lies within rounding of 1.1.  So lanes 0..3 of the warp each run one chain over a frame pair (one float4) per step,
	// and the whole warp keeps SPK_STAGES - 1 tiles of pairs in flight with coalesced cp.async copies into shared memory, so the chains
	// never wait for HBM.  Pairs past the segment, and the missing odd frame of an odd count, are zero-filled: +0 leaves a chain as it is.
	constexpr int SPK_WARPS = 4;
	constexpr int SPK_STAGES = 3;
	constexpr int SPK_PER_LANE = 8;
	constexpr int SPK_TILE = 32 * SPK_PER_LANE;   // frame pairs per stage
	static_assert( SPK_WARPS * SPK_STAGES * SPK_TILE * 16 <= 48 * 1024, "static shared memory" );
	__global__ void __launch_bounds__( SPK_WARPS * 32 )
		speaker_kernel( const SpeakerJob* __restrict__ jobs, int32_t* __restrict__ out, int n )
	{
		__shared__ float4 tiles[ SPK_WARPS ][ SPK_STAGES ][ SPK_TILE ];
		const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
		const int seg = blockIdx.x * SPK_WARPS + warp;
		if( seg >= n ) return;
		const SpeakerJob job = jobs[ seg ];
		if( job.pre != wsp::kSpeakerSums )
		{
			if( lane == 0 ) out[ seg ] = job.pre;
			return;
		}
		const float4* src = reinterpret_cast<const float4*>( job.lr );
		const int64_t count = job.count;
		const int nTiles = (int)( ( ( count + 1 ) / 2 + SPK_TILE - 1 ) / SPK_TILE );
		float4( *buf )[ SPK_TILE ] = tiles[ warp ];
		auto stage = [ & ]( int t ) {
			if( t < nTiles )
#pragma unroll
				for( int k = 0; k < SPK_PER_LANE; k++ )
				{
					const int64_t p = (int64_t)t * SPK_TILE + k * 32 + lane;
					const uint32_t bytes = 2 * p + 2 <= count ? 16u : ( 2 * p < count ? 8u : 0u );
					ptx::cp_async16_zfill( &buf[ t % SPK_STAGES ][ k * 32 + lane ], bytes ? src + p : src, bytes );
				}
			ptx::cp_async_commit();   // an empty group past the last tile keeps the wait count below uniform
		};
#pragma unroll
		for( int t = 0; t < SPK_STAGES - 1; t++ ) stage( t );
		float acc = 0.0f;   // lane c < 4: lane c of the reference's accumulator
		for( int t = 0; t < nTiles; t++ )
		{
			stage( t + SPK_STAGES - 1 );                 // into the buffer folded in step t - 1
			ptx::cp_async_wait<SPK_STAGES - 1>();
			__syncwarp();
			if( lane < 4 )
			{
				const float* f = reinterpret_cast<const float*>( buf[ t % SPK_STAGES ] ) + lane;
#pragma unroll 32
				for( int j = 0; j < SPK_TILE; j++ ) acc = wsp::speakerFold( acc, f[ 4 * j ] );
			}
			__syncwarp();
		}
		const float lEven = __shfl_sync( 0xFFFFFFFFu, acc, 0 ), rEven = __shfl_sync( 0xFFFFFFFFu, acc, 1 );
		const float lOdd = __shfl_sync( 0xFFFFFFFFu, acc, 2 ), rOdd = __shfl_sync( 0xFFFFFFFFu, acc, 3 );
		if( lane == 0 ) out[ seg ] = wsp::speakerDecide( lEven, rEven, lOdd, rOdd );
	}
	cudaError_t chunkSpeakers( const SpeakerJob* jobs, int32_t* out, int n, cudaStream_t s )
	{
		if( n < 1 ) return cudaErrorInvalidValue;
		speaker_kernel<<<( n + SPK_WARPS - 1 ) / SPK_WARPS, SPK_WARPS * 32, 0, s>>>( jobs, out, n );
		return cudaGetLastError();
	}

	// ---------------------------------------------------------------------------------------------------------------
	// LayerNorm (eps 1e-5 inside the sqrt) + affine -> f16: one warp per row, the row stays in registers.
	// Oracle: ggml_compute_forward_norm_f32 (ggml.c:4098-4156) then mul/add with gamma/beta (whisper.cpp:1190-1198);
	// the f16 rounding is the activation conversion the next mul_mat performs (ggml.c:4592-4603).
	constexpr int LN_MAX_V4 = 10;   // d <= 1280

	__global__ void __launch_bounds__( 256 )
		layernorm_f16_kernel( const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta, __half* __restrict__ out, int rows, int d )
	{
		const int row = blockIdx.x * ( blockDim.x >> 5 ) + ( threadIdx.x >> 5 );
		if( row >= rows ) return;
		const int lane = threadIdx.x & 31;
		const int n4 = d >> 7;   // float4 per lane (d multiple of 128)
		const float4* xr = reinterpret_cast<const float4*>( x + (size_t)row * d );
		float4 v[ LN_MAX_V4 ];
		float sum = 0.0f;
#pragma unroll
		for( int i = 0; i < LN_MAX_V4; i++ )
			if( i < n4 )
			{
				v[ i ] = xr[ i * 32 + lane ];
				sum += v[ i ].x + v[ i ].y + v[ i ].z + v[ i ].w;
			}
		const float mean = ptx::warp_sum( sum ) / (float)d;
		float sq = 0.0f;
#pragma unroll
		for( int i = 0; i < LN_MAX_V4; i++ )
			if( i < n4 )
			{
				v[ i ].x -= mean; v[ i ].y -= mean; v[ i ].z -= mean; v[ i ].w -= mean;
				sq += v[ i ].x * v[ i ].x + v[ i ].y * v[ i ].y + v[ i ].z * v[ i ].z + v[ i ].w * v[ i ].w;
			}
		const float rstd = 1.0f / sqrtf( ptx::warp_sum( sq ) / (float)d + 1e-5f );
		const float4* g4 = reinterpret_cast<const float4*>( gamma );
		const float4* b4 = reinterpret_cast<const float4*>( beta );
		uint2* o2 = reinterpret_cast<uint2*>( out + (size_t)row * d );
#pragma unroll
		for( int i = 0; i < LN_MAX_V4; i++ )
			if( i < n4 )
			{
				const float4 g = g4[ i * 32 + lane ];
				const float4 b = b4[ i * 32 + lane ];
				__half2 h0 = __floats2half2_rn( v[ i ].x * rstd * g.x + b.x, v[ i ].y * rstd * g.y + b.y );
				__half2 h1 = __floats2half2_rn( v[ i ].z * rstd * g.z + b.z, v[ i ].w * rstd * g.w + b.w );
				uint2 u;
				u.x = *reinterpret_cast<uint32_t*>( &h0 );
				u.y = *reinterpret_cast<uint32_t*>( &h1 );
				o2[ i * 32 + lane ] = u;
			}
	}
	cudaError_t layerNormF16( const float* x, const float* gamma, const float* beta, __half* out, int rows, int d, cudaStream_t s )
	{
		if( ( d & 127 ) != 0 || d > LN_MAX_V4 * 128 ) return cudaErrorInvalidValue;
		const int warpsPerBlock = 8;
		layernorm_f16_kernel<<<( rows + warpsPerBlock - 1 ) / warpsPerBlock, warpsPerBlock * 32, 0, s>>>( x, gamma, beta, out, rows, d );
		return cudaGetLastError();
	}

	// ---------------------------------------------------------------------------------------------------------------
	// token + positional embedding (whisper.cpp:1536-1548: ggml_get_rows of the f16 embedding, f32 add)
	__global__ void embed_kernel( const __half* __restrict__ te, const float* __restrict__ pe, const int* __restrict__ tokens, const int* __restrict__ dNPast,
		float* __restrict__ x, int N, int d )
	{
		ptx::pdl_launch_dependents();
		ptx::pdl_wait();
		const int col = blockIdx.x;   // b*N + i
		const int i = col % N;
		const int tok = tokens[ col ];
		const int pos = *dNPast + i;
		const __half* src = te + (size_t)tok * d;
		const float* p = pe + (size_t)pos * d;
		float* dst = x + (size_t)col * d;
		for( int e = threadIdx.x; e < d; e += blockDim.x )
			dst[ e ] = __half2float( src[ e ] ) + p[ e ];
	}
	cudaError_t embedTokens( const __half* te, const float* pe, const int* tokens, const int* dNPast, float* x, int B, int N, int d, cudaStream_t s )
	{
		return launchPdl( embed_kernel, dim3( B * N ), dim3( 128 ), 0, s, te, pe, tokens, dNPast, x, N, d );
	}

	__global__ void set_ints_kernel( int* dst, int a, int b ) { dst[ 0 ] = a; dst[ 1 ] = b; }
	cudaError_t setInts( int* dst, int a, int b, cudaStream_t s )
	{
		set_ints_kernel<<<1, 1, 0, s>>>( dst, a, b );
		return cudaGetLastError();
	}
}

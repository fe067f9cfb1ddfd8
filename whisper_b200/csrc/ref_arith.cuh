// The reference's CPU arithmetic that every decoder kernel has to reproduce operation by operation (DESIGN.md §2), and the
// attention pieces built on it.  One definition, shared by the per-op kernels (kernels_decode.cu), the dataflow step kernel
// (decode_flow.cu) and round 1's barrier kernel (decode_mega.cu).
#pragma once
#include "ptx.cuh"
#include <cuda_fp16.h>
#include <math.h>

namespace kern
{
	// reference thread counts whose V^T*P split the decoder reproduces (wsp_set_reference_threads)
	constexpr int kMaxRefThreads = 16;

	// V^T * P with the reference's arithmetic.  In the CPU reference this product takes ggml's "mad" path because V is read
	// transposed (ggml.c:4680-4722): thread ith of nth owns the contiguous key range [ith*dc, (ith+1)*dc), dc = ceil(nkv/nth), and
	// accumulates y[e] = f16( fma( V[j][e], P[j], f32(y[e]) ) ) key by key in an f16 work row (ggml_vec_mad_f16, ggml.c:871-893, with
	// AVX2/F16C: f32 FMA then a round-to-nearest-even store to f16); FINALIZE adds the nth partial rows in f32 in thread order
	// (ggml.c:4613-4640).  With ~1500 keys the f16 running sum swamps the small P[j]*V increments, so the result depends on nth and
	// differs from the exact sum by several percent — that IS the reference's output, and the greedy token sequence depends on it.
	// `refThreads` reproduces it for a given thread count (the reference's default is min(4, cores), whisper.cpp:2605; its own
	// compat shader also "fakes 4 CPU threads", ComputeShaders/mulMatMadMain.hlsl:107).
	__device__ __forceinline__ float pvChainF16( const float* __restrict__ sp, const __half* __restrict__ v, size_t vStride, int j0, int j1 )
	{
		float y = 0.0f;   // always exactly representable in f16
		int j = j0;
		for( ; j + 4 <= j1; j += 4 )
		{
			const float x0 = __half2float( v[ (size_t)j * vStride ] );
			const float x1 = __half2float( v[ (size_t)( j + 1 ) * vStride ] );
			const float x2 = __half2float( v[ (size_t)( j + 2 ) * vStride ] );
			const float x3 = __half2float( v[ (size_t)( j + 3 ) * vStride ] );
			y = __half2float( __float2half_rn( __fmaf_rn( x0, sp[ j ], y ) ) );
			y = __half2float( __float2half_rn( __fmaf_rn( x1, sp[ j + 1 ], y ) ) );
			y = __half2float( __float2half_rn( __fmaf_rn( x2, sp[ j + 2 ], y ) ) );
			y = __half2float( __float2half_rn( __fmaf_rn( x3, sp[ j + 3 ], y ) ) );
		}
		for( ; j < j1; j++ )
			y = __half2float( __float2half_rn( __fmaf_rn( __half2float( v[ (size_t)j * vStride ] ), sp[ j ], y ) ) );
		return y;
	}
	// exp through the reference's f16 table semantics: f32( f16( exp( f16(x) ) ) )  (ggml.c:5075-5077, table :1372-1383)
	__device__ __forceinline__ float expF16Table( float x )
	{
		return __half2float( __float2half_rn( expf( __half2float( __float2half_rn( x ) ) ) ) );
	}

	// ---------------------------------------------------------------------------------------------------------------
	// Attention over one (chunk, head, query) by 256 threads (8 warps): the shape of every decoder attention kernel.
	constexpr int kAttnThreads = 256;
	constexpr int kAttnWarps = kAttnThreads / 32;

	__device__ __forceinline__ void ctaSync() { __syncthreads(); }

	// softmax over sp[0, n) exactly as the reference does it: max in f32, e = f16-table exp, sum, scale by 1/sum (ggml.c:5026-5095).
	// lmax: the caller's running maximum of the scores it wrote.  sred: 16 floats.  SYNC: the barrier of the 256 calling threads.
	template<void ( *SYNC )()>
	__device__ __forceinline__ void softmaxRow( float* sp, int n, float lmax, float* sred, int tid, int warp, int lane )
	{
		lmax = ptx::warp_max( lmax );
		if( lane == 0 ) sred[ warp ] = lmax;
		SYNC();
		float mx = sred[ 0 ];
		for( int w = 1; w < kAttnWarps; w++ ) mx = fmaxf( mx, sred[ w ] );
		float lsum = 0.0f;
		for( int j = tid; j < n; j += kAttnThreads )
		{
			const float e = expF16Table( sp[ j ] - mx );
			sp[ j ] = e;
			lsum += e;
		}
		lsum = ptx::warp_sum( lsum );
		if( lane == 0 ) sred[ kAttnWarps + warp ] = lsum;   // (the maxima in sred[0..8) may still be being read)
		SYNC();
		float tot = 0.0f;
		for( int w = 0; w < kAttnWarps; w++ ) tot += sred[ kAttnWarps + w ];
		const float inv = 1.0f / tot;
		for( int j = tid; j < n; j += kAttnThreads ) sp[ j ] *= inv;
		SYNC();
	}

	// out[0, 64) = V^T * P for one query as `parts` reference threads compute it (pvChainF16): part k chains keys
	// [k * dc, (k + 1) * dc) clipped to the nkv keys the query sees (masked keys contribute 0), then the partial rows are added in f32
	// in part order.  sv: the V rows in shared memory, 64 halves apart; so: kMaxRefThreads * 64 floats.  Called by all 256 threads.
	__device__ __forceinline__ void pvSplitF16( const float* sp, const __half* sv, int nkv, int parts, int dc, float* so, __half* out, int tid )
	{
		for( int idx = tid; idx < parts * 64; idx += kAttnThreads )
		{
			const int part = idx >> 6, e = idx & 63;
			const int j0 = min( part * dc, nkv ), j1 = min( ( part + 1 ) * dc, nkv );
			so[ idx ] = pvChainF16( sp, sv + e, 64, j0, j1 );
		}
		__syncthreads();
		if( tid < 64 )
		{
			float acc = so[ tid ];
			for( int k = 1; k < parts; k++ ) acc += so[ k * 64 + tid ];
			out[ tid ] = __float2half_rn( acc );
		}
	}

	// Scores q . K[j] of n keys with K (128-byte f16 rows) streamed from global memory through registers: a warp covers 4 key rows
	// per load instruction (512 contiguous bytes, lane = (row in group, 16-byte piece)), kKBatch loads in flight per lane.
	// kStreamPrefetch fills the first register batch (it may be issued long before the scores are needed); kStreamScores consumes
	// it, refills it batch by batch, writes sp[0, n) and returns the lane's running maximum.  qf: the query elements of the lane's piece.
	constexpr int kKBatch = 12;
	constexpr int kKStep = kAttnWarps * 4;   // key rows per load instruction of the CTA
	__device__ __forceinline__ void kStreamLoad( uint4 ( &u )[ kKBatch ], const uint4* K4, int n, int jb, int lane )
	{
#pragma unroll
		for( int k = 0; k < kKBatch; k++ )
		{
			const int j = jb + k * kKStep;
			u[ k ] = j < n ? K4[ (size_t)j * 8 + ( lane & 7 ) ] : make_uint4( 0, 0, 0, 0 );
		}
	}
	__device__ __forceinline__ void kStreamPrefetch( uint4 ( &u )[ kKBatch ], const uint4* K4, int n, int warp, int lane )
	{
		kStreamLoad( u, K4, n, warp * 4 + ( lane >> 3 ), lane );
	}
	__device__ __forceinline__ float kStreamScores( uint4 ( &u )[ kKBatch ], const uint4* K4, int n, const float ( &qf )[ 8 ], float* sp, int warp, int lane )
	{
		float lmax = -INFINITY;
		// the loop runs while the WARP's first row is a key, so that every lane reaches the shuffles below (a lane's own row may
		// already be past n: with n = 1, only lanes 0..7 of warp 0 have one)
		for( int jw = warp * 4; jw < n; jw += kKStep * kKBatch )
		{
			const int jb = jw + ( lane >> 3 );
#pragma unroll
			for( int k = 0; k < kKBatch; k++ )
			{
				const int j = jb + k * kKStep;
				const __half2* h2 = reinterpret_cast<const __half2*>( &u[ k ] );
				float s = 0.0f;
#pragma unroll
				for( int e = 0; e < 4; e++ )
				{
					const float2 f = __half22float2( h2[ e ] );
					s += f.x * qf[ e * 2 ] + f.y * qf[ e * 2 + 1 ];
				}
				s += __shfl_xor_sync( 0xffffffffu, s, 1 );
				s += __shfl_xor_sync( 0xffffffffu, s, 2 );
				s += __shfl_xor_sync( 0xffffffffu, s, 4 );
				if( j < n )
				{
					if( ( lane & 7 ) == 0 ) sp[ j ] = s;
					lmax = fmaxf( lmax, s );
				}
			}
			if( jw + kKStep * kKBatch < n ) kStreamLoad( u, K4, n, jb + kKStep * kKBatch, lane );
		}
		return lmax;
	}
}

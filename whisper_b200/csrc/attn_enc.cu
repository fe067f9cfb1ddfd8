// Fused flash attention for the Whisper encoder on sm_90a (non-causal, head dim 64, T = audio_ctx: 1500 unless overridden).
//
// Replaces flashAttention.hlsl / the mulMatTiled -> softMax -> mulMatTiled chain the reference actually runs
// (Whisper/ML/Context.ops.cpp:194-227) and the CPU oracle's ggml_compute_forward_flash_attn_f16 (Whisper/source/ggml.c:5912-6097):
//   S = (K q) / sqrt(64)  (f16 x f16 -> f32),  P = softmax(S),  P rounded to f16,  O = V^T P  (f16 x f16 -> f32).
// Here: one CTA = 128 queries of one (chunk, head), two warpgroups of 64 queries each; K / V^T tiles of 128 keys arrive by TMA,
// double-buffered, the loads of tile j+2 issued as soon as tile j is consumed.  S = Q K^T is wgmma with A and B in shared memory
// and the scores in registers; the online softmax runs on the accumulator fragments (a row's 128 scores are spread over the four
// threads of a quad: two shuffles per reduction), and P is converted in registers straight into the A fragments of O += P V
// (wgmma with A from registers), so P never goes through shared memory.  O stays in registers and is rescaled when the row maximum
// grows.  Two CTAs co-reside per SM (81 KB smem each), so one CTA's softmax overlaps the other's MMAs.
//
// Rounding points kept from the oracle: Q, K, V and P are f16, all accumulation is f32.  Deliberate difference: exp is
// exp2f (not the oracle's f16 exp LUT, ggml.c:6065-6067) and P is rounded before the 1/sum normalisation (the oracle rounds after, :6082).
#include "attn_enc.cuh"
#include "per_device.h"
#include "ptx.cuh"

namespace attn
{
	constexpr int TQ = 128;      // queries per CTA (two warpgroups of 64)
	constexpr int TK = 128;      // keys per tile
	constexpr int HD = 64;       // head dim
	constexpr int SQ_BYTES = TQ * HD * 2;         // 16 KB
	constexpr int SK_BYTES = TK * HD * 2;         // 16 KB per buffer
	constexpr int SV_BYTES = HD * TK * 2;         // 16 KB per buffer, two [64][64] sub-tiles
	constexpr int SMEM_BYTES = SQ_BYTES + 2 * SK_BYTES + 2 * SV_BYTES + 128 + 1024;

	// 2^x on the MUFU pipe without exp2f's range-reduction wrapper (x <= 0 here; results below 2^-126 may flush to zero, far below
	// the f16 P that is kept).
	__device__ __forceinline__ float ex2Approx( float x )
	{
		float y;
		asm( "ex2.approx.ftz.f32 %0, %1;" : "=f"( y ) : "f"( x ) );
		return y;
	}
	__device__ __forceinline__ uint32_t packHalf2( float lo, float hi )
	{
		__half2 h = __floats2half2_rn( lo, hi );
		return *reinterpret_cast<uint32_t*>( &h );
	}
	__device__ __forceinline__ float quadMax( float v )
	{
		v = fmaxf( v, __shfl_xor_sync( 0xffffffffu, v, 1 ) );
		return fmaxf( v, __shfl_xor_sync( 0xffffffffu, v, 2 ) );
	}
	__device__ __forceinline__ float quadSum( float v )
	{
		v += __shfl_xor_sync( 0xffffffffu, v, 1 );
		return v + __shfl_xor_sync( 0xffffffffu, v, 2 );
	}

	__global__ void __launch_bounds__( 256, 2 )
		attn_enc_kernel( const __grid_constant__ CUtensorMap mapQ, const __grid_constant__ CUtensorMap mapK, const __grid_constant__ CUtensorMap mapVt, EncParams p )
	{
		extern __shared__ uint8_t smem_raw[];
		uint8_t* smem = reinterpret_cast<uint8_t*>( ( reinterpret_cast<uintptr_t>( smem_raw ) + 1023 ) & ~(uintptr_t)1023 );
		uint8_t* sQ = smem;
		uint8_t* sK = sQ + SQ_BYTES;                  // [2]
		uint8_t* sV = sK + 2 * SK_BYTES;              // [2]
		uint64_t* bars = reinterpret_cast<uint64_t*>( sV + 2 * SV_BYTES );
		uint64_t* bar_q = bars + 0;
		uint64_t* bar_k = bars + 1;                   // [2]: one per K buffer
		uint64_t* bar_v = bars + 3;                   // [2]: one per V^T buffer

		const int tid = threadIdx.x;
		const int lane = tid & 31;
		const int wg = tid >> 7;                      // warpgroup: queries [64 wg, 64 wg + 64) of the tile
		const int wq = ( tid >> 5 ) & 3;
		const int q0 = blockIdx.x * TQ;
		const int bh = blockIdx.y;
		const int nkv = ( p.T + TK - 1 ) / TK;

		auto loadKV = [ & ]( int j ) {
			const int buf = j & 1;
			ptx::mbar_expect_tx( bar_k + buf, SK_BYTES );
			ptx::tma_load_2d( sK + buf * SK_BYTES, &mapK, bar_k + buf, 0, bh * p.T + j * TK );
			ptx::mbar_expect_tx( bar_v + buf, SV_BYTES );
			ptx::tma_load_2d( sV + buf * SV_BYTES, &mapVt, bar_v + buf, j * TK, bh * HD );
			ptx::tma_load_2d( sV + buf * SV_BYTES + SV_BYTES / 2, &mapVt, bar_v + buf, j * TK + 64, bh * HD );
		};
		if( tid == 0 )
		{
			ptx::prefetch_tensormap( &mapQ );
			ptx::prefetch_tensormap( &mapK );
			ptx::prefetch_tensormap( &mapVt );
			for( int i = 0; i < 5; i++ )
				ptx::mbar_init( &bars[ i ], 1 );
			ptx::fence_barrier_init();
			ptx::mbar_expect_tx( bar_q, SQ_BYTES );
			ptx::tma_load_2d( sQ, &mapQ, bar_q, 0, bh * p.T + q0 );
			loadKV( 0 );
			if( nkv > 1 ) loadKV( 1 );
		}
		__syncthreads();

		const float c = p.scale_log2;
		const int qd = lane & 3;                      // column pair 2qd of every 8-column block
		float o[ HD / 2 ];                            // O rows (r0, r0 + 8): o[4n + 0/1] row r0, o[4n + 2/3] row r0 + 8, columns 8n + 2qd
#pragma unroll
		for( int i = 0; i < HD / 2; i++ ) o[ i ] = 0.0f;
		float mRun[ 2 ] = { -INFINITY, -INFINITY };   // running row maxima (raw scores)
		float lPart[ 2 ] = { 0.0f, 0.0f };            // this thread's share of the row sums, relative to mRun
		const uint64_t dq = ptx::gmma_desc_sw128( ptx::smem_u32( sQ + wg * 64 * 128 ) );
		ptx::mbar_wait( bar_q, 0 );

		for( int j = 0; j < nkv; j++ )
		{
			const int buf = j & 1;
			const uint32_t ph = (uint32_t)( ( j >> 1 ) & 1 );
			ptx::mbar_wait( bar_k + buf, ph );
			float s[ TK / 2 ];
			{
				const uint64_t dk = ptx::gmma_desc_sw128( ptx::smem_u32( sK + buf * SK_BYTES ) );
				ptx::wgmma_fence();
#pragma unroll
				for( int k = 0; k < HD / 16; k++ )
					ptx::wgmma_m64n128k16_ss( s, dq + (uint64_t)( k * 2 ), dk + (uint64_t)( k * 2 ), k != 0 ? 1u : 0u );
				ptx::wgmma_commit();
				ptx::wgmma_wait<0>();
				ptx::fence_regs<TK / 2>( s );
			}

			// columns >= nvalid are padding / the next head's rows (only in the last tile of a head)
			const int nvalid = p.T - j * TK;
			if( nvalid < TK )
			{
#pragma unroll
				for( int i = 0; i < TK / 2; i++ )
					if( 8 * ( i >> 2 ) + 2 * qd + ( i & 1 ) >= nvalid ) s[ i ] = -INFINITY;
			}
			float mx[ 2 ] = { -INFINITY, -INFINITY };
#pragma unroll
			for( int i = 0; i < TK / 2; i++ ) mx[ ( i >> 1 ) & 1 ] = fmaxf( mx[ ( i >> 1 ) & 1 ], s[ i ] );
			float f[ 2 ], nmc[ 2 ];
#pragma unroll
			for( int r = 0; r < 2; r++ )
			{
				const float mNew = fmaxf( mRun[ r ], quadMax( mx[ r ] ) );
				f[ r ] = ex2Approx( ( mRun[ r ] - mNew ) * c );
				mRun[ r ] = mNew;
				nmc[ r ] = -mNew * c;
				lPart[ r ] *= f[ r ];
			}
#pragma unroll
			for( int i = 0; i < HD / 2; i++ ) o[ i ] *= f[ ( i >> 1 ) & 1 ];

			// probabilities -> f16 A fragments: k-slice kk (keys 16kk..16kk+15) is score blocks 2kk and 2kk+1
			uint32_t pa[ TK / 4 ];
#pragma unroll
			for( int i = 0; i < TK / 2; i += 2 )
			{
				const int r = ( i >> 1 ) & 1;
				const float e0 = ex2Approx( fmaf( s[ i ], c, nmc[ r ] ) );
				const float e1 = ex2Approx( fmaf( s[ i + 1 ], c, nmc[ r ] ) );
				lPart[ r ] += e0 + e1;
				pa[ i >> 1 ] = packHalf2( e0, e1 );
			}

			ptx::mbar_wait( bar_v + buf, ph );
			{
				const uint32_t sv = ptx::smem_u32( sV + buf * SV_BYTES );
				ptx::fence_regs<HD / 2>( o );
				ptx::wgmma_fence();
#pragma unroll
				for( int kk = 0; kk < TK / 16; kk++ )
				{
					const uint64_t dv = ptx::gmma_desc_sw128( sv + (uint32_t)( ( kk >> 2 ) * ( SV_BYTES / 2 ) ) ) + (uint64_t)( ( kk & 3 ) * 2 );
					ptx::wgmma_m64n64k16_rs( o, pa + kk * 4, dv, 1u );
				}
				ptx::wgmma_commit();
				ptx::wgmma_wait<0>();
				ptx::fence_regs<HD / 2>( o );
			}

			// both warpgroups are done with buffer `buf`: refill it with tile j+2
			__syncthreads();
			if( tid == 0 && j + 2 < nkv ) loadKV( j + 2 );
		}

		// O / l as f16, merged-heads layout [chunk][t][h*64 + e]
		const int b = bh / p.H;
		const int h = bh - b * p.H;
#pragma unroll
		for( int r = 0; r < 2; r++ )
		{
			const int t = q0 + wg * 64 + wq * 16 + ( lane >> 2 ) + 8 * r;
			const float inv = 1.0f / quadSum( lPart[ r ] );
			if( t < p.T )
			{
				__half* dst = p.out + ( (size_t)b * p.T + t ) * p.d + h * HD + 2 * qd;
#pragma unroll
				for( int n = 0; n < HD / 8; n++ )
					*reinterpret_cast<uint32_t*>( dst + 8 * n ) = packHalf2( o[ 4 * n + 2 * r ] * inv, o[ 4 * n + 2 * r + 1 ] * inv );
			}
		}
	}

	cudaError_t launchEnc( const CUtensorMap& mapQ, const CUtensorMap& mapK, const CUtensorMap& mapVt, const EncParams& p, cudaStream_t stream )
	{
		static kern::PerDeviceMax attr;
		{
			cudaError_t e = attr.raise( SMEM_BYTES, []( size_t n ) { return cudaFuncSetAttribute( attn_enc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n ); } );
			if( e != cudaSuccess ) return e;
		}
		dim3 grid( ( p.T + TQ - 1 ) / TQ, p.nBH );
		attn_enc_kernel<<<grid, 256, SMEM_BYTES, stream>>>( mapQ, mapK, mapVt, p );
		return cudaGetLastError();
	}
}

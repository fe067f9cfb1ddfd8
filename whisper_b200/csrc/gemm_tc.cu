// wgmma + TMA GEMM for sm_90a — see gemm_tc.cuh for the design notes.
#include "gemm_tc.cuh"
#include "per_device.h"
#include <stdio.h>
#include <mutex>

namespace gemm
{
	// ---------------------------------------------------------------------------------------------------------------
	// epilogues: one thread owns output row `m` and 32 consecutive columns [n0, n0+32)
	__device__ __forceinline__ void store_f16x32( __half* dst, const float* v )
	{
		uint4* p = reinterpret_cast<uint4*>( dst );
#pragma unroll
		for( int i = 0; i < 4; i++ )
		{
			__half2 h0 = __floats2half2_rn( v[ i * 8 + 0 ], v[ i * 8 + 1 ] );
			__half2 h1 = __floats2half2_rn( v[ i * 8 + 2 ], v[ i * 8 + 3 ] );
			__half2 h2 = __floats2half2_rn( v[ i * 8 + 4 ], v[ i * 8 + 5 ] );
			__half2 h3 = __floats2half2_rn( v[ i * 8 + 6 ], v[ i * 8 + 7 ] );
			uint4 u;
			u.x = *reinterpret_cast<uint32_t*>( &h0 );
			u.y = *reinterpret_cast<uint32_t*>( &h1 );
			u.z = *reinterpret_cast<uint32_t*>( &h2 );
			u.w = *reinterpret_cast<uint32_t*>( &h3 );
			p[ i ] = u;
		}
	}

	// f16 outputs (EPI_CONV1, EPI_QKV, EPI_BIAS_GELU_F16, EPI_CROSSKV)
	template<int MODE>
	__device__ __forceinline__ void epilogue( const EpiParams& ep, int m, int n0, float* v )
	{
		if( n0 >= ep.N )
			return;
		if constexpr( MODE == EPI_CONV1 )
		{
			const int b = m / ep.rows_per_chunk;
			const int t = m - b * ep.rows_per_chunk;
			if( b >= ep.nchunks ) return;
			if( t >= ep.valid_per_chunk )
			{
				// the two rows past a chunk's frames are its trailing halo and the next chunk's leading one (conv2's zero padding):
				// rewritten on every call, because where they lie depends on audio_ctx (row 0, the first chunk's halo, never moves)
				if( m + 1 < ep.nchunks * ep.rows_per_chunk )
				{
#pragma unroll
					for( int i = 0; i < 32; i++ ) v[ i ] = 0.0f;
					store_f16x32( ep.out_a + (size_t)( m + 1 ) * ep.ld + n0, v );
				}
				return;
			}
#pragma unroll
			for( int i = 0; i < 32; i++ )
				v[ i ] = ptx::gelu_f16_semantics( v[ i ] + ep.bias[ n0 + i ] );
			store_f16x32( ep.out_a + (size_t)( m + 1 ) * ep.ld + n0, v );
		}
		else if constexpr( MODE == EPI_QKV )
		{
			if( m >= ep.M ) return;
			const int b = m / ep.T;
			const int t = m - b * ep.T;
			const int which = n0 / ep.d;
			const int nn = n0 - which * ep.d;
			const int h = nn >> 6;
			const int e = nn & 63;
#pragma unroll
			for( int i = 0; i < 32; i++ )
				v[ i ] += ep.bias[ n0 + i ];
			if( which < 2 )
			{
				__half* base = which == 0 ? ep.out_a : ep.out_b;
				store_f16x32( base + ( ( (size_t)b * ep.H + h ) * ep.T + t ) * 64 + e, v );
			}
			else
			{
				__half* dst = ep.out_c + ( ( (size_t)b * ep.H + h ) * 64 + e ) * ep.Tp + t;
#pragma unroll
				for( int i = 0; i < 32; i++ )
					dst[ (size_t)i * ep.Tp ] = __float2half_rn( v[ i ] );
				// V^T columns [T, T rounded up to 128) are read by the attention's last key tile: masked keys get P = 0, but 0 times a
				// stale Inf from an earlier, longer audio_ctx would be NaN.  Time step t clears columns T + t, T + t + T, ...
				const int tEnd = ( ep.T + 127 ) & ~127;
				for( int tz = ep.T + t; tz < tEnd; tz += ep.T )
				{
#pragma unroll
					for( int i = 0; i < 32; i++ )
						dst[ (size_t)i * ep.Tp + ( tz - t ) ] = __float2half_rn( 0.0f );
				}
			}
		}
		else if constexpr( MODE == EPI_BIAS_GELU_F16 )
		{
			if( m >= ep.M ) return;
#pragma unroll
			for( int i = 0; i < 32; i++ )
				v[ i ] = ptx::gelu_f16_semantics( v[ i ] + ep.bias[ n0 + i ] );
			store_f16x32( ep.out_a + (size_t)m * ep.ld + n0, v );
		}
		else if constexpr( MODE == EPI_CROSSKV )
		{
			if( m >= ep.M ) return;
			const int b = m / ep.T;
			const int t = m - b * ep.T;
			const int d2 = 2 * ep.d;
			const int l = n0 / d2;
			const int r = n0 - l * d2;
			const bool isV = r >= ep.d;
			const int nn = isV ? r - ep.d : r;
			const int h = nn >> 6;
			const int e = nn & 63;
			if( isV )
			{
#pragma unroll
				for( int i = 0; i < 32; i++ )
					v[ i ] += ep.bias[ n0 + i ];
			}
			else
			{
#pragma unroll
				for( int i = 0; i < 32; i++ )
					v[ i ] *= ep.scale;
			}
			__half* base = ( isV ? ep.out_b : ep.out_a ) + (size_t)l * ep.layer_stride;
			store_f16x32( base + ( ( (size_t)b * ep.H + h ) * ep.T + t ) * 64 + e, v );
		}
	}

	// ---------------------------------------------------------------------------------------------------------------
	constexpr int STG_LD = 72;   // staging row stride (floats): the float2 fragment stores of a half-warp hit 32 distinct banks

	// Coalesced epilogues.  Giving every thread one ROW of the tile makes each warp instruction touch 32 different rows (16 bytes
	// each): half of every 32-byte sector is wasted and a 128-byte line needs 8 separate instructions.  For f32 outputs the
	// 32 x 32 chunk is therefore read from the staging tile so that a thread owns one COLUMN: every load / store instruction of the
	// warp then covers 32 consecutive elements of one output row.  `w` points at the thread's column in the staging tile
	// (row stride STG_LD).  f32 outputs (EPI_F32, EPI_CONV2, EPI_BIAS_RESID).
	template<int MODE>
	__device__ __forceinline__ void epilogueT( const EpiParams& ep, int mBase, int n, const float* w )
	{
		if( n >= ep.N ) return;
		if constexpr( MODE == EPI_F32 )
		{
			const float b = ep.bias ? ep.bias[ n ] : 0.0f;
#pragma unroll
			for( int rr = 0; rr < 32; rr++ )
			{
				const int m = mBase + rr;
				if( m < ep.M ) ep.out_f32[ (size_t)m * ep.ld + n ] = w[ rr * STG_LD ] + b;
			}
		}
		else if constexpr( MODE == EPI_CONV2 )
		{
			const float b = ep.bias[ n ];
			const int cb0 = mBase / ep.rows_per_chunk;
			const int j0 = mBase - cb0 * ep.rows_per_chunk;
			// positional rows first, 16 at a time (loads must not be serialised behind the stores: pos and out_f32 are both float*)
#pragma unroll
			for( int h = 0; h < 32; h += 16 )
			{
				float pe[ 16 ];
				int j = j0 + h, cb = cb0;
				while( j >= ep.rows_per_chunk ) { j -= ep.rows_per_chunk; cb++; }
				{
					int jj = j;
#pragma unroll
					for( int rr = 0; rr < 16; rr++ )
					{
						pe[ rr ] = jj < ep.valid_per_chunk ? ep.pos[ (size_t)jj * ep.d + n ] : 0.0f;
						if( ++jj == ep.rows_per_chunk ) jj = 0;
					}
				}
#pragma unroll
				for( int rr = 0; rr < 16; rr++ )
				{
					if( cb < ep.nchunks && j < ep.valid_per_chunk )
						ep.out_f32[ ( (size_t)cb * ep.T + j ) * ep.ld + n ] = ptx::gelu_f16_semantics( w[ ( h + rr ) * STG_LD ] + b ) + pe[ rr ];
					if( ++j == ep.rows_per_chunk ) { j = 0; cb++; }
				}
			}
		}
		else if constexpr( MODE == EPI_BIAS_RESID )
		{
			// the residual column 16 rows at a time ahead of the stores: issued one by one behind each store, its L2 round trips and
			// not bandwidth would set the epilogue time
			const float b = ep.bias[ n ];
#pragma unroll
			for( int h = 0; h < 32; h += 16 )
			{
				float rs[ 16 ];
#pragma unroll
				for( int rr = 0; rr < 16; rr++ )
				{
					const int m = mBase + h + rr;
					rs[ rr ] = m < ep.M ? ep.resid[ (size_t)m * ep.ld + n ] : 0.0f;
				}
#pragma unroll
				for( int rr = 0; rr < 16; rr++ )
				{
					const int m = mBase + h + rr;
					if( m < ep.M ) ep.out_f32[ (size_t)m * ep.ld + n ] = w[ ( h + rr ) * STG_LD ] + b + rs[ rr ];
				}
			}
		}
	}

	// ---------------------------------------------------------------------------------------------------------------
	template<int BN, int STAGES>
	struct SmemLayout
	{
		static constexpr int A_BYTES = BM * BK * 2;
		static constexpr int B_BYTES = BN * BK * 2;
		static constexpr int STAGE_BYTES = A_BYTES + B_BYTES;
		static constexpr int STG_OFFSET = STAGES * STAGE_BYTES;
		static constexpr int STG_BYTES = 2 * 64 * STG_LD * 4;   // one 64 x 64 f32 staging tile per consumer warpgroup
		static constexpr int BAR_OFFSET = STG_OFFSET + STG_BYTES;
		static constexpr int TOTAL = BAR_OFFSET + 256 + 1024;   // + barriers + alignment slack
		static_assert( TOTAL <= 232448, "227 KB of shared memory per block on sm_90" );
	};

	template<int BN, int STAGES, int MODE, int AMODE>
	__global__ void __launch_bounds__( 384, 1 )
		gemm_tc_kernel( const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapA2, const __grid_constant__ CUtensorMap mapB,
			int M, int N, int K, int kTap, EpiParams ep )
	{
		using SL = SmemLayout<BN, STAGES>;
		extern __shared__ uint8_t smem_raw[];
		uint8_t* smem = reinterpret_cast<uint8_t*>( ( reinterpret_cast<uintptr_t>( smem_raw ) + 1023 ) & ~(uintptr_t)1023 );
		uint64_t* bar_full = reinterpret_cast<uint64_t*>( smem + SL::BAR_OFFSET );
		uint64_t* bar_empty = bar_full + STAGES;

		const int warp = threadIdx.x >> 5;
		const int lane = threadIdx.x & 31;
		const int wg = warp >> 2;

		const int num_m = ( M + BM - 1 ) / BM;
		const int num_n = ( N + BN - 1 ) / BN;
		const int num_tiles = num_m * num_n;
		const int num_kb = ( K + BK - 1 ) / BK;

		if( warp == 0 && lane == 0 )
		{
			ptx::prefetch_tensormap( &mapA );
			ptx::prefetch_tensormap( &mapB );
			if( AMODE == A_CONV_S2 ) ptx::prefetch_tensormap( &mapA2 );
			for( int s = 0; s < STAGES; s++ )
			{
				ptx::mbar_init( &bar_full[ s ], 1 );
				ptx::mbar_init( &bar_empty[ s ], 8 );   // one arrive per consumer warp
			}
			ptx::fence_barrier_init();
		}
		__syncthreads();

		if( wg == 0 )
		{
			// ===== TMA producer (one thread); the warpgroup hands its registers to the consumers =====
			asm volatile( "setmaxnreg.dec.sync.aligned.u32 40;" );
			if( warp == 0 && lane == 0 )
			{
				int stage = 0;
				uint32_t phase = 0;
				for( int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x )
				{
					const int m0 = ( tile / num_n ) * BM;
					const int n0 = ( tile % num_n ) * BN;
					for( int kb = 0; kb < num_kb; kb++ )
					{
						ptx::mbar_wait( &bar_empty[ stage ], phase ^ 1 );
						ptx::mbar_expect_tx( &bar_full[ stage ], SL::STAGE_BYTES );
						uint8_t* sa = smem + stage * SL::STAGE_BYTES;
						uint8_t* sb = sa + SL::A_BYTES;
						if constexpr( AMODE == A_PLAIN )
							ptx::tma_load_2d( sa, &mapA, &bar_full[ stage ], kb * BK, m0 );
						else
						{
							const int tap = kb / kTap;
							const int c0 = ( kb - tap * kTap ) * BK;
							if constexpr( AMODE == A_CONV_S1 )
								ptx::tma_load_2d( sa, &mapA, &bar_full[ stage ], c0, m0 + tap );
							else
							{
								if( tap == 1 )
									ptx::tma_load_2d( sa, &mapA2, &bar_full[ stage ], c0, m0 );
								else
									ptx::tma_load_2d( sa, &mapA, &bar_full[ stage ], c0, m0 + ( tap >> 1 ) );
							}
						}
						ptx::tma_load_2d( sb, &mapB, &bar_full[ stage ], kb * BK, n0 );
						if( ++stage == STAGES ) { stage = 0; phase ^= 1; }
					}
				}
			}
			return;
		}

		// ===== consumer warpgroups: warpgroup c owns rows [64c, 64c + 64) of the 128-row tile =====
		asm volatile( "setmaxnreg.inc.sync.aligned.u32 232;" );
		const int c = wg - 1;
		const int wq = warp & 3;   // warp inside the warpgroup
		float* stg = reinterpret_cast<float*>( smem + SL::STG_OFFSET ) + c * 64 * STG_LD;
		int stage = 0;
		uint32_t phase = 0;
		for( int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x )
		{
			const int m0 = ( tile / num_n ) * BM;
			const int n0 = ( tile % num_n ) * BN;
			float acc[ BN / 2 ];
			int prev = -1;
			for( int kb = 0; kb < num_kb; kb++ )
			{
				ptx::mbar_wait( &bar_full[ stage ], phase );
				const uint32_t sa = ptx::smem_u32( smem + stage * SL::STAGE_BYTES );
				const uint64_t da = ptx::gmma_desc_sw128( sa + (uint32_t)( c * 64 * 128 ) );
				const uint64_t db = ptx::gmma_desc_sw128( sa + SL::A_BYTES );
				ptx::fence_regs<BN / 2>( acc );
				ptx::wgmma_fence();
#pragma unroll
				for( int k = 0; k < BK / 16; k++ )
				{
					if constexpr( BN == 256 )
						ptx::wgmma_m64n256k16_ss( acc, da + (uint64_t)( k * 2 ), db + (uint64_t)( k * 2 ), ( kb | k ) != 0 ? 1u : 0u );
					else
						ptx::wgmma_m64n128k16_ss( acc, da + (uint64_t)( k * 2 ), db + (uint64_t)( k * 2 ), ( kb | k ) != 0 ? 1u : 0u );
				}
				ptx::wgmma_commit();
				ptx::fence_regs<BN / 2>( acc );
				// one k-block in flight: the previous one has finished reading its stage
				ptx::wgmma_wait<1>();
				if( prev >= 0 )
				{
					__syncwarp();
					if( lane == 0 ) ptx::mbar_arrive( &bar_empty[ prev ] );
				}
				prev = stage;
				if( ++stage == STAGES ) { stage = 0; phase ^= 1; }
			}
			ptx::wgmma_wait<0>();
			ptx::fence_regs<BN / 2>( acc );
			__syncwarp();
			if( lane == 0 ) ptx::mbar_arrive( &bar_empty[ prev ] );

			// epilogue: 64 columns at a time through the staging tile; warp wq then handles the 32 x 32 chunk
			// (rows 32 * (wq >> 1), columns 32 * (wq & 1)) of it with the epilogue of the old row- / column-per-thread layouts
			const int fr = wq * 16 + ( lane >> 2 );
			const int fc = ( lane & 3 ) * 2;
			const int mBase = m0 + c * 64 + ( wq >> 1 ) * 32;
			const int cOff = ( wq & 1 ) * 32;
#pragma unroll
			for( int piece = 0; piece < BN / 64; piece++ )
			{
				ptx::named_bar_sync( 1 + c, 128 );   // the previous piece has been read
#pragma unroll
				for( int j = 0; j < 8; j++ )
				{
					const float* a = acc + ( piece * 8 + j ) * 4;
					*reinterpret_cast<float2*>( stg + fr * STG_LD + j * 8 + fc ) = make_float2( a[ 0 ], a[ 1 ] );
					*reinterpret_cast<float2*>( stg + ( fr + 8 ) * STG_LD + j * 8 + fc ) = make_float2( a[ 2 ], a[ 3 ] );
				}
				ptx::named_bar_sync( 1 + c, 128 );
				const int nc = n0 + piece * 64 + cOff;
				// f32 outputs are read column-per-thread; f16 outputs keep the row-per-thread layout with 16-byte stores (2-byte scalar
				// stores, even though contiguous across the warp, are slower), and the V^T band of the QKV GEMM is stored transposed,
				// for which row-per-thread is the coalesced layout
				constexpr bool rowLayout = ( MODE == EPI_QKV ) || ( MODE == EPI_CONV1 ) || ( MODE == EPI_BIAS_GELU_F16 ) || ( MODE == EPI_CROSSKV );
				if constexpr( rowLayout )
				{
					float v[ 32 ];
					const float* src = stg + ( ( wq >> 1 ) * 32 + lane ) * STG_LD + cOff;
#pragma unroll
					for( int i = 0; i < 8; i++ )
					{
						const float4 t = reinterpret_cast<const float4*>( src )[ i ];
						v[ i * 4 + 0 ] = t.x; v[ i * 4 + 1 ] = t.y; v[ i * 4 + 2 ] = t.z; v[ i * 4 + 3 ] = t.w;
					}
					epilogue<MODE>( ep, mBase + lane, nc, v );
				}
				else
				{
					epilogueT<MODE>( ep, mBase, nc + lane, stg + ( ( wq >> 1 ) * 32 ) * STG_LD + cOff + lane );
				}
			}
		}
	}

	// ---------------------------------------------------------------------------------------------------------------
	// host side
	typedef CUresult ( *PFN_encodeTiled )( CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
		const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill );

	static PFN_encodeTiled getEncodeTiled()
	{
		static PFN_encodeTiled fn = nullptr;
		static std::once_flag once;
		std::call_once( once, []() {
			void* p = nullptr;
			cudaDriverEntryPointQueryResult qres;
			if( cudaGetDriverEntryPoint( "cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres ) == cudaSuccess && qres == cudaDriverEntryPointSuccess )
				fn = (PFN_encodeTiled)p;
		} );
		return fn;
	}

	bool makeMap2D( CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t rowStrideBytes, uint32_t boxRows )
	{
		PFN_encodeTiled enc = getEncodeTiled();
		if( !enc ) return false;
		cuuint64_t dims[ 2 ] = { inner, rows };
		cuuint64_t strides[ 1 ] = { rowStrideBytes };
		cuuint32_t box[ 2 ] = { (cuuint32_t)BK, boxRows };
		cuuint32_t estr[ 2 ] = { 1, 1 };
		CUresult r = enc( map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>( base ), dims, strides, box, estr,
			CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE );
		if( r != CUDA_SUCCESS )
		{
			fprintf( stderr, "whisper_b200: cuTensorMapEncodeTiled failed (%d): inner=%llu rows=%llu stride=%llu box=%u\n", (int)r,
				(unsigned long long)inner, (unsigned long long)rows, (unsigned long long)rowStrideBytes, boxRows );
			return false;
		}
		return true;
	}

	template<int BN, int STAGES, int MODE, int AMODE>
	static cudaError_t launchT( const Launch& L, int numSMs, cudaStream_t stream )
	{
		using SL = SmemLayout<BN, STAGES>;
		auto kfn = gemm_tc_kernel<BN, STAGES, MODE, AMODE>;
		static kern::PerDeviceMax attr;
		{
			cudaError_t e = attr.raise( SL::TOTAL, [ & ]( size_t n ) { return cudaFuncSetAttribute( kfn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n ); } );
			if( e != cudaSuccess ) return e;
		}
		const int num_tiles = ( ( L.M + BM - 1 ) / BM ) * ( ( L.N + BN - 1 ) / BN );
		const int grid = num_tiles < numSMs ? num_tiles : numSMs;
		if( grid <= 0 ) return cudaSuccess;
		kfn<<<grid, 384, SL::TOTAL, stream>>>( L.mapA, L.mapA2, L.mapB, L.M, L.N, L.K, L.kTap, L.ep );
		return cudaGetLastError();
	}

	template<int MODE, int AMODE>
	static cudaError_t launchBN( const Launch& L, int bn, int numSMs, cudaStream_t stream )
	{
		if( bn == 256 ) return launchT<256, 3, MODE, AMODE>( L, numSMs, stream );
		return launchT<128, 5, MODE, AMODE>( L, numSMs, stream );
	}

	cudaError_t launch( const Launch& L, EpiMode epi, AMode amode, int bn, int numSMs, cudaStream_t stream )
	{
		if( amode == A_CONV_S1 && epi == EPI_CONV1 ) return launchBN<EPI_CONV1, A_CONV_S1>( L, bn, numSMs, stream );
		if( amode == A_CONV_S2 && epi == EPI_CONV2 ) return launchBN<EPI_CONV2, A_CONV_S2>( L, bn, numSMs, stream );
		if( amode != A_PLAIN ) return cudaErrorInvalidValue;
		switch( epi )
		{
		case EPI_F32: return launchBN<EPI_F32, A_PLAIN>( L, bn, numSMs, stream );
		case EPI_QKV: return launchBN<EPI_QKV, A_PLAIN>( L, bn, numSMs, stream );
		case EPI_BIAS_RESID: return launchBN<EPI_BIAS_RESID, A_PLAIN>( L, bn, numSMs, stream );
		case EPI_BIAS_GELU_F16: return launchBN<EPI_BIAS_GELU_F16, A_PLAIN>( L, bn, numSMs, stream );
		case EPI_CROSSKV: return launchBN<EPI_CROSSKV, A_PLAIN>( L, bn, numSMs, stream );
		default: return cudaErrorInvalidValue;
		}
	}
}

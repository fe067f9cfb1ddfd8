// Decoder per-token kernels (weight/KV streaming, HBM-bound): skinny GEMM, self/cross attention over f16 KV, sampler.
#include "kernels.cuh"
#include "per_device.h"
#include "ptx.cuh"
#include "ref_arith.cuh"
#include <math.h>
#include <cooperative_groups.h>

namespace kern
{
	// ---------------------------------------------------------------------------------------------------------------
	// Skinny GEMM: out[col][n] = sum_k W[n][k] * x[col][k] for a handful of columns (decoder tokens x chunks).
	//
	// Replaces mulMatByRowTiled.hlsl (32 % of the reference's GPU time, ComputeShaders/mulMatByRowTiled.hlsl:42-169) and the N=1
	// case of ggml_compute_forward_mul_mat_f16_f32 (ggml.c:4447-4749).  The op is pure weight streaming, so the design goal is
	// HBM rate: each lane issues 16-byte loads covering 64 contiguous bytes of a weight row per quad, several in flight; the f16
	// activations (optionally LayerNorm-ed on the fly) sit in shared memory; products go through mma.sync.m16n8k16 (f16 x f16
	// -> f32, the oracle's arithmetic) because 8..16 columns exactly fill the n dimension and the tensor pipe is idle otherwise.
	// The k index is permuted identically for A and B fragments so that every fragment load is one 128-bit access.
	//
	// CTA = 16 weight rows x (up to 16 columns); 8 warps split K; cross-warp reduction through shared memory; fused epilogue.
	constexpr int SK_ROWS = 16;
	constexpr int SK_COLS = 16;      // columns per CTA pass (2 n-tiles of 8)
	constexpr int SK_WARPS = 8;
	constexpr int SK_PAD = 32;       // halves of padding per activation row: row stride = 64 (mod 128) bytes -> conflict-free LDS.128

	__global__ void __launch_bounds__( SK_WARPS * 32 )
		skinny_gemm_kernel( SkinnyArgs a )
	{
		extern __shared__ __align__( 16 ) uint8_t sk_smem[];
		const int K = a.K;
		const int rowStride = K + SK_PAD;   // halves
		__half* sx = reinterpret_cast<__half*>( sk_smem );                       // [SK_COLS][rowStride]
		float* red = reinterpret_cast<float*>( sx + (size_t)SK_COLS * rowStride ); // [SK_WARPS][SK_ROWS][SK_COLS]

		const int tid = threadIdx.x;
		const int warp = tid >> 5;
		const int lane = tid & 31;
		const int row0 = blockIdx.x * SK_ROWS;
		const int col0 = blockIdx.y * SK_COLS;
		const int ncols = min( SK_COLS, a.nCols - col0 );
		ptx::pdl_launch_dependents();

		// ---- weight stream: the first batch of 16-byte loads is issued before anything else, so HBM latency overlaps the
		//      activation staging below (weights do not depend on the previous kernel's output) ----
		const int g = lane >> 2, t = lane & 3;
		const int rA = min( row0 + g, a.nOut - 1 );
		const int rB = min( row0 + g + 8, a.nOut - 1 );
		const uint4* wA = reinterpret_cast<const uint4*>( a.W + (size_t)rA * K + 8 * t );
		const uint4* wB = reinterpret_cast<const uint4*>( a.W + (size_t)rB * K + 8 * t );
		const int steps = K / 32;
		constexpr int U = 8;
		uint4 va[ U ], vb[ U ];
#pragma unroll
		for( int u = 0; u < U; u++ )
		{
			const int st = warp + u * SK_WARPS;
			if( st < steps )
			{
				va[ u ] = ptx::ldg_stream( wA + st * 4 );   // 32 halves = 4 uint4 per step
				vb[ u ] = ptx::ldg_stream( wB + st * 4 );
			}
		}

		// everything below reads what the previous kernel wrote
		ptx::pdl_wait();

		// ---- stage activations as f16 (LayerNorm fused when gamma is given) ----
		for( int c = warp; c < SK_COLS; c += SK_WARPS )
		{
			__half* dst = sx + (size_t)c * rowStride;
			if( c >= ncols )
			{
				// unused columns of a tile that is computed must be finite; the second n-tile is skipped entirely when ncols <= 8
				if( c < 8 || ncols > 8 )
				{
					uint4* z4 = reinterpret_cast<uint4*>( dst );
					for( int k = lane; k < K / 8; k += 32 ) z4[ k ] = make_uint4( 0, 0, 0, 0 );
				}
				continue;
			}
			if( a.xF32 )
			{
				const float* src = a.xF32 + (size_t)( col0 + c ) * a.xStride;
				if( a.gamma )
				{
					// oracle: ggml_norm (ggml.c:4098-4156) + gamma/beta, then f16 conversion at the mul_mat (ggml.c:4592-4603).
					// The row (K = d <= 1280, multiple of 128) is loaded once into registers, all loads in flight together.
					constexpr int MAXV = 10;
					const int n4 = K >> 7;
					const float4* s4 = reinterpret_cast<const float4*>( src );
					float4 v[ MAXV ];
					float s = 0.0f;
#pragma unroll
					for( int q4 = 0; q4 < MAXV; q4++ )
						if( q4 < n4 )
						{
							v[ q4 ] = s4[ q4 * 32 + lane ];
							s += v[ q4 ].x + v[ q4 ].y + v[ q4 ].z + v[ q4 ].w;
						}
					const float mean = ptx::warp_sum( s ) / (float)K;
					float sq = 0.0f;
#pragma unroll
					for( int q4 = 0; q4 < MAXV; q4++ )
						if( q4 < n4 )
						{
							v[ q4 ].x -= mean; v[ q4 ].y -= mean; v[ q4 ].z -= mean; v[ q4 ].w -= mean;
							sq += v[ q4 ].x * v[ q4 ].x + v[ q4 ].y * v[ q4 ].y + v[ q4 ].z * v[ q4 ].z + v[ q4 ].w * v[ q4 ].w;
						}
					const float rstd = 1.0f / sqrtf( ptx::warp_sum( sq ) / (float)K + 1e-5f );
					const float4* g4 = reinterpret_cast<const float4*>( a.gamma );
					const float4* b4 = reinterpret_cast<const float4*>( a.beta );
					uint2* d2 = reinterpret_cast<uint2*>( dst );
#pragma unroll
					for( int q4 = 0; q4 < MAXV; q4++ )
						if( q4 < n4 )
						{
							const float4 g = g4[ q4 * 32 + lane ];
							const float4 bb = b4[ q4 * 32 + lane ];
							__half2 h0 = __floats2half2_rn( v[ q4 ].x * rstd * g.x + bb.x, v[ q4 ].y * rstd * g.y + bb.y );
							__half2 h1 = __floats2half2_rn( v[ q4 ].z * rstd * g.z + bb.z, v[ q4 ].w * rstd * g.w + bb.w );
							uint2 u;
							u.x = *reinterpret_cast<uint32_t*>( &h0 );
							u.y = *reinterpret_cast<uint32_t*>( &h1 );
							d2[ q4 * 32 + lane ] = u;
						}
				}
				else
					for( int k = lane; k < K; k += 32 ) dst[ k ] = __float2half_rn( src[ k ] );
			}
			else
			{
				const uint4* src = reinterpret_cast<const uint4*>( a.xF16 + (size_t)( col0 + c ) * a.xStride );
				uint4* d4 = reinterpret_cast<uint4*>( dst );
				for( int k = lane; k < K / 8; k += 32 ) d4[ k ] = src[ k ];
			}
		}
		__syncthreads();

		// ---- main loop: 32 k per step, steps interleaved across the 8 warps (8 warps x 64 B = 512 contiguous bytes per row) ----
		const __half* xb0 = sx + (size_t)g * rowStride + 8 * t;         // n-tile 0: column g
		const __half* xb1 = sx + (size_t)( g + 8 ) * rowStride + 8 * t; // n-tile 1: column g+8
		float acc0[ 4 ] = { 0, 0, 0, 0 }, acc1[ 4 ] = { 0, 0, 0, 0 };
		const bool twoTiles = ncols > 8;
		for( int s0 = warp; s0 < steps; )
		{
#pragma unroll
			for( int u = 0; u < U; u++ )
			{
				const int st = s0 + u * SK_WARPS;
				if( st < steps )
				{
					const uint4 x0 = *reinterpret_cast<const uint4*>( xb0 + st * 32 );
					ptx::mma_m16n8k16( acc0, va[ u ].x, vb[ u ].x, va[ u ].y, vb[ u ].y, x0.x, x0.y );
					ptx::mma_m16n8k16( acc0, va[ u ].z, vb[ u ].z, va[ u ].w, vb[ u ].w, x0.z, x0.w );
					if( twoTiles )
					{
						const uint4 x1 = *reinterpret_cast<const uint4*>( xb1 + st * 32 );
						ptx::mma_m16n8k16( acc1, va[ u ].x, vb[ u ].x, va[ u ].y, vb[ u ].y, x1.x, x1.y );
						ptx::mma_m16n8k16( acc1, va[ u ].z, vb[ u ].z, va[ u ].w, vb[ u ].w, x1.z, x1.w );
					}
				}
			}
			s0 += SK_WARPS * U;
			if( s0 < steps )
			{
#pragma unroll
				for( int u = 0; u < U; u++ )
				{
					const int st = s0 + u * SK_WARPS;
					if( st < steps )
					{
						va[ u ] = ptx::ldg_stream( wA + st * 4 );
						vb[ u ] = ptx::ldg_stream( wB + st * 4 );
					}
				}
			}
		}

		// ---- cross-warp reduction ----
		// c0,c1: (row g, cols 2t, 2t+1); c2,c3: (row g+8, same cols)
		float* my = red + (size_t)warp * SK_ROWS * SK_COLS;
		my[ g * SK_COLS + 2 * t + 0 ] = acc0[ 0 ];
		my[ g * SK_COLS + 2 * t + 1 ] = acc0[ 1 ];
		my[ ( g + 8 ) * SK_COLS + 2 * t + 0 ] = acc0[ 2 ];
		my[ ( g + 8 ) * SK_COLS + 2 * t + 1 ] = acc0[ 3 ];
		my[ g * SK_COLS + 8 + 2 * t + 0 ] = acc1[ 0 ];
		my[ g * SK_COLS + 8 + 2 * t + 1 ] = acc1[ 1 ];
		my[ ( g + 8 ) * SK_COLS + 8 + 2 * t + 0 ] = acc1[ 2 ];
		my[ ( g + 8 ) * SK_COLS + 8 + 2 * t + 1 ] = acc1[ 3 ];
		__syncthreads();

		// ---- epilogue: thread -> (col = tid / 16, row = tid % 16): consecutive threads write consecutive output features ----
		const int c = tid >> 4, r = tid & 15;
		const int n = row0 + r;
		if( c >= ncols || n >= a.nOut ) return;
		float v = 0.0f;
#pragma unroll
		for( int w = 0; w < SK_WARPS; w++ ) v += red[ ( (size_t)w * SK_ROWS + r ) * SK_COLS + c ];
		const int col = col0 + c;
		switch( a.epi )
		{
		case SK_QKV:
		{
			const int which = n / a.d;
			const int nn = n - which * a.d;
			if( which == 0 )
				a.outF32[ (size_t)col * a.ld + nn ] = ( v + a.bias[ n ] ) * a.scale;
			else
			{
				const int b = col / a.N, i = col - b * a.N;
				// self-KV cache rows are head-major [b][h][pos][64]: one head's rows are contiguous (bulk-copied by decode_flow.cu)
				const int pos = min( *a.dNPast + i, a.nTextCtx - 1 );
				const size_t off = ( ( (size_t)b * ( a.d >> 6 ) + ( nn >> 6 ) ) * a.nTextCtx + pos ) * 64 + ( nn & 63 );
				if( which == 1 ) a.kCache[ off ] = __float2half_rn( v * a.scale );
				else a.vCache[ off ] = __float2half_rn( v + a.bias[ n ] );
			}
			break;
		}
		case SK_BIAS_RESID:
		{
			float* p = a.outF32 + (size_t)col * a.ld + n;
			*p = v + a.bias[ n ] + *p;
			break;
		}
		case SK_Q_SCALE:
			a.outF32[ (size_t)col * a.ld + n ] = ( v + a.bias[ n ] ) * a.scale;
			break;
		case SK_GELU_F16:
			a.outF16[ (size_t)col * a.ld + n ] = __float2half_rn( ptx::gelu_f16_semantics( v + a.bias[ n ] ) );
			break;
		default:
			a.outF32[ (size_t)col * a.ld + n ] = v;
			break;
		}
	}

	static size_t skinnySmem( int K ) { return (size_t)SK_COLS * ( K + SK_PAD ) * sizeof( __half ) + (size_t)SK_WARPS * SK_ROWS * SK_COLS * sizeof( float ); }
	static PerDeviceMax g_skinnyAttr;
	static cudaError_t attnPrepare();
	cudaError_t prepare( int maxK )
	{
		cudaError_t ce = attnPrepare();
		if( ce != cudaSuccess ) return ce;
		return g_skinnyAttr.raise( skinnySmem( maxK ), []( size_t n ) { return cudaFuncSetAttribute( skinny_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n ); } );
	}
	cudaError_t skinnyGemm( const SkinnyArgs& a, cudaStream_t s )
	{
		if( a.K % 32 != 0 ) return cudaErrorInvalidValue;
		if( a.gamma && ( a.K % 128 != 0 || a.K > 1280 ) ) return cudaErrorInvalidValue;   // fused LayerNorm keeps the row in registers
		const size_t smem = skinnySmem( a.K );
		{
			cudaError_t e = prepare( a.K );
			if( e != cudaSuccess ) return e;
		}
		dim3 grid( ( a.nOut + SK_ROWS - 1 ) / SK_ROWS, ( a.nCols + SK_COLS - 1 ) / SK_COLS );
		return launchPdl( skinny_gemm_kernel, grid, dim3( SK_WARPS * 32 ), smem, s, a );
	}

	// ---------------------------------------------------------------------------------------------------------------
	// Decoder attention, one CTA per (chunk, head, query): softmax( q . K ) . V over an f16 memory [b][h][rows][64], with the
	// reference's arithmetic (ref_arith.cuh).
	//   SELF:  the self-KV cache, rows = n_text_ctx.  Causal: query i of chunk b sees keys [0, nPast + i]; the reference cuts its
	//          threads' key ranges from the keys of the whole call, min( nPast + N, n_text_ctx ).  Oracle: whisper.cpp:1616-1661 —
	//          K*Q (Q rounded to f16 by the mul_mat, ggml.c:4599), causal mask, softmax, V^T * P.
	//   cross: the encoder's cross-KV memory, rows = T, no mask.  Oracle: whisper.cpp:1688-1749 (K pre-scaled at encode time :1465).
	//          Its 2*T*d bytes per layer are the dominant per-chunk HBM traffic of a decode step (SURVEY.md §8 a15).
	// K streams through registers (kStreamScores, every access a coalesced 16-byte load); V streams into shared memory by cp.async
	// behind the scoring.  The cross memory was written by the encoder before the PDL chain, so both are requested before the
	// dependency wait; the self cache gets this call's rows from the preceding QKV GEMM, so nothing of it (nor n_past) is read before.
	template<bool SELF>
	constexpr int attnMaxRows = SELF ? 448 : 1500;

	template<bool SELF>
	__global__ void __launch_bounds__( kAttnThreads )
		attn_decode_kernel( const float* __restrict__ q, const __half* __restrict__ kMem, const __half* __restrict__ vMem, __half* __restrict__ out,
			int N, int H, int d, int rows, const int* __restrict__ dNPast, int refThreads )
	{
		extern __shared__ __align__( 16 ) uint8_t at_smem[];   // the V rows of this (chunk, head): rows x 128 bytes
		__shared__ float sp[ attnMaxRows<SELF> ];
		__shared__ float sred[ 16 ];
		__shared__ float so[ kMaxRefThreads * 64 ];
		const int bh = blockIdx.x;
		const int b = bh / H, h = bh - b * H;
		const int i = blockIdx.y;
		const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
		const int col = b * N + i;
		const uint4* K4 = reinterpret_cast<const uint4*>( kMem + (size_t)bh * rows * 64 );
		const uint4* V4 = reinterpret_cast<const uint4*>( vMem + (size_t)bh * rows * 64 );

		ptx::pdl_launch_dependents();
		if( SELF ) ptx::pdl_wait();
		const int nPast = SELF ? *dNPast : 0;
		const int nkv = SELF ? min( nPast + i + 1, rows ) : rows;      // keys visible to query i
		const int nkvAll = SELF ? min( nPast + N, rows ) : rows;     // keys the reference partitions over its threads
		{
			uint4* sv = reinterpret_cast<uint4*>( at_smem );
			for( int idx = tid; idx < nkv * 8; idx += kAttnThreads ) ptx::cp_async16( sv + idx, V4 + idx );
			ptx::cp_async_commit();
		}
		uint4 u[ kKBatch ];
		kStreamPrefetch( u, K4, nkv, warp, lane );
		if( !SELF ) ptx::pdl_wait();

		float qf[ 8 ];
#pragma unroll
		for( int e = 0; e < 8; e++ )
			qf[ e ] = __half2float( __float2half_rn( q[ (size_t)col * d + h * 64 + ( lane & 7 ) * 8 + e ] ) );
		const float lmax = kStreamScores( u, K4, nkv, qf, sp, warp, lane );
		softmaxRow<ctaSync>( sp, nkv, lmax, sred, tid, warp, lane );
		ptx::cp_async_wait_all();
		__syncthreads();
		pvSplitF16( sp, reinterpret_cast<const __half*>( at_smem ), nkv, refThreads, ( nkvAll + refThreads - 1 ) / refThreads, so,
			out + (size_t)col * d + h * 64, tid );
	}
	static PerDeviceMax g_attnAttr;
	static cudaError_t attnPrepare()
	{
		return g_attnAttr.raise( 1, []( size_t ) {
			cudaError_t e = cudaFuncSetAttribute( attn_decode_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, attnMaxRows<false> * 128 );
			if( e != cudaSuccess ) return e;
			return cudaFuncSetAttribute( attn_decode_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, attnMaxRows<true> * 128 );
		} );
	}
	template<bool SELF>
	static cudaError_t attnDecode( const float* q, const __half* kMem, const __half* vMem, __half* out, int B, int N, int H, int d, int rows, const int* dNPast, int refThreads, cudaStream_t s )
	{
		if( rows < 1 || rows > attnMaxRows<SELF> || refThreads < 1 || refThreads > kMaxRefThreads ) return cudaErrorInvalidValue;
		return launchPdl( attn_decode_kernel<SELF>, dim3( B * H, N ), dim3( kAttnThreads ), (size_t)rows * 128, s, q, kMem, vMem, out, N, H, d, rows, dNPast, refThreads );
	}
	cudaError_t selfAttnDecode( const float* q, const __half* kCache, const __half* vCache, __half* out, int B, int N, int H, int d, int nTextCtx, const int* dNPast, int refThreads, cudaStream_t s )
	{
		return attnDecode<true>( q, kCache, vCache, out, B, N, H, d, nTextCtx, dNPast, refThreads, s );
	}
	cudaError_t crossAttnDecode( const float* q, const __half* kMem, const __half* vMem, __half* out, int B, int N, int H, int d, int T, int refThreads, cudaStream_t s )
	{
		return attnDecode<false>( q, kMem, vMem, out, B, N, H, d, T, nullptr, refThreads, s );
	}

	// ---------------------------------------------------------------------------------------------------------------
	// softmax over the vocabulary + greedy sampling with the timestamp rules, one cluster of 4 CTAs per chunk.
	// Oracle: ggml_soft_max (ggml.c:5026-5095) then whisper_sample_best (whisper.cpp:1875-1964):
	//   max_tx = max p(text); if is_initial: p(ts > beg+100) = -inf; sum_ts, max_ts/tid over timestamp tokens;
	//   if sum_ts > max_tx or force_timestamp: p(text) = -inf;  top-4 by p; skip sot/solm/not among the first three.
	constexpr int SM_THREADS = 1024;

	// arg-max candidate; `tie`: another token has exactly the same probability (then the reference's pick depends on how
	// std::partial_sort happens to arrange equal keys, see emulatePartialSortCta)
	struct Top1 { float v; int i; int tie; };
	__device__ __forceinline__ Top1 better( Top1 a, Top1 b )
	{
		Top1 r = ( b.v > a.v || ( b.v == a.v && b.i < a.i ) ) ? b : a;
		if( a.v == b.v && a.i != b.i && a.v > -INFINITY ) r.tie = 1;
		return r;
	}

	// The reference ranks candidates with std::partial_sort( top 4 ) on (probability, id) pairs compared by probability only
	// (whisper.cpp:1932-1941).  With distinct probabilities that is "the largest"; with EXACT ties — typically a whole range of
	// probabilities that underflowed to 0 in the f16-table softmax — the winner is whatever libstdc++'s heap-select + sort-heap leaves
	// first.  emulatePartialSortCta replays that algorithm, statement by statement (bits/stl_heap.h: __push_heap, __adjust_heap,
	// __make_heap, __sort_heap; bits/stl_algo.h: __heap_select), and is only entered when a tie decides the token.
	struct ProbId { double v; int i; };
	__device__ void heapPush( ProbId* f, int hole, int top, ProbId val )
	{
		int parent = ( hole - 1 ) / 2;
		while( hole > top && f[ parent ].v > val.v )
		{
			f[ hole ] = f[ parent ];
			hole = parent;
			parent = ( hole - 1 ) / 2;
		}
		f[ hole ] = val;
	}
	__device__ void heapAdjust( ProbId* f, int hole, int len, ProbId val )
	{
		const int top = hole;
		int second = hole;
		while( second < ( len - 1 ) / 2 )
		{
			second = 2 * ( second + 1 );
			if( f[ second ].v > f[ second - 1 ].v ) second--;
			f[ hole ] = f[ second ];
			hole = second;
		}
		if( ( len & 1 ) == 0 && second == ( len - 2 ) / 2 )
		{
			second = 2 * ( second + 1 );
			f[ hole ] = f[ second - 1 ];
			hole = second - 1;
		}
		heapPush( f, hole, top, val );
	}

	// The whole CTA at work on one row.  std::__heap_select only ever moves an element into the heap that compares
	// strictly above the heap's root, and the root — the 4th largest value of the prefix processed so far — never decreases.  So
	// after thread 0 has run the exact algorithm over the first TIE_PRE elements, every later element that is not above the root
	// reached there (T1) can be dropped without changing a single heap operation: all warps filter their contiguous region of the row
	// against T1 (coalesced loads, ballot, survivors appended in index order to `scratch`), and thread 0 replays the exact algorithm
	// over the survivors only, which keeps degenerate rows (they tie at every step) cheap.  Called by every thread of the CTA; the result is valid
	// in thread 0.  scratch: nv + 32 * warps ints.
	constexpr int TIE_PRE = 1024;
	struct TieShared
	{
		float t1;
		int tie, maskText;
		int cnt[ 32 ];
	};
	__device__ Top1 emulatePartialSortCta( const float* probs, int nv, int beg, bool maskText, bool isInitial, int sot, int solm, int nott, int* scratch, TieShared& sh, int nThreads )
	{
		auto val = [ & ]( int i, float p ) -> double {
			if( ( maskText && i < beg ) || ( isInitial && i >= beg + 101 ) ) return -(double)INFINITY;
			return (double)p;
		};
		const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, nWarps = nThreads >> 5;
		const int pre = nv < TIE_PRE ? nv : TIE_PRE;
		ProbId f[ 4 ];
		if( tid == 0 )
		{
			for( int k = 0; k < 4; k++ ) f[ k ] = ProbId{ val( k, __ldcg( probs + k ) ), k };
			// __make_heap( first, first + 4 )
			for( int parent = ( 4 - 2 ) / 2;; parent-- )
			{
				const ProbId v = f[ parent ];
				heapAdjust( f, parent, 4, v );
				if( parent == 0 ) break;
			}
			// __heap_select: every later element that compares before the root replaces it
			for( int i = 4; i < pre; i++ )
			{
				const double v = val( i, __ldcg( probs + i ) );
				if( v > f[ 0 ].v ) heapAdjust( f, 0, 4, ProbId{ v, i } );
			}
			sh.t1 = (float)f[ 0 ].v;    // (the values are floats or -inf: exact)
		}
		__syncthreads();
		const float t1 = sh.t1;
		const int region = ( ( ( nv - pre + nWarps - 1 ) / nWarps + 31 ) / 32 ) * 32;
		{
			const int i0 = pre + warp * region, i1 = min( nv, i0 + region );
			int cnt = 0;
			for( int base = i0; base < i1; base += 512 )
			{
				float v[ 16 ];   // sixteen independent loads in flight per lane: the filter is bound by L2 latency, not by work
#pragma unroll
				for( int u = 0; u < 16; u++ )
				{
					const int i = base + u * 32 + lane;
					v[ u ] = i < i1 ? (float)val( i, __ldcg( probs + i ) ) : -INFINITY;
				}
#pragma unroll
				for( int u = 0; u < 16; u++ )
				{
					const bool keep = v[ u ] > t1;
					const unsigned m = __ballot_sync( 0xffffffffu, keep );
					if( keep ) scratch[ warp * region + cnt + __popc( m & ( ( 1u << lane ) - 1u ) ) ] = base + u * 32 + lane;
					cnt += __popc( m );
				}
			}
			if( lane == 0 ) sh.cnt[ warp ] = cnt;
		}
		__syncthreads();
		if( tid != 0 ) return Top1{ 0.0f, 0, 0 };
		for( int w = 0; w < nWarps; w++ )
		{
			const int* list = scratch + w * region;
			const int n = sh.cnt[ w ];
			for( int k = 0; k < n; k++ )
			{
				const int i = list[ k ];
				const double v = val( i, __ldcg( probs + i ) );
				if( v > f[ 0 ].v ) heapAdjust( f, 0, 4, ProbId{ v, i } );
			}
		}
		for( int last = 3; last >= 1; last-- )
		{
			const ProbId v = f[ last ];
			f[ last ] = f[ 0 ];
			heapAdjust( f, 0, last, v );
		}
		int res = 0;
		while( ( f[ res ].i == sot || f[ res ].i == solm || f[ res ].i == nott ) && res < 3 ) res++;
		return Top1{ (float)f[ res ].v, f[ res ].i, 0 };
	}

	__device__ Top1 blockArgmax( Top1 x, Top1* sbuf )
	{
		for( int o = 16; o > 0; o >>= 1 )
		{
			Top1 y;
			y.v = __shfl_xor_sync( 0xffffffffu, x.v, o );
			y.i = __shfl_xor_sync( 0xffffffffu, x.i, o );
			y.tie = __shfl_xor_sync( 0xffffffffu, x.tie, o );
			x = better( x, y );
		}
		__syncthreads();
		if( ( threadIdx.x & 31 ) == 0 ) sbuf[ threadIdx.x >> 5 ] = x;
		__syncthreads();
		Top1 r = sbuf[ 0 ];
		for( int w = 1; w < SM_THREADS / 32; w++ ) r = better( r, sbuf[ w ] );
		return r;
	}
	__device__ float blockMaxF( float v, float* sbuf )
	{
		v = ptx::warp_max( v );
		__syncthreads();
		if( ( threadIdx.x & 31 ) == 0 ) sbuf[ threadIdx.x >> 5 ] = v;
		__syncthreads();
		float r = sbuf[ 0 ];
		for( int w = 1; w < SM_THREADS / 32; w++ ) r = fmaxf( r, sbuf[ w ] );
		return r;
	}
	__device__ double blockSumD( double v, double* sbuf )
	{
		v = ptx::warp_sum( v );
		__syncthreads();
		if( ( threadIdx.x & 31 ) == 0 ) sbuf[ threadIdx.x >> 5 ] = v;
		__syncthreads();
		double r = 0.0;
		for( int w = 0; w < SM_THREADS / 32; w++ ) r += sbuf[ w ];
		return r;
	}

	// `pick` is the arg-max over the eligible, non-banned tokens (lowest id among equals).  If its probability is shared — by another
	// eligible token or by one of the banned ones — the reference's choice depends on std::partial_sort's handling of equal keys:
	// reproduce it exactly.  The whole probability row must be visible in global memory (it is: written before the last barrier).
	__device__ __forceinline__ bool needsTieEmulation( Top1 pick, const SampleArgs& a, const float* probsRow, bool maskText )
	{
		bool tie = pick.tie != 0;
		if( !tie && !maskText )
		{
			const int banned[ 3 ] = { a.tokenSot, a.tokenSolm, a.tokenNot };
			for( int k = 0; k < 3; k++ )
				if( banned[ k ] >= 0 && banned[ k ] < a.tokenBeg && __ldcg( probsRow + banned[ k ] ) == pick.v ) tie = true;
		}
		return tie;
	}
	// called by every thread of the CTA that finishes a row; `pick` and the result are thread 0's
	__device__ __forceinline__ Top1 resolveTies( Top1 pick, const SampleArgs& a, int b, bool maskText, bool isInitial, TieShared& sh )
	{
		const float* probsRow = a.probs + (size_t)b * a.nVocab;
		if( threadIdx.x == 0 ) sh.tie = needsTieEmulation( pick, a, probsRow, maskText ) ? 1 : 0;
		__syncthreads();
		if( !sh.tie ) return pick;
		const Top1 r = emulatePartialSortCta( probsRow, a.nVocab, a.tokenBeg, maskText, isInitial, a.tokenSot, a.tokenSolm, a.tokenNot,
			a.tieScratch + (size_t)b * ( a.nVocab + 32 * ( SM_THREADS / 32 ) ), sh, SM_THREADS );
		return threadIdx.x == 0 ? r : pick;
	}

	// One vocabulary row spread over a cluster of SC_CL CTAs: every CTA keeps its slice of the row in shared memory, the three
	// row-wide reductions go through distributed shared memory (each CTA publishes its partial, cluster barrier, everybody combines
	// the SC_CL partials in rank order).  One CTA per row would leave most SMs idle and keep only a short row in shared memory.
	struct ClusterPart
	{
		float mx, maxTx;
		double dsum, sumTs;
		Top1 bestTs, bestTx;
	};
	template<int SC_CL>
	__global__ void __launch_bounds__( SM_THREADS )
		sample_cluster_kernel( SampleArgs a )
	{
		namespace cg = cooperative_groups;
		cg::cluster_group cluster = cg::this_cluster();
		const unsigned rank = cluster.block_rank();
		__shared__ ClusterPart part;
		__shared__ float sf[ SM_THREADS / 32 ];
		__shared__ double sd[ SM_THREADS / 32 ];
		__shared__ Top1 st[ SM_THREADS / 32 ];
		extern __shared__ float sampleRow[];
		const int b = blockIdx.y;
		const int tid = threadIdx.x;
		const int nv = a.nVocab;
		const int per = ( nv + SC_CL - 1 ) / SC_CL;
		const int i0 = min( (int)rank * per, nv ), i1 = min( i0 + per, nv );
		const int n = i1 - i0;
		const float* lg = a.logits + (size_t)b * nv + i0;
		float* gpr = a.probs + (size_t)b * nv + i0;
		float* pr = sampleRow;
		const bool forceTs = a.dForceTs && a.dForceTs[ 0 ] != 0;
		const bool isInitial = a.dForceTs && a.dForceTs[ 1 ] != 0;

		float mx = -INFINITY;
		for( int i = tid; i < n; i += SM_THREADS )
		{
			const float v = __ldcg( lg + i );
			pr[ i ] = v;
			mx = fmaxf( mx, v );
		}
		mx = blockMaxF( mx, sf );
		if( tid == 0 ) part.mx = mx;
		cluster.sync();
		for( unsigned r = 0; r < SC_CL; r++ ) mx = fmaxf( mx, cluster.map_shared_rank( &part, r )->mx );

		double dsum = 0.0;
		for( int i = tid; i < n; i += SM_THREADS )
		{
			const float e = expF16Table( pr[ i ] - mx );
			pr[ i ] = e;
			dsum += (double)e;
		}
		dsum = blockSumD( dsum, sd );
		if( tid == 0 ) part.dsum = dsum;
		cluster.sync();
		double total = 0.0;   // the terms are f16 values: this double sum is exact, so the split does not change it
		for( unsigned r = 0; r < SC_CL; r++ ) total += cluster.map_shared_rank( &part, r )->dsum;
		const float inv = (float)( 1.0 / total );

		const int beg = a.tokenBeg;
		const int tsEnd = isInitial ? min( beg + 101, nv ) : nv;
		float maxTx = -1.0f;
		double sumTs = 0.0;
		Top1 bestTs = { -INFINITY, 0x7fffffff, 0 };
		Top1 bestTx = { -INFINITY, 0x7fffffff, 0 };
		for( int i = tid; i < n; i += SM_THREADS )
		{
			const float p = pr[ i ] * inv;
			gpr[ i ] = p;
			const int gi = i0 + i;
			if( gi < beg )
			{
				maxTx = fmaxf( maxTx, p );
				if( gi != a.tokenSot && gi != a.tokenSolm && gi != a.tokenNot ) bestTx = better( bestTx, Top1{ p, gi, 0 } );
			}
			else if( gi < tsEnd )
			{
				sumTs += (double)p;
				bestTs = better( bestTs, Top1{ p, gi, 0 } );
			}
		}
		maxTx = blockMaxF( maxTx, sf );
		sumTs = blockSumD( sumTs, sd );
		bestTs = blockArgmax( bestTs, st );
		bestTx = blockArgmax( bestTx, st );
		if( tid == 0 )
		{
			part.maxTx = maxTx; part.sumTs = sumTs; part.bestTs = bestTs; part.bestTx = bestTx;
		}
		cluster.sync();
		__shared__ TieShared tieSh;
		if( rank == 0 )
		{
			// the row is finished by the first CTA of its cluster: thread 0 combines the partials, all threads help if the top
			// probability is shared (resolveTies)
			Top1 pick = bestTs;
			if( tid == 0 )
			{
				for( unsigned r = 1; r < SC_CL; r++ )
				{
					const ClusterPart* q = cluster.map_shared_rank( &part, r );
					maxTx = fmaxf( maxTx, q->maxTx );
					sumTs += q->sumTs;
					bestTs = better( bestTs, q->bestTs );
					bestTx = better( bestTx, q->bestTx );
				}
				const bool mt = ( sumTs > (double)maxTx ) || forceTs;
				pick = bestTs;
				if( !mt ) pick = better( bestTx, bestTs );
				if( pick.i == 0x7fffffff ) pick = Top1{ 0.0f, 0, 1 };
				tieSh.maskText = mt ? 1 : 0;
			}
			__syncthreads();
			const bool maskText = tieSh.maskText != 0;
			pick = resolveTies( pick, a, b, maskText, isInitial, tieSh );
		if( tid == 0 )
		{
			TokenData td;
			td.id = pick.i;
			td.tid = bestTs.i == 0x7fffffff ? 0 : bestTs.i;
			td.p = pick.v;
			td.pt = (float)( (double)bestTs.v / ( sumTs + 1e-10 ) );
			td.ptsum = (float)sumTs;
			a.out[ b ] = td;
			if( a.nextTokens ) a.nextTokens[ b ] = td.id;
			if( a.history && a.dStep && *a.dStep < a.histCap ) a.history[ (size_t)b * a.histCap + *a.dStep ] = td.id;
			if( a.tokenLog && a.dStep && *a.dStep < a.histCap ) a.tokenLog[ (size_t)b * a.histCap + *a.dStep ] = td;
			if( a.endStep && a.endStep[ b ] == 0 )
			{
				bool ended = td.id == a.tokenEot;
				if( a.winCtl && a.winCtl[ 0 ] )
				{
					const wsp::WindowRule rule{ a.tokenEot, a.tokenBeg, a.winCtl[ 1 ], a.winCtl[ 2 ], a.winCtl[ 3 ] };
					wsp::WindowState st = a.winState[ b ];
					ended = wsp::windowStep( st, rule, 0, a.winCtl[ 4 + b ], *a.dStep, td.id );
					a.winState[ b ] = st;
				}
				if( ended )
				{
					a.endStep[ b ] = *a.dStep + 1;
					atomicAdd( a.nEnded, 1 );
				}
			}
		}
		}
		cluster.sync();   // nobody leaves while a peer may still read its partials
	}

	__global__ void __launch_bounds__( SM_THREADS )
		softmax_rows_kernel( const float* __restrict__ logits, float* __restrict__ probs, int n )
	{
		__shared__ float sf[ SM_THREADS / 32 ];
		__shared__ double sd[ SM_THREADS / 32 ];
		const float* lg = logits + (size_t)blockIdx.x * n;
		float* pr = probs + (size_t)blockIdx.x * n;
		const int tid = threadIdx.x;
		float mx = -INFINITY;
		for( int i = tid; i < n; i += SM_THREADS ) mx = fmaxf( mx, lg[ i ] );
		mx = blockMaxF( mx, sf );
		double dsum = 0.0;
		for( int i = tid; i < n; i += SM_THREADS )
		{
			const float e = expF16Table( lg[ i ] - mx );
			pr[ i ] = e;
			dsum += (double)e;
		}
		dsum = blockSumD( dsum, sd );
		const float inv = (float)( 1.0 / dsum );
		for( int i = tid; i < n; i += SM_THREADS ) pr[ i ] *= inv;
	}
	cudaError_t softmaxRows( const float* logits, float* probs, int rows, int n, cudaStream_t s )
	{
		softmax_rows_kernel<<<rows, SM_THREADS, 0, s>>>( logits, probs, n );
		return cudaGetLastError();
	}

	// one CTA per row; the rank of each language is counted against all others, so the descending order (and the f32 sum taken in it)
	// is the reference's whatever the thread count
	constexpr int LP_THREADS = 128;
	__global__ void __launch_bounds__( LP_THREADS )
		lang_pick_kernel( const LangPickArgs a )
	{
		extern __shared__ float langSh[];
		float* val = langSh;              // [nLangs] the row's language probabilities, by language
		float* ord = langSh + a.nLangs;   // [nLangs] the same values, descending
		__shared__ float sum;
		__shared__ int top;
		const int b = blockIdx.x, n = a.nLangs, tid = threadIdx.x;
		const float* row = a.probs + (size_t)b * a.nVocab + a.tokLang0;
		// a NaN counts as the lowest value, so the ranks below are a permutation whatever the row holds
		for( int i = tid; i < n; i += LP_THREADS ) { const float p = row[ i ]; val[ i ] = isnan( p ) ? -INFINITY : p; }
		__syncthreads();
		for( int i = tid; i < n; i += LP_THREADS )
		{
			const float v = val[ i ];
			int r = 0;
			for( int j = 0; j < n; j++ )
			{
				const float w = val[ j ];
				r += ( w > v || ( w == v && j < i ) ) ? 1 : 0;   // stable: a tie goes to the lower id, as wsp_detect_language's stable_sort
			}
			ord[ r ] = v;
			if( r == 0 ) top = i;
		}
		__syncthreads();
		if( tid == 0 )
		{
			float s = 0;
			for( int k = 0; k < n; k++ ) s += (float)exp( (double)ord[ k ] );
			sum = s;
			a.langIds[ b ] = top;
		}
		__syncthreads();
		for( int i = tid; i < n; i += LP_THREADS ) a.langProbs[ (size_t)b * n + i ] = (float)( exp( (double)val[ i ] ) / (double)sum );
		for( int i = tid; i < a.nPrompt; i += LP_THREADS )
			a.tokens[ (size_t)b * a.nPrompt + i ] = i == a.autoPos ? a.tokLang0 + top : a.tmpl[ i ];
	}
	cudaError_t langPick( const LangPickArgs& a, int B, cudaStream_t s )
	{
		if( a.nLangs < 1 || a.nPrompt < 1 || a.nPrompt > kLangPromptMax || a.autoPos < 0 || a.autoPos >= a.nPrompt ) return cudaErrorInvalidValue;
		lang_pick_kernel<<<B, LP_THREADS, (size_t)2 * a.nLangs * sizeof( float ), s>>>( a );
		return cudaGetLastError();
	}

	__global__ void advance_kernel( int* dNPast, int N, int* dForceTs, int* dStep, const int* nEnded, volatile int* nEndedHost )
	{
		ptx::pdl_launch_dependents();
		ptx::pdl_wait();
		if( dNPast ) *dNPast += N;
		if( dForceTs ) { dForceTs[ 0 ] = 0; dForceTs[ 1 ] = 0; }
		if( dStep ) *dStep += 1;
		// one writer after the whole sampler grid: the host never sees the counter go backwards
		if( nEndedHost ) *nEndedHost = *nEnded;
	}

	cudaError_t sampleGreedy( const SampleArgs& a, cudaStream_t s )
	{
		// 4 CTAs per row; a CTA's slice must fit its 227 KB of shared memory, which bounds the vocabulary at about 230 K tokens
		constexpr int CL = 4;
		if( !a.tieScratch ) return cudaErrorInvalidValue;
		const size_t sliceBytes = (size_t)( ( a.nVocab + CL - 1 ) / CL ) * sizeof( float );
		static PerDeviceMax sliceAttr;
		cudaError_t e = sliceAttr.raise( sliceBytes, []( size_t n ) { return cudaFuncSetAttribute( sample_cluster_kernel<CL>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n ); } );
		if( e != cudaSuccess ) return e;
		cudaLaunchConfig_t cfg{};
		cfg.gridDim = dim3( CL, a.B );
		cfg.blockDim = dim3( SM_THREADS );
		cfg.dynamicSmemBytes = sliceBytes;
		cfg.stream = s;
		cudaLaunchAttribute at[ 1 ];
		at[ 0 ].id = cudaLaunchAttributeClusterDimension;
		at[ 0 ].val.clusterDim.x = CL; at[ 0 ].val.clusterDim.y = 1; at[ 0 ].val.clusterDim.z = 1;
		cfg.attrs = at;
		cfg.numAttrs = 1;
		e = cudaLaunchKernelEx( &cfg, sample_cluster_kernel<CL>, a );
		if( e != cudaSuccess ) return e;
		// step-global state is advanced by a separate 1-thread kernel so that no CTA of the sampler races with it
		if( a.endStep && ( !a.nEnded || !a.nEndedHost ) ) return cudaErrorInvalidValue;
		return launchPdl( advance_kernel, dim3( 1 ), dim3( 1 ), 0, s, a.dNPast, a.N, const_cast<int*>( a.dForceTs ), a.dStep,
			(const int*)a.nEnded, a.endStep ? a.nEndedHost : (volatile int*)nullptr );
	}
}

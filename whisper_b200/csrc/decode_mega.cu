// Persistent decoder-step kernel: one launch runs a whole single-token decoder step (embedding, every layer, final LayerNorm and
// logits) for up to 16 chunks, with grid-wide barriers between the data-dependent phases instead of ~190 kernel launches.
//
// Why: at batch 8 the step is a chain of ~190 tiny weight-streaming ops (SURVEY.md §7 "Decode latency").  Launched as separate
// kernels each one pays launch / drain / first-byte latency while it moves only 2-8 MB, far below the HBM rate.
// Here one CTA per SM stays resident; every phase is split into small units (8 weight rows, or one (chunk, head)) distributed
// round-robin over the resident CTAs; each CTA issues the HBM loads of its NEXT phase (weights / cross-KV, which do not depend on the
// previous phase) BEFORE it waits at the grid barrier, so memory latency overlaps the barrier and the predecessor's tail.
//
// Arithmetic is identical to the kernel-per-op path (kernels_decode.cu): f16 x f16 -> f32 through mma.sync.m16n8k16 with the
// k-permuted fragments, LayerNorm / bias / scale / residual / GELU fused, reference-exact f16 V^T*P chains (pvChainF16).
#include "decode_mega.cuh"
#include "per_device.h"
#include "ptx.cuh"
#include "ref_arith.cuh"
#include <math.h>
#include <type_traits>

namespace kern
{
	namespace
	{
		constexpr int MG_THREADS = 256;
		constexpr int MG_WARPS = 8;
		static_assert( MG_THREADS == kAttnThreads, "the attention phases use the 256-thread helpers of ref_arith.cuh" );
		constexpr int MG_PAD = 32;         // halves of padding per activation row (conflict-free LDS.128)
		constexpr int MG_ROWS = 8;         // weight rows per unit
		constexpr int MG_MAXUPB = 4;       // units per register batch
		constexpr int MG_SMEM_A = 192000;  // activations [16][K+32] f16  |  V tile [1500][64] f16
		constexpr int MG_SMEM_RED = MG_MAXUPB * MG_WARPS * MG_ROWS * 16 * 4;   // 16 KB: cross-warp partials | attention partial outputs
		constexpr int MG_SMEM_SP = 1536 * 4;
		constexpr int MG_SMEM_MISC = 256;
		constexpr int MG_SMEM_PARAM = 2 * 1280 * 4 + 8 * MG_ROWS * 4;   // LayerNorm gamma | beta of the next phase + biases of this CTA's units
		constexpr int MG_MAXBIASUNITS = 8;

		// data written by other CTAs earlier in this launch: read at L2 (never through a possibly stale L1 line)
		__device__ __forceinline__ float4 ldcg4( const float* p ) { return __ldcg( reinterpret_cast<const float4*>( p ) ); }
		__device__ __forceinline__ uint4 ldcgU4( const void* p ) { return __ldcg( reinterpret_cast<const uint4*>( p ) ); }

		// debug: CTA 0 / thread 0 writes %globaltimer into a fixed slot (last layer wins); tm == nullptr in normal runs
		__device__ __forceinline__ void subMark( unsigned long long* tm, int k )
		{
			if( tm && threadIdx.x == 0 ) tm[ k ] = ptx::globaltimer();
		}

		struct Smem
		{
			uint8_t* a;      // MG_SMEM_A
			float* red;      // MG_SMEM_RED
			float* sp;       // MG_SMEM_SP
			float* misc;     // 64 floats
			float* gamma;    // [D] staged by cp.async before the barrier
			float* beta;     // [D]
			float* bias;     // [MG_MAXBIASUNITS][8]
		};

		// Grid-wide barrier for the resident CTAs.  Arrival is one release-atomic on a counter; the last arriver publishes the epoch
		// in a separate 128-byte line that everybody else polls with acquire loads, so the pollers do not queue behind the atomics.
		struct Grid
		{
			unsigned* counter;   // [0] arrivals, [32] epoch flag (separate line); zeroed by the launcher
			unsigned target;
			unsigned epoch;
			// (alternative: per-CTA epoch slots polled by warp 0 of every CTA, no atomics — arrive gets cheaper, but observing one slot
			// per SM costs more than it saves)
			// Split barrier: arrive() right after a phase's last global store, wait() after the next phase's prefetches have been
			// issued.  (A release-atomic drains the issuing warp's outstanding loads first, so arriving AFTER the prefetch issue put
			// an HBM round trip on every barrier's critical path.)
			__device__ __forceinline__ void arrive( unsigned long long* tm = nullptr )
			{
				target += gridDim.x;
				epoch += 1;
				__syncthreads();
				if( threadIdx.x == 0 )
				{
					unsigned old;
					asm volatile( "atom.add.release.gpu.global.u32 %0, [%1], 1;" : "=r"( old ) : "l"( counter ) : "memory" );
					if( old == target - 1 )
						asm volatile( "st.release.gpu.global.u32 [%0], %1;" ::"l"( counter + 32 ), "r"( epoch ) : "memory" );
					if( tm ) tm[ 5 ] = ptx::globaltimer();
				}
			}
			__device__ __forceinline__ void wait()
			{
				if( threadIdx.x == 0 )
				{
					const unsigned* flag = counter + 32;
					unsigned spins = 0;
					while( true )
					{
						unsigned v;
						asm volatile( "ld.acquire.gpu.global.u32 %0, [%1];" : "=r"( v ) : "l"( flag ) : "memory" );
						if( v >= epoch ) break;
						if( ++spins > ( 1u << 25 ) ) __trap();   // a protocol bug must not hang the GPU
					}
				}
				__syncthreads();
			}
		};

		// -----------------------------------------------------------------------------------------------------------
		// weight-streaming GEMV phase:  out[col][n] = sum_k W[n][k] * act[col][k],  n in [0, nOut), col in [0, B)
		enum { EP_QKV = 0, EP_RESID = 1, EP_QSCALE = 2, EP_GELU = 3, EP_LOGITS = 4 };
		struct GemvOp
		{
			const __half* W;
			int nOut;
			const float* xF32;      // LayerNorm input rows (stride = xStride)  — or —
			const __half* xF16;     // ready f16 rows
			int xStride;
			const float* gamma;
			const float* beta;
			int epi;
			const float* bias;
			float scale;
			float* outF32;
			__half* outF16;
			int ld;
			__half* kCache;
			__half* vCache;
			int d, nTextCtx, nPast;
		};

		template<int K>
		struct GemvShape
		{
			static constexpr int STEPS = K / 32;
			static constexpr int SPW = ( STEPS + MG_WARPS - 1 ) / MG_WARPS;        // 32-wide k steps per warp per unit
			static constexpr int SUB = SPW < 16 ? SPW : 16;                         // steps per register batch
			static constexpr int NSUB = ( SPW + SUB - 1 ) / SUB;
			static constexpr int UPB = SPW <= 16 ? ( 16 / SPW < MG_MAXUPB ? 16 / SPW : MG_MAXUPB ) : 1;   // units per batch
		};

		// registers holding one batch of weights
		// (one type for every K, so that the d-wide phases and fc2 share the same 16 x 128-bit registers in the phase loop)
		struct WRegs
		{
			uint4 w[ 16 ];
		};
		template<int K>
		using WBatch = WRegs;

		template<int K>
		__device__ __forceinline__ void loadBatch( WBatch<K>& wb, const GemvOp& op, int firstUnitIdx, int nMine, int sub, int warp, int lane )
		{
			using S = GemvShape<K>;
			const int g = lane >> 2, t = lane & 3;
#pragma unroll
			for( int u = 0; u < S::UPB; u++ )
			{
				const int ui = firstUnitIdx + u;
				const int unit = blockIdx.x + ui * gridDim.x;
				const int row = min( unit * MG_ROWS + g, op.nOut - 1 );
				const uint4* wr = reinterpret_cast<const uint4*>( op.W + (size_t)row * K + 8 * t );
#pragma unroll
				for( int s = 0; s < S::SUB; s++ )
				{
					const int st = warp + MG_WARPS * ( sub * S::SUB + s );
					if( ui < nMine && st < S::STEPS )
						wb.w[ u * S::SUB + s ] = ptx::ldg_stream( wr + st * 4 );
				}
			}
		}

		__device__ __forceinline__ void prefetchL2( const void* p ) { asm volatile( "prefetch.global.L2 [%0];" ::"l"( p ) ); }

		// LayerNorm gamma/beta and the bias entries of this CTA's units of the NEXT phase -> shared memory, requested before the
		// barrier: per-layer parameters are cold in L2 (every step streams ~2 GB through it), and a DRAM miss on them would sit in the
		// middle of the post-barrier critical path
		__device__ __forceinline__ void prefetchParams( const GemvOp& op, int K, const Smem& sm, int tid )
		{
			if( op.gamma )
			{
				const int n16 = K / 4;   // 16-byte chunks per vector
				for( int i = tid; i < 2 * n16; i += MG_THREADS )
				{
					if( i < n16 ) ptx::cp_async16( sm.gamma + i * 4, op.gamma + i * 4 );
					else ptx::cp_async16( sm.beta + ( i - n16 ) * 4, op.beta + ( i - n16 ) * 4 );
				}
			}
			if( op.bias )
			{
				const int units = ( op.nOut + MG_ROWS - 1 ) / MG_ROWS;
				if( tid < MG_MAXBIASUNITS * 2 )
				{
					const int ui = tid >> 1, half = tid & 1;
					const int unit = blockIdx.x + ui * gridDim.x;
					if( unit < units && unit * MG_ROWS + half * 4 + 4 <= op.nOut )
						ptx::cp_async16( sm.bias + ui * MG_ROWS + half * 4, op.bias + unit * MG_ROWS + half * 4 );
				}
			}
			ptx::cp_async_commit();
		}

		template<int K>
		__device__ __forceinline__ int myUnits( const GemvOp& op )
		{
			const int units = ( op.nOut + MG_ROWS - 1 ) / MG_ROWS;
			return units > (int)blockIdx.x ? ( units - (int)blockIdx.x + (int)gridDim.x - 1 ) / (int)gridDim.x : 0;
		}

		// stage the B activation rows as f16 into smem: LayerNorm fused (K == D <= 1280, multiple of 128: one warp per column, the
		// row is held in registers)
		template<int K>
		__device__ __forceinline__ void stageLN( const GemvOp& op, int B, __half* sx, const Smem& sm, int warp, int lane )
		{
			constexpr int RS = K + MG_PAD;
			constexpr int N4 = K / 128;
			const int ncolTiles = B > 8 ? 16 : 8;
			for( int c = warp; c < ncolTiles; c += MG_WARPS )
			{
				__half* dst = sx + (size_t)c * RS;
				if( c >= B )
				{
					uint4* z4 = reinterpret_cast<uint4*>( dst );
					for( int k = lane; k < K / 8; k += 32 ) z4[ k ] = make_uint4( 0, 0, 0, 0 );
					continue;
				}
				const float* src = op.xF32 + (size_t)c * op.xStride;
				float4 v[ N4 ];
				float s = 0.0f;
#pragma unroll
				for( int i = 0; i < N4; i++ )
				{
					v[ i ] = ldcg4( src + ( i * 32 + lane ) * 4 );
					s += v[ i ].x + v[ i ].y + v[ i ].z + v[ i ].w;
				}
				const float mean = ptx::warp_sum( s ) / (float)K;
				float sq = 0.0f;
#pragma unroll
				for( int i = 0; i < N4; i++ )
				{
					v[ i ].x -= mean; v[ i ].y -= mean; v[ i ].z -= mean; v[ i ].w -= mean;
					sq += v[ i ].x * v[ i ].x + v[ i ].y * v[ i ].y + v[ i ].z * v[ i ].z + v[ i ].w * v[ i ].w;
				}
				const float rstd = 1.0f / sqrtf( ptx::warp_sum( sq ) / (float)K + 1e-5f );
				const float4* g4 = reinterpret_cast<const float4*>( sm.gamma );
				const float4* b4 = reinterpret_cast<const float4*>( sm.beta );
				uint2* d2 = reinterpret_cast<uint2*>( dst );
#pragma unroll
				for( int i = 0; i < N4; i++ )
				{
					const float4 gg = g4[ i * 32 + lane ];
					const float4 bb = b4[ i * 32 + lane ];
					__half2 h0 = __floats2half2_rn( v[ i ].x * rstd * gg.x + bb.x, v[ i ].y * rstd * gg.y + bb.y );
					__half2 h1 = __floats2half2_rn( v[ i ].z * rstd * gg.z + bb.z, v[ i ].w * rstd * gg.w + bb.w );
					uint2 u;
					u.x = *reinterpret_cast<uint32_t*>( &h0 );
					u.y = *reinterpret_cast<uint32_t*>( &h1 );
					d2[ i * 32 + lane ] = u;
				}
			}
		}
		// ... or ready f16 rows (attention output, GELU output)
		template<int K>
		__device__ __forceinline__ void stageF16( const GemvOp& op, int B, __half* sx, int tid )
		{
			constexpr int RS = K + MG_PAD;
			constexpr int V8 = K / 8;   // uint4 per row
			const int ncolTiles = B > 8 ? 16 : 8;
			for( int i = tid; i < ncolTiles * V8; i += MG_THREADS )
			{
				const int c = i / V8, k = i - c * V8;
				uint4 val = make_uint4( 0, 0, 0, 0 );
				if( c < B ) val = ldcgU4( op.xF16 + (size_t)c * op.xStride + k * 8 );
				*reinterpret_cast<uint4*>( sx + (size_t)c * RS + k * 8 ) = val;
			}
		}

		__device__ __forceinline__ void gemvEpilogue( const GemvOp& op, int col, int n, float v, float biasN )
		{
			switch( op.epi )
			{
			case EP_QKV:
			{
				const int which = n / op.d;
				const int nn = n - which * op.d;
				if( which == 0 ) op.outF32[ (size_t)col * op.ld + nn ] = ( v + biasN ) * op.scale;
				else
				{
					const size_t off = ( ( (size_t)col * ( op.d >> 6 ) + ( nn >> 6 ) ) * op.nTextCtx + op.nPast ) * 64 + ( nn & 63 );
					if( which == 1 ) op.kCache[ off ] = __float2half_rn( v * op.scale );
					else op.vCache[ off ] = __float2half_rn( v + biasN );
				}
				break;
			}
			case EP_RESID:
			{
				float* p = op.outF32 + (size_t)col * op.ld + n;
				*p = v + biasN + __ldcg( p );
				break;
			}
			case EP_QSCALE:
				op.outF32[ (size_t)col * op.ld + n ] = ( v + biasN ) * op.scale;
				break;
			case EP_GELU:
				op.outF16[ (size_t)col * op.ld + n ] = __float2half_rn( ptx::gelu_f16_semantics( v + biasN ) );
				break;
			default:
				op.outF32[ (size_t)col * op.ld + n ] = v;
				break;
			}
		}

		// compute all units of this CTA; `wb` already holds the first batch (loaded before the barrier)
		template<int K>
		__device__ __forceinline__ void gemvCompute( const GemvOp& op, int B, WBatch<K>& wb, const Smem& sm, int warp, int lane, int tid, unsigned long long* tm = nullptr )
		{
			subMark( tm, 0 );
			using S = GemvShape<K>;
			constexpr int RS = K + MG_PAD;
			const __half* sx = reinterpret_cast<const __half*>( sm.a );
			const int g = lane >> 2, t = lane & 3;
			const __half* xb0 = sx + (size_t)g * RS + 8 * t;
			const __half* xb1 = sx + (size_t)( g + 8 ) * RS + 8 * t;
			const bool twoTiles = B > 8;
			const int nMine = myUnits<K>( op );
			const int ncols = twoTiles ? 16 : 8;
			for( int u0 = 0; u0 < nMine; u0 += S::UPB )
			{
				float acc0[ S::UPB ][ 4 ], acc1[ S::UPB ][ 4 ];
#pragma unroll
				for( int u = 0; u < S::UPB; u++ )
#pragma unroll
					for( int i = 0; i < 4; i++ ) { acc0[ u ][ i ] = 0.0f; acc1[ u ][ i ] = 0.0f; }
#pragma unroll
				for( int sub = 0; sub < S::NSUB; sub++ )
				{
					if( sub != 0 ) loadBatch<K>( wb, op, u0, nMine, sub, warp, lane );   // (sub 0 of every batch is already in flight)
#pragma unroll
					for( int u = 0; u < S::UPB; u++ )
#pragma unroll
						for( int s = 0; s < S::SUB; s++ )
						{
							const int st = warp + MG_WARPS * ( sub * S::SUB + s );
							if( u0 + u < nMine && st < S::STEPS )
							{
								const uint4 w = wb.w[ u * S::SUB + s ];
								const uint4 x0 = *reinterpret_cast<const uint4*>( xb0 + st * 32 );
								ptx::mma_m16n8k16_rows8( acc0[ u ], w.x, w.y, x0.x, x0.y );
								ptx::mma_m16n8k16_rows8( acc0[ u ], w.z, w.w, x0.z, x0.w );
								if( twoTiles )
								{
									const uint4 x1 = *reinterpret_cast<const uint4*>( xb1 + st * 32 );
									ptx::mma_m16n8k16_rows8( acc1[ u ], w.x, w.y, x1.x, x1.y );
									ptx::mma_m16n8k16_rows8( acc1[ u ], w.z, w.w, x1.z, x1.w );
								}
							}
						}
				}
				subMark( tm, 1 );   // MMA loop done (the weight registers had to have landed)
				// the weight registers are dead now: request the next batch before the reduction / epilogue of this one (the logits
				// phase walks 11 batches per CTA; this hides one reduction + epilogue behind every HBM round trip)
				if( u0 + S::UPB < nMine ) loadBatch<K>( wb, op, u0 + S::UPB, nMine, 0, warp, lane );
				// cross-warp reduction: red[u][warp][row g][col]
#pragma unroll
				for( int u = 0; u < S::UPB; u++ )
				{
					float* my = sm.red + ( ( u * MG_WARPS + warp ) * MG_ROWS + g ) * 16;
					my[ 2 * t ] = acc0[ u ][ 0 ];
					my[ 2 * t + 1 ] = acc0[ u ][ 1 ];
					if( twoTiles ) { my[ 8 + 2 * t ] = acc1[ u ][ 0 ]; my[ 8 + 2 * t + 1 ] = acc1[ u ][ 1 ]; }
				}
				__syncthreads();
				subMark( tm, 2 );
				for( int idx = tid; idx < S::UPB * ncols * MG_ROWS; idx += MG_THREADS )
				{
					const int u = idx / ( ncols * MG_ROWS );
					const int rem = idx - u * ncols * MG_ROWS;
					const int c = rem / MG_ROWS, r = rem - c * MG_ROWS;
					const int unit = blockIdx.x + ( u0 + u ) * gridDim.x;
					const int n = unit * MG_ROWS + r;
					if( u0 + u < nMine && c < B && n < op.nOut )
					{
						float v = 0.0f;
#pragma unroll
						for( int w = 0; w < MG_WARPS; w++ ) v += sm.red[ ( ( u * MG_WARPS + w ) * MG_ROWS + r ) * 16 + c ];
						float biasN = 0.0f;
						if( op.bias ) biasN = ( u0 + u < MG_MAXBIASUNITS ) ? sm.bias[ ( u0 + u ) * MG_ROWS + r ] : op.bias[ n ];
						gemvEpilogue( op, c, n, v, biasN );
					}
				}
				subMark( tm, 3 );
				__syncthreads();
			}
			subMark( tm, 4 );
		}

		// -----------------------------------------------------------------------------------------------------------
		// self attention over the self-KV cache (N = 1): units = (chunk, head).  The rows of earlier tokens are final, so they are
		// copied to shared memory by cp.async BEFORE the barrier that publishes this step's new row; after it only 2 x 128 bytes remain.
		constexpr int SA_KSTRIDE = 144;   // bytes per K row in smem (128 + 16: conflict-free 16-byte reads of one row per thread)
		constexpr int SA_MAXKV = 448;
		__device__ __forceinline__ void selfLoadRows( const MegaArgs& a, const DecStepLayer& L, int d, const Smem& sm, int unit, int j0, int j1, int tid )
		{
			if( unit >= a.B * a.H ) return;
			const int b = unit / a.H, h = unit - b * a.H;
			const __half* kb = L.kCache + ( (size_t)b * a.H + h ) * a.nTextCtx * 64;
			const __half* vb = L.vCache + ( (size_t)b * a.H + h ) * a.nTextCtx * 64;
			uint8_t* sK = sm.a;
			uint8_t* sV = sm.a + SA_MAXKV * SA_KSTRIDE;
			const int n = ( j1 - j0 ) * 8;   // 16-byte chunks per matrix
			for( int i = tid; i < 2 * n; i += MG_THREADS )
			{
				const bool isV = i >= n;
				const int k = isV ? i - n : i;
				const int j = j0 + ( k >> 3 ), c = k & 7;
				if( isV ) ptx::cp_async16( sV + j * 128 + c * 16, vb + (size_t)j * 64 + c * 8 );
				else ptx::cp_async16( sK + j * SA_KSTRIDE + c * 16, kb + (size_t)j * 64 + c * 8 );
			}
		}
		__device__ void selfAttnPhase( const MegaArgs& a, const DecStepLayer& L, int d, int nPast, const Smem& sm, int warp, int lane, int tid )
		{
			const int H = a.H;
			const int nkv = min( nPast + 1, a.nTextCtx );
			float* sq = sm.misc;
			float* sred = sm.misc + 64;
			float* so = sm.red;
			const uint8_t* sK = sm.a;
			const __half* sV = reinterpret_cast<const __half*>( sm.a + SA_MAXKV * SA_KSTRIDE );
			bool first = true;
			for( int unit = blockIdx.x; unit < a.B * H; unit += gridDim.x )
			{
				const int b = unit / H, h = unit - b * H;
				// rows [0, nkv-1) of the first unit were requested before the barrier; the new row (and everything for further units) now
				selfLoadRows( a, L, d, sm, unit, first ? nkv - 1 : 0, nkv, tid );
				ptx::cp_async_commit();
				first = false;
				if( tid < 64 ) sq[ tid ] = __half2float( __float2half_rn( __ldcg( a.q + (size_t)b * d + h * 64 + tid ) ) );
				ptx::cp_async_wait_all();
				__syncthreads();
				float lmax = -INFINITY;
				for( int j = tid; j < nkv; j += MG_THREADS )
				{
					const uint4* kr = reinterpret_cast<const uint4*>( sK + j * SA_KSTRIDE );
					float s = 0.0f;
#pragma unroll
					for( int c = 0; c < 8; c++ )
					{
						const uint4 u = kr[ c ];
						const __half2* h2 = reinterpret_cast<const __half2*>( &u );
#pragma unroll
						for( int e = 0; e < 4; e++ )
						{
							const float2 f = __half22float2( h2[ e ] );
							s += f.x * sq[ c * 8 + e * 2 ] + f.y * sq[ c * 8 + e * 2 + 1 ];
						}
					}
					sm.sp[ j ] = s;
					lmax = fmaxf( lmax, s );
				}
				softmaxRow<ctaSync>( sm.sp, nkv, lmax, sred, tid, warp, lane );
				pvSplitF16( sm.sp, sV, nkv, a.refThreads, ( nkv + a.refThreads - 1 ) / a.refThreads, so, a.attn + (size_t)b * d + h * 64, tid );
				__syncthreads();
			}
		}

		// -----------------------------------------------------------------------------------------------------------
		// cross attention over the encoder's f16 K/V memories: units = (chunk, head).  The V tile and the first batch of K rows are
		// requested BEFORE the grid barrier (they do not depend on this step), q is read after it.
		struct CrossPrefetch
		{
			uint4 u[ kKBatch ];
			int unit;
		};
		__device__ __forceinline__ void crossPrefetch( const MegaArgs& a, const DecStepLayer& L, CrossPrefetch& pf, const Smem& sm, int unit, int warp, int lane, int tid )
		{
			pf.unit = unit;
			if( unit >= a.B * a.H ) return;
			const int T = a.T;
			const size_t base = (size_t)unit * T * 64;   // unit = b * H + h
			const uint4* V4 = reinterpret_cast<const uint4*>( L.crossV + base );
			uint4* sv = reinterpret_cast<uint4*>( sm.a );
			for( int idx = tid; idx < T * 8; idx += MG_THREADS ) ptx::cp_async16( sv + idx, V4 + idx );
			ptx::cp_async_commit();
			kStreamPrefetch( pf.u, reinterpret_cast<const uint4*>( L.crossK + base ), T, warp, lane );
		}
		__device__ void crossAttnPhase( const MegaArgs& a, const DecStepLayer& L, int d, CrossPrefetch& pf, const Smem& sm, int warp, int lane, int tid )
		{
			const int T = a.T, H = a.H;
			float* sred = sm.misc + 64;
			float* so = sm.red;
			bool first = true;
			for( int unit = blockIdx.x; unit < a.B * H; unit += gridDim.x )
			{
				if( !first ) { crossPrefetch( a, L, pf, sm, unit, warp, lane, tid ); }
				first = false;
				const int b = unit / H, h = unit - b * H;
				const uint4* K4 = reinterpret_cast<const uint4*>( L.crossK + (size_t)unit * T * 64 );
				float qf[ 8 ];
#pragma unroll
				for( int e = 0; e < 8; e++ ) qf[ e ] = __half2float( __float2half_rn( __ldcg( a.q + (size_t)b * d + h * 64 + ( lane & 7 ) * 8 + e ) ) );
				const float lmax = kStreamScores( pf.u, K4, T, qf, sm.sp, warp, lane );
				softmaxRow<ctaSync>( sm.sp, T, lmax, sred, tid, warp, lane );
				ptx::cp_async_wait_all();
				__syncthreads();
				pvSplitF16( sm.sp, reinterpret_cast<const __half*>( sm.a ), T, a.refThreads, ( T + a.refThreads - 1 ) / a.refThreads, so,
					a.attn + (size_t)b * d + h * 64, tid );
				__syncthreads();
			}
		}

		// -----------------------------------------------------------------------------------------------------------
		template<int D>
		__global__ void __launch_bounds__( MG_THREADS, 1 )
			decode_step_kernel( MegaArgs a )
		{
			extern __shared__ __align__( 16 ) uint8_t mg_smem[];
			Smem sm;
			sm.a = mg_smem;
			sm.red = reinterpret_cast<float*>( mg_smem + MG_SMEM_A );
			sm.sp = reinterpret_cast<float*>( mg_smem + MG_SMEM_A + MG_SMEM_RED );
			sm.misc = reinterpret_cast<float*>( mg_smem + MG_SMEM_A + MG_SMEM_RED + MG_SMEM_SP );
			sm.gamma = reinterpret_cast<float*>( mg_smem + MG_SMEM_A + MG_SMEM_RED + MG_SMEM_SP + MG_SMEM_MISC * 4 );
			sm.beta = sm.gamma + 1280;
			sm.bias = sm.beta + 1280;
			const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
			const int B = a.B;
			const int nPast = *a.dNPast;              // read once: the sampler's advance kernel updates it after this launch
			const int nkvOld = min( nPast, a.nTextCtx - 1 );
			const float qkScale = 0.35355339059327379f;   // 64^-1/4 (whisper.cpp:1588, 1595, 1700)
			Grid grid{ a.barrier, 0u, 0u };
			int markIdx = 0;
			auto markId = [ & ]( int id ) {
				if( a.timing && blockIdx.x == 0 && tid == 0 && markIdx < 2040 )
				{
					const unsigned long long t = ptx::globaltimer();
					a.timing[ 2 * markIdx ] = (unsigned long long)id;
					a.timing[ 2 * markIdx + 1 ] = t;
				}
				markIdx++;
			};
			int phaseId = 0;
			auto mark = [ & ]() { markId( phaseId++ ); };   // even ids: before a barrier, odd: after it
			mark();
			__half* sx = reinterpret_cast<__half*>( sm.a );

			static_assert( GemvShape<D>::UPB * GemvShape<D>::SUB <= 16 && GemvShape<4 * D>::UPB * GemvShape<4 * D>::SUB <= 16, "register batch" );
			WRegs wb;
			GemvOp base{};
			base.d = D; base.nTextCtx = a.nTextCtx; base.nPast = nPast; base.scale = 1.0f;

			// The phases of a layer.  The step is ONE loop over (layer, phase) with a single call site per code path: the straight-line
			// version instantiated the GEMV code seven times (12.4 K SASS instructions = 199 KB, 16 % of all stall samples were
			// instruction-fetch misses); this form keeps the kernel within reach of the instruction cache.
			enum { PH_QKV = 0, PH_SELF = 1, PH_O = 2, PH_CQ = 3, PH_CROSS = 4, PH_CO = 5, PH_FC1 = 6, PH_FC2 = 7, PH_COUNT = 8 };
			// operands of GEMV phase `ph` of layer `il`; il == L is the final LayerNorm + logits (a17)
			auto makeOp = [ & ]( int il, int ph ) {
				GemvOp o = base;
				if( il >= a.L )
				{
					o.W = a.tokEmb; o.nOut = a.nVocab; o.xF32 = a.x; o.xStride = D; o.gamma = a.lnfg; o.beta = a.lnfb;
					o.epi = EP_LOGITS; o.outF32 = a.logits; o.ld = a.nVocab;
					return o;
				}
				const DecStepLayer& L = a.layers[ il ];
				switch( ph )
				{
				case PH_QKV:   // LN1 + (Q | K | V), K/V appended to the cache (a14)
					o.W = L.wqkv; o.nOut = 3 * D; o.xF32 = a.x; o.xStride = D; o.gamma = L.ln1g; o.beta = L.ln1b;
					o.epi = EP_QKV; o.bias = L.bqkv; o.scale = qkScale; o.outF32 = a.q; o.ld = D; o.kCache = L.kCache; o.vCache = L.vCache;
					break;
				case PH_O:     // self-attention out projection + residual
					o.W = L.wo; o.nOut = D; o.xF16 = a.attn; o.xStride = D; o.epi = EP_RESID; o.bias = L.bo; o.outF32 = a.x; o.ld = D;
					break;
				case PH_CQ:    // cross-attention query (a15)
					o.W = L.wcq; o.nOut = D; o.xF32 = a.x; o.xStride = D; o.gamma = L.lncg; o.beta = L.lncb;
					o.epi = EP_QSCALE; o.bias = L.bcq; o.scale = qkScale; o.outF32 = a.q; o.ld = D;
					break;
				case PH_CO:    // cross-attention out projection + residual
					o.W = L.wco; o.nOut = D; o.xF16 = a.attn; o.xStride = D; o.epi = EP_RESID; o.bias = L.bco; o.outF32 = a.x; o.ld = D;
					break;
				case PH_FC1:   // LN3 + fc1 + GELU (a16)
					o.W = L.w1; o.nOut = 4 * D; o.xF32 = a.x; o.xStride = D; o.gamma = L.ln3g; o.beta = L.ln3b;
					o.epi = EP_GELU; o.bias = L.b1; o.outF16 = a.h; o.ld = 4 * D;
					break;
				default:       // PH_FC2: fc2 + residual
					o.W = L.w2; o.nOut = D; o.xF16 = a.h; o.xStride = 4 * D; o.epi = EP_RESID; o.bias = L.b2; o.outF32 = a.x; o.ld = D;
					break;
				}
				return o;
			};
			// everything a phase needs that does not depend on the previous phase is requested before the barrier wait
			// (alternative: prefetching these rows into L2 only and loading the registers after the barrier is exactly as fast)
			auto prepD = [ & ]( const GemvOp& o ) {
				loadBatch<D>( wb, o, 0, myUnits<D>( o ), 0, warp, lane );
				prefetchParams( o, D, sm, tid );
			};
			// after the barrier: parameters have landed
			auto landed = [ & ]() { ptx::cp_async_wait_all(); __syncthreads(); };

			// a layer's cross-attention K/V tile of "my" (chunk, head) starts moving HBM -> L2 several phases ahead of its use (those
			// phases are latency-bound and leave the DRAM pipe idle); issued while waiting at a barrier, off the critical path
			auto crossL2 = [ & ]( const DecStepLayer& L ) {
				if( (int)blockIdx.x < B * a.H )
				{
					const size_t cb = (size_t)blockIdx.x * a.T * 64;
					const uint8_t* kp = reinterpret_cast<const uint8_t*>( L.crossK + cb );
					const uint8_t* vp = reinterpret_cast<const uint8_t*>( L.crossV + cb );
					for( int i = tid; i < a.T; i += MG_THREADS ) { prefetchL2( kp + (size_t)i * 128 ); prefetchL2( vp + (size_t)i * 128 ); }
				}
			};

			// ---- embedding (a13) by the first B CTAs; layer 0's QKV weights and LayerNorm parameters are already in flight ----
			GemvOp op = makeOp( 0, PH_QKV );
			prepD( op );
			for( int b = blockIdx.x; b < B; b += gridDim.x )
			{
				const int tok = a.tokens[ b ];
				const __half* src = a.tokEmb + (size_t)tok * D;
				const float* pe = a.decPos + (size_t)nPast * D;
				for( int e = tid; e < D; e += MG_THREADS ) a.x[ (size_t)b * D + e ] = __half2float( src[ e ] ) + pe[ e ];
			}
			grid.arrive();
			crossL2( a.layers[ 0 ] );
			mark(); grid.wait(); mark();

			unsigned long long* tmBase = ( a.timing && blockIdx.x == 0 ) ? a.timing + 4000 : nullptr;
			CrossPrefetch pf;
			pf.unit = 0;
#pragma unroll 1
			for( int il = 0; il <= a.L; il++ )
			{
				const DecStepLayer& L = a.layers[ il < a.L ? il : a.L - 1 ];
#pragma unroll 1
				for( int ph = 0; ph < PH_COUNT; ph++ )
				{
					// ---------------- the phase's work ----------------
					if( ph == PH_SELF ) selfAttnPhase( a, L, D, nPast, sm, warp, lane, tid );
					else if( ph == PH_CROSS ) crossAttnPhase( a, L, D, pf, sm, warp, lane, tid );
					else if( ph == PH_FC2 )
					{
						landed();
						stageF16<4 * D>( op, B, sx, tid );
						__syncthreads();
						markId( 1001 + 2 * PH_FC2 );
						gemvCompute<4 * D>( op, B, wb, sm, warp, lane, tid, tmBase ? tmBase + ph * 8 : nullptr );
						markId( 1002 + 2 * PH_FC2 );
					}
					else
					{
						landed();
						if( ph == PH_FC1 && il + 1 == a.L )
						{
							// last layer: start pulling this CTA's rows of the unembedding matrix into L2 (106 MB over all CTAs)
							const int units = ( a.nVocab + MG_ROWS - 1 ) / MG_ROWS;
							for( int u = blockIdx.x; u < units; u += gridDim.x )
							{
								const uint8_t* wp = reinterpret_cast<const uint8_t*>( a.tokEmb + (size_t)u * MG_ROWS * D );
								const int rows = min( MG_ROWS, a.nVocab - u * MG_ROWS );
								for( int i = tid; i < rows * D * 2 / 128; i += MG_THREADS ) prefetchL2( wp + (size_t)i * 128 );
							}
						}
						if( op.xF32 ) stageLN<D>( op, B, sx, sm, warp, lane );
						else stageF16<D>( op, B, sx, tid );
						__syncthreads();
						markId( 1001 + 2 * ph );
						gemvCompute<D>( op, B, wb, sm, warp, lane, tid, tmBase ? tmBase + ph * 8 : nullptr );
						markId( 1002 + 2 * ph );
					}
					if( il == a.L ) break;   // the logits were the last thing to do
					grid.arrive( tmBase ? tmBase + ph * 8 : nullptr );
					// ---------------- requests for what follows, issued while the other CTAs arrive ----------------
					int nextPh = -1, nextIl = il;
					switch( ph )
					{
					case PH_QKV: nextPh = PH_O; break;          // (self attention does not use the weight registers)
					case PH_O: nextPh = PH_CQ; break;
					case PH_CROSS: nextPh = PH_CO; break;
					case PH_CO: nextPh = PH_FC1; break;
					case PH_FC2: nextPh = PH_QKV; nextIl = il + 1; break;
					default: break;
					}
					if( nextPh >= 0 )
					{
						op = makeOp( nextIl, nextPh );
						prepD( op );
					}
					if( ph == PH_QKV )
					{
						// earlier tokens' K/V rows of my (chunk, head) -> smem (region A is free: the activations are consumed)
						selfLoadRows( a, L, D, sm, blockIdx.x, 0, nkvOld, tid );
						ptx::cp_async_commit();
					}
					else if( ph == PH_CQ )
						crossPrefetch( a, L, pf, sm, blockIdx.x, warp, lane, tid );   // V tile -> smem (region A is free now), first K rows -> registers
					else if( ph == PH_FC1 )
					{
						op = makeOp( il, PH_FC2 );
						loadBatch<4 * D>( wb, op, 0, myUnits<4 * D>( op ), 0, warp, lane );
						prefetchParams( op, 4 * D, sm, tid );
					}
					else if( ph == PH_FC2 && il + 1 < a.L ) crossL2( a.layers[ il + 1 ] );
					subMark( tmBase ? tmBase + ph * 8 : nullptr, 6 );
					mark(); grid.wait(); mark();
					subMark( tmBase ? tmBase + ph * 8 : nullptr, 7 );
				}
			}
			mark();
		}

		constexpr int SMEM = MG_SMEM_A + MG_SMEM_RED + MG_SMEM_SP + MG_SMEM_MISC * 4 + MG_SMEM_PARAM;
		template<int D>
		cudaError_t prepareD()
		{
			static_assert( 16 * ( 4 * D + MG_PAD ) * 2 <= MG_SMEM_A, "activation rows must fit region A" );
			static PerDeviceMax attr;
			return attr.raise( SMEM, []( size_t n ) { return cudaFuncSetAttribute( decode_step_kernel<D>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n ); } );
		}
		template<int D>
		cudaError_t launchD( const MegaArgs& a, int numSMs, cudaStream_t s )
		{
			cudaError_t e = prepareD<D>();
			if( e != cudaSuccess ) return e;
			e = cudaMemsetAsync( a.barrier, 0, 64 * sizeof( unsigned ), s );
			if( e != cudaSuccess ) return e;
			decode_step_kernel<D><<<numSMs, MG_THREADS, SMEM, s>>>( a );
			return cudaGetLastError();
		}

		// the decoder widths the kernel is instantiated for: f( integral_constant<int, D> ) for d == D, `unsupported` for any other d
		template<class R, class F>
		R dispatchD( int d, R unsupported, F&& f )
		{
			switch( d )
			{
			case 128: return f( std::integral_constant<int, 128>() );
			case 384: return f( std::integral_constant<int, 384>() );
			case 512: return f( std::integral_constant<int, 512>() );
			case 768: return f( std::integral_constant<int, 768>() );
			case 1024: return f( std::integral_constant<int, 1024>() );
			case 1280: return f( std::integral_constant<int, 1280>() );
			default: return unsupported;
			}
		}
	}

	bool megaSupported( int d, int B, int T )
	{
		if( B < 1 || B > 16 || T * 128 > MG_SMEM_A ) return false;
		return dispatchD( d, false, []( auto ) { return true; } );
	}

	cudaError_t megaPrepare( int d )
	{
		return dispatchD( d, cudaSuccess, []( auto D ) { return prepareD<decltype( D )::value>(); } );
	}

	cudaError_t decodeStepMega( const MegaArgs& a, int d, int numSMs, cudaStream_t s )
	{
		return dispatchD( d, cudaErrorInvalidValue, [ & ]( auto D ) { return launchD<decltype( D )::value>( a, numSMs, s ); } );
	}
}

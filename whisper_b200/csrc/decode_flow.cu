// Dataflow decoder-step kernel: one launch runs a whole single-token decoder step (embedding, every layer, final LayerNorm and
// logits) for up to 16 chunks.  Reference: whisper_decode, Whisper/source/whisper.cpp:1508-1872 (what one step must compute);
// it replaces the per-token dispatch chain around ComputeShaders/mulMatByRowTiled.hlsl (Whisper/Whisper/WhisperContext.cpp:578-639).
//
// Round 1 ran the step as a persistent kernel with a grid-wide counter barrier between the ~190 data-dependent phases; it sat at
// 20 % of the HBM rate because every phase paid  arrive (block barrier + release fence + atomic round trip) + flag poll + an L2
// round trip for the activations + a burst of weight loads that the in-order load queue put in front of everything else.
// This kernel removes both costs:
//
//  * Weights, LayerNorm parameters and the self / cross K,V rows never depend on the current step.  A PRODUCER WARP streams them
//    in consumption order into a shared-memory ring with TMA bulk copies (cp.async.bulk + mbarrier complete_tx), as far ahead as
//    the ring allows (~180 KB per SM), so the HBM pipe is busy for the whole step and the consumers' loads never queue behind it.
//  * There is NO grid barrier.  Every (layer, phase) output has its own exchange buffer, pre-filled with a sentinel that the
//    arithmetic cannot produce (all-ones: a NaN payload no FP instruction generates).  Producers of a phase simply store their
//    results; consumers poll the data itself (ld.relaxed.gpu) until no sentinel is left.  One L2 write + one L2 read is the
//    whole exchange; a 4-byte (f32) or 2-byte (f16) element is its own flag, so no fences or ordering between stores are needed.
//    Two buffer sets alternate between launches; each step re-arms the idle set (whose readers finished with the previous launch).
//
// Arithmetic is identical to round 1's kernels: f16 x f16 -> f32 through mma.sync.m16n8k16 with k-permuted fragments, 8 warps
// splitting K in the same order, LayerNorm / bias / scale / residual / GELU fused, reference-exact f16 V^T*P chains.
#include "decode_flow.cuh"
#include "per_device.h"
#include "ptx.cuh"
#include "ref_arith.cuh"
#include <math.h>
#include <type_traits>

namespace kern
{
	namespace
	{
		constexpr int FL_WARPS = 8;                    // consumer warps
		constexpr int FL_CONSUMERS = FL_WARPS * 32;
		constexpr int FL_THREADS = FL_CONSUMERS + 32;  // + the producer warp
		static_assert( FL_CONSUMERS == kAttnThreads, "softmaxRow (ref_arith.cuh) runs on the consumer warps" );
		constexpr int FL_NSMAX = 32;
		constexpr int FL_MAXT = 1536;
		constexpr int FL_SMEM_MAX = 232448;            // 227 KB opt-in limit per CTA on sm_90
		constexpr uint32_t SENT32 = 0xFFFFFFFFu;

		template<int D>
		struct Cfg
		{
			static constexpr int RS = 2 * D + 64;                                  // bytes per weight / activation row in shared memory (conflict-free LDS.128)
			static constexpr int SLOT = ( 8 * RS > 16384 ) ? 8 * RS : 16384;       // one ring slot: 8 weight rows x D, or a run of K/V rows
			static constexpr int CR = ( SLOT / 128 ) & ~7;                         // K/V rows (128 bytes each) per slot
			static constexpr int STEPS = D / 32;
			static constexpr int SPW = ( STEPS + FL_WARPS - 1 ) / FL_WARPS;
			static constexpr int N4 = D / 128;
		};

		struct SmemLayout
		{
			int act, red, sp, bias, xres, so, sred, qkv, bars, total;
		};
		__host__ __device__ inline SmemLayout smemLayout( int slot, int rs, int NS, int ncols )
		{
			SmemLayout l;
			int o = NS * slot;
			l.act = o; o += ncols * rs;
			l.red = o; o += 4 * FL_WARPS * 8 * ncols * 4;
			l.sp = o; o += FL_MAXT * 4;
			l.bias = o; o += 256 * 4;
			l.xres = o; o += 16 * 16 * 4;
			l.so = o; o += kMaxRefThreads * 64 * 4;
			l.sred = o; o += 64;
			l.qkv = o; o += 3 * 128;
			l.bars = o; o += 2 * FL_NSMAX * 8;
			l.total = o;
			return l;
		}
		inline int ringSlots( int slot, int rs, int ncols )
		{
			const int fixed = smemLayout( slot, rs, 0, ncols ).total;
			int ns = ( FL_SMEM_MAX - fixed ) / slot;
			return ns > FL_NSMAX ? FL_NSMAX : ns;
		}

		// ---- small device helpers ------------------------------------------------------------------------------------
		__device__ __forceinline__ void consumerSync() { asm volatile( "bar.sync 1, 256;" ::: "memory" ); }

		// exchange accesses: performed at L2 (gpu scope), never through a possibly stale L1 line
		__device__ __forceinline__ uint4 ldPoll( const void* p )
		{
			uint4 r;
			asm volatile( "ld.relaxed.gpu.global.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"( r.x ), "=r"( r.y ), "=r"( r.z ), "=r"( r.w ) : "l"( p ) : "memory" );
			return r;
		}
		__device__ __forceinline__ uint32_t ldPoll32( const void* p )
		{
			uint32_t r;
			asm volatile( "ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"( r ) : "l"( p ) : "memory" );
			return r;
		}
		__device__ __forceinline__ bool hasSent32( const uint4& v ) { return v.x == SENT32 || v.y == SENT32 || v.z == SENT32 || v.w == SENT32; }
		__device__ __forceinline__ bool hasSent16w( uint32_t w ) { return ( w & 0xFFFFu ) == 0xFFFFu || ( w >> 16 ) == 0xFFFFu; }
		__device__ __forceinline__ bool hasSent16( const uint4& v ) { return hasSent16w( v.x ) || hasSent16w( v.y ) || hasSent16w( v.z ) || hasSent16w( v.w ); }
		__device__ __forceinline__ void stX32( float* p, float v )
		{
			uint32_t b = __float_as_uint( v );
			if( b == SENT32 ) b = 0x7FFFFFFFu;   // a NaN stays a NaN, but never looks like "not written yet"
			asm volatile( "st.relaxed.gpu.global.u32 [%0], %1;" ::"l"( p ), "r"( b ) : "memory" );
		}
		__device__ __forceinline__ void stX16( __half* p, __half v )
		{
			unsigned short b = __half_as_ushort( v );
			if( b == 0xFFFFu ) b = 0x7FFFu;
			asm volatile( "st.relaxed.gpu.global.u16 [%0], %1;" ::"l"( p ), "h"( b ) : "memory" );
		}
		// a protocol bug must not hang the GPU: every wait gives up (trap = launch failure) after ~2 s of wall time
		__device__ __noinline__ void spinCheck( unsigned long long& t0 )
		{
			const unsigned long long t = ptx::globaltimer();
			if( t0 == 0 ) t0 = t;
			else if( t - t0 > 2000000000ull ) __trap();
		}
		struct SpinGuard
		{
			unsigned spins = 0;
			unsigned long long t0 = 0;
			__device__ __forceinline__ void tick()
			{
				if( ( ++spins & 1023u ) == 0 ) spinCheck( t0 );
			}
		};
		__device__ __forceinline__ void mbarWaitLong( uint64_t* bar, uint32_t parity )
		{
			SpinGuard g;
			while( !ptx::mbar_try_wait( bar, parity ) ) g.tick();
		}


		// The reference's f16-accumulated V^T*P (ggml.c:4680-4722, 871-893): y = f16( fma( V[j][e], P[j], y ) ) key by key — three dependent
		// ALU instructions per key (FFMA -> F2FP.F16.F32 -> HADD2.F32), inherent to the reference's arithmetic (staging the
		// operands of eight keys ahead of the chain changed nothing: it is not load-bound).
		__device__ __forceinline__ float chainStep( float y, float x, float p ) { return __half2float( __float2half_rn( __fmaf_rn( x, p, y ) ) ); }
		__device__ __forceinline__ float chainRows( float y, const float* __restrict__ sp, const __half* __restrict__ v, int n )
		{
			int j = 0;
			for( ; j + 4 <= n; j += 4 )
			{
				const float x0 = __half2float( v[ j * 64 ] );
				const float x1 = __half2float( v[ ( j + 1 ) * 64 ] );
				const float x2 = __half2float( v[ ( j + 2 ) * 64 ] );
				const float x3 = __half2float( v[ ( j + 3 ) * 64 ] );
				y = chainStep( y, x0, sp[ j ] );
				y = chainStep( y, x1, sp[ j + 1 ] );
				y = chainStep( y, x2, sp[ j + 2 ] );
				y = chainStep( y, x3, sp[ j + 3 ] );
			}
			for( ; j < n; j++ ) y = chainStep( y, __half2float( v[ j * 64 ] ), sp[ j ] );
			return y;
		}
		// Four chains of one thread side by side (reference thread counts above 4: 64 dims x `parts` chains over 256 threads).  The chains
		// are independent, so their dependent steps overlap: four cost about what one does.  Chain k reads rows [0, n[k]) at
		// v + k * rr * 64 and the probabilities sp[j0[k] ...]; n[] does not increase with k (a group's parts are consecutive key ranges
		// clipped to the same end).  The rows every live chain has go through the interleaved loop — no predicates, every load hoisted
		// above the arithmetic; a chain without rows rides along as a copy of chain 0 whose result is dropped — and what is left of the
		// longer ones (the last part is the short one) follows.
		__device__ __forceinline__ void chainSide( float ( &y )[ 4 ], const float* __restrict__ sp, const __half* __restrict__ v, const int ( &j0 )[ 4 ], const int ( &n )[ 4 ], int rr )
		{
			int nmin = n[ 0 ];
			const __half* vb[ 4 ];
			const float* pb[ 4 ];
			float t[ 4 ];
#pragma unroll
			for( int k = 0; k < 4; k++ )
			{
				const bool on = n[ k ] > 0;
				if( on ) nmin = min( nmin, n[ k ] );
				vb[ k ] = v + ( on ? k * rr * 64 : 0 );
				pb[ k ] = sp + ( on ? j0[ k ] : j0[ 0 ] );
				t[ k ] = y[ k ];
			}
			int j = 0;
			for( ; j + 2 <= nmin; j += 2 )
			{
				float x[ 4 ][ 2 ], pj[ 4 ][ 2 ];
#pragma unroll
				for( int k = 0; k < 4; k++ )
#pragma unroll
					for( int i = 0; i < 2; i++ )
					{
						x[ k ][ i ] = __half2float( vb[ k ][ ( j + i ) * 64 ] );
						pj[ k ][ i ] = pb[ k ][ j + i ];
					}
#pragma unroll
				for( int i = 0; i < 2; i++ )
#pragma unroll
					for( int k = 0; k < 4; k++ ) t[ k ] = chainStep( t[ k ], x[ k ][ i ], pj[ k ][ i ] );
			}
#pragma unroll
			for( int k = 0; k < 4; k++ )
			{
				if( n[ k ] > 0 ) y[ k ] = t[ k ];
#pragma unroll 1
				for( int i = j; i < n[ k ]; i++ ) y[ k ] = chainStep( y[ k ], __half2float( vb[ k ][ i * 64 ] ), pb[ k ][ i ] );
			}
		}

		// The 16-byte pieces of a 128-byte K row (or of the query) that lane (g, t) of an MMA holds: pieces t and t + 4, the two swapped
		// for odd g.  Rows are 128 bytes apart — every row starts in bank 0 — so the eight lanes of a quarter warp (g = 2i, 2i + 1; t = 0..3)
		// read eight DIFFERENT 16-byte columns in one LDS.128.  A dot product does not care in which order k is walked as long as both
		// operands agree: B column n carries the query in the order of parity n & 1, and row m's score is C[m][m & 1].
		__device__ __forceinline__ int scorePiece( int lane, int i ) { return ( ( ( lane & 3 ) + 4 * ( ( lane >> 2 ) & 1 ) + 4 * i ) & 7 ) * 16; }

		// Scores of n K rows (128 bytes each, contiguous in shared memory) against the query: q . K[r] on the tensor cores, m16n8k16 tiles
		// of 16 rows, f16 products accumulated in f32 like the reference's ggml_vec_dot_f16 (in another order).  (The first versions did
		// this on the FMA pipe — 8 lanes per row, then 2 lanes per row with four accumulators: 130 instructions per lane and slot.)  qB = the query pieces of this lane (scorePiece).
		// The calling warp takes the tiles tile0, tile0 + tileStep, ..., TI of them at a time: their loads are issued together and their
		// four-HMMA chains interleaved.  <1>( warp, 8 ) spreads one slot over the eight warps (self-attention: one short slot);
		// <4>( 0, 1 ) gives a whole 128-row slot to one warp — the way a long run of slots is scored: whatever a warp computes on a slot,
		// the slot costs it a fixed stretch of dependent latency (barrier wait -> LDS -> chained HMMAs -> STS -> release), so eight
		// warps on eight DIFFERENT slots score a resident key memory about twice as fast as eight warps sharing every slot
		// Returns the running maximum.
		template<int TI>
		__device__ __forceinline__ float scoreRows( const uint8_t* kc, int n, int jBase, const uint4 ( &qB )[ 2 ], float* sp, int tile0, int tileStep, int lane, float lmax )
		{
			const int g = lane >> 2, odd = g & 1;
			const int p0 = scorePiece( lane, 0 ), p1 = scorePiece( lane, 1 );
			for( int tb = tile0; tb * 16 < n; tb += tileStep * TI )
			{
				uint4 a0[ TI ], a1[ TI ], b0[ TI ], b1[ TI ];
				float c[ TI ][ 4 ];
#pragma unroll
				for( int i = 0; i < TI; i++ )
				{
					// rows past n are read from row n - 1 (inside the slot) and their results dropped
					const int r0 = ( tb + i * tileStep ) * 16;
					const uint8_t* ra = kc + (size_t)min( r0 + g, n - 1 ) * 128;
					const uint8_t* rb = kc + (size_t)min( r0 + g + 8, n - 1 ) * 128;
					a0[ i ] = *reinterpret_cast<const uint4*>( ra + p0 ); a1[ i ] = *reinterpret_cast<const uint4*>( ra + p1 );
					b0[ i ] = *reinterpret_cast<const uint4*>( rb + p0 ); b1[ i ] = *reinterpret_cast<const uint4*>( rb + p1 );
					c[ i ][ 0 ] = c[ i ][ 1 ] = c[ i ][ 2 ] = c[ i ][ 3 ] = 0.0f;
				}
#pragma unroll
				for( int i = 0; i < TI; i++ ) ptx::mma_m16n8k16( c[ i ], a0[ i ].x, b0[ i ].x, a0[ i ].y, b0[ i ].y, qB[ 0 ].x, qB[ 0 ].y );
#pragma unroll
				for( int i = 0; i < TI; i++ ) ptx::mma_m16n8k16( c[ i ], a0[ i ].z, b0[ i ].z, a0[ i ].w, b0[ i ].w, qB[ 0 ].z, qB[ 0 ].w );
#pragma unroll
				for( int i = 0; i < TI; i++ ) ptx::mma_m16n8k16( c[ i ], a1[ i ].x, b1[ i ].x, a1[ i ].y, b1[ i ].y, qB[ 1 ].x, qB[ 1 ].y );
#pragma unroll
				for( int i = 0; i < TI; i++ ) ptx::mma_m16n8k16( c[ i ], a1[ i ].z, b1[ i ].z, a1[ i ].w, b1[ i ].w, qB[ 1 ].z, qB[ 1 ].w );
				if( ( lane & 3 ) == 0 )
				{
#pragma unroll
					for( int i = 0; i < TI; i++ )
					{
						const int r0 = ( tb + i * tileStep ) * 16;
						const float sa = odd ? c[ i ][ 1 ] : c[ i ][ 0 ], sb = odd ? c[ i ][ 3 ] : c[ i ][ 2 ];
						if( r0 + g < n ) { sp[ jBase + r0 + g ] = sa; lmax = fmaxf( lmax, sa ); }
						if( r0 + g + 8 < n ) { sp[ jBase + r0 + g + 8 ] = sb; lmax = fmaxf( lmax, sb ); }
					}
				}
			}
			return lmax;
		}

		// one f32 row of D elements from an exchange buffer: every lane polls its N4 16-byte pieces until no sentinel is left
		template<int D>
		__device__ __forceinline__ void pollRowF32( const float* row, float4* v, int lane )
		{
			constexpr int N4 = Cfg<D>::N4;
			const uint4* src = reinterpret_cast<const uint4*>( row );
			SpinGuard guard;
			// Probe before reading: four words at the quarter points of the row, polled with back-off, until they are written.  132
			// CTAs re-reading whole 32 KB activation blocks while they wait would by themselves saturate the L2 (one round = 4.7 MB,
			// ~10 TB/s when spinning) and starve the weight stream; the probes cost four sectors per round.  (An optimistic
			// full read first, probes only after a miss, is slower: CTAs arrive early as a rule.)
			{
				const uint32_t* w = reinterpret_cast<const uint32_t*>( row ) + ( lane & 3 ) * ( D / 4 ) + D / 8;
				unsigned ns = 32;
				while( !__all_sync( 0xffffffffu, ldPoll32( w ) != SENT32 ) )
				{
					__nanosleep( ns );
					if( ns < 256 ) ns <<= 1;
					guard.tick();
				}
			}
			uint4 u[ N4 ];
#pragma unroll
			for( int i = 0; i < N4; i++ ) u[ i ] = ldPoll( src + i * 32 + lane );
			while( true )
			{
				bool miss = false;
#pragma unroll
				for( int i = 0; i < N4; i++ )
					if( hasSent32( u[ i ] ) )
					{
						u[ i ] = ldPoll( src + i * 32 + lane );
						miss = true;
					}
				if( !miss ) break;
				guard.tick();
			}
#pragma unroll
			for( int i = 0; i < N4; i++ )
				v[ i ] = make_float4( __uint_as_float( u[ i ].x ), __uint_as_float( u[ i ].y ), __uint_as_float( u[ i ].z ), __uint_as_float( u[ i ].w ) );
		}
		// token + positional embedding row (a13: whisper.cpp:1536-1548), computed by every CTA for itself: no exchange for layer 0's input
		template<int D>
		__device__ __forceinline__ void embedRow( const __half* te, const float* pe, float4* v, int lane )
		{
			constexpr int N4 = Cfg<D>::N4;
#pragma unroll
			for( int i = 0; i < N4; i++ )
			{
				const uint2 h = *reinterpret_cast<const uint2*>( te + ( i * 32 + lane ) * 4 );
				const float4 p = *reinterpret_cast<const float4*>( pe + ( i * 32 + lane ) * 4 );
				const float2 a = __half22float2( *reinterpret_cast<const __half2*>( &h.x ) );
				const float2 b = __half22float2( *reinterpret_cast<const __half2*>( &h.y ) );
				v[ i ] = make_float4( a.x + p.x, a.y + p.y, b.x + p.z, b.y + p.w );
			}
		}
		// LayerNorm of one row held in registers (one warp per row) -> f16 activations; keeps this CTA's residual rows
		template<int D>
		__device__ __forceinline__ void normRow( float4* v, const float* gamma, const float* beta, __half* dst, float* xresRow, int r0, int nr, int lane )
		{
			constexpr int N4 = Cfg<D>::N4;
			if( nr > 0 )
			{
#pragma unroll
				for( int i = 0; i < N4; i++ )
				{
					const int e0 = ( i * 32 + lane ) * 4;
					if( e0 + 3 >= r0 && e0 < r0 + nr )
					{
						const float f[ 4 ] = { v[ i ].x, v[ i ].y, v[ i ].z, v[ i ].w };
#pragma unroll
						for( int k = 0; k < 4; k++ )
						{
							const int r = e0 + k - r0;
							if( r >= 0 && r < nr ) xresRow[ r ] = f[ k ];
						}
					}
				}
			}
			float s = 0.0f;
#pragma unroll
			for( int i = 0; i < N4; i++ ) s += v[ i ].x + v[ i ].y + v[ i ].z + v[ i ].w;
			const float mean = ptx::warp_sum( s ) / (float)D;
			float sq = 0.0f;
#pragma unroll
			for( int i = 0; i < N4; i++ )
			{
				v[ i ].x -= mean; v[ i ].y -= mean; v[ i ].z -= mean; v[ i ].w -= mean;
				sq += v[ i ].x * v[ i ].x + v[ i ].y * v[ i ].y + v[ i ].z * v[ i ].z + v[ i ].w * v[ i ].w;
			}
			const float rstd = 1.0f / sqrtf( ptx::warp_sum( sq ) / (float)D + 1e-5f );
			const float4* g4 = reinterpret_cast<const float4*>( gamma );
			const float4* b4 = reinterpret_cast<const float4*>( beta );
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
		// B rows of D ready f16 activations (attention output, GELU output) from an exchange buffer -> shared memory, one warp per row
		// (two for B > 8).  Split in three so that fc2 can issue the loads of its next K chunk before the MMAs of the current one:
		//   f16Issue: optimistic loads into registers;  f16Verify: wait (probe + back-off, see pollRowF32) until no sentinel is left;
		//   f16Put: registers -> the activation rows in shared memory.
		template<int D>
		struct F16Rows
		{
			static constexpr int V8 = D / 8;                   // 16-byte pieces per row
			static constexpr int NI = ( V8 + 31 ) / 32;
			uint4 u[ 2 ][ NI ];
		};
		template<int D>
		__device__ __forceinline__ void f16Probe( const __half* src, size_t colStride, int B, int warp, int lane )
		{
			for( int c = warp; c < B; c += FL_WARPS )
			{
				const uint32_t* w = reinterpret_cast<const uint32_t*>( src + (size_t)c * colStride ) + ( lane & 3 ) * ( D / 8 ) + D / 16;
				SpinGuard guard;
				unsigned ns = 32;
				while( !__all_sync( 0xffffffffu, !hasSent16w( ldPoll32( w ) ) ) )
				{
					__nanosleep( ns );
					if( ns < 256 ) ns <<= 1;
					guard.tick();
				}
			}
		}
		// PL = -1: both register planes, plane q = column warp + 8 q (B > 8).  PL = 0 / 1: ONE plane for column `warp` (B <= 8) — the
		// other plane is then free to hold the NEXT chunk, so that fc2 keeps two of its four K chunks in flight.
		template<int D, int PL>
		__device__ __forceinline__ void f16Issue( F16Rows<D>& rg, const __half* src, size_t colStride, int B, int warp, int lane )
		{
			using R = F16Rows<D>;
#pragma unroll
			for( int q = 0; q < 2; q++ )
			{
				if( PL >= 0 && q != PL ) continue;
				const int c = PL >= 0 ? warp : warp + q * FL_WARPS;
				if( c >= B ) continue;
				const __half* row = src + (size_t)c * colStride;
#pragma unroll
				for( int k = 0; k < R::NI; k++ )
				{
					const int i = k * 32 + lane;
					rg.u[ q ][ k ] = make_uint4( 0, 0, 0, 0 );
					if( i < R::V8 ) rg.u[ q ][ k ] = ldPoll( row + i * 8 );
				}
			}
		}
		template<int D, int PL>
		__device__ __forceinline__ void f16Verify( F16Rows<D>& rg, const __half* src, size_t colStride, int B, int warp, int lane )
		{
			using R = F16Rows<D>;
#pragma unroll
			for( int q = 0; q < 2; q++ )
			{
				if( PL >= 0 && q != PL ) continue;
				const int c = PL >= 0 ? warp : warp + q * FL_WARPS;
				if( c >= B ) continue;
				const __half* row = src + (size_t)c * colStride;
				SpinGuard guard;
				bool first = true;
				while( true )
				{
					bool miss = false;
#pragma unroll
					for( int k = 0; k < R::NI; k++ ) miss |= ( k * 32 + lane < R::V8 ) && hasSent16( rg.u[ q ][ k ] );
					if( !__any_sync( 0xffffffffu, miss ) ) break;
					if( first )
					{
						first = false;
						const uint32_t* w = reinterpret_cast<const uint32_t*>( row ) + ( lane & 3 ) * ( D / 8 ) + D / 16;
						unsigned ns = 32;
						while( !__all_sync( 0xffffffffu, !hasSent16w( ldPoll32( w ) ) ) )
						{
							__nanosleep( ns );
							if( ns < 256 ) ns <<= 1;
							guard.tick();
						}
					}
#pragma unroll
					for( int k = 0; k < R::NI; k++ )
					{
						const int i = k * 32 + lane;
						if( i < R::V8 && hasSent16( rg.u[ q ][ k ] ) ) rg.u[ q ][ k ] = ldPoll( row + i * 8 );
					}
					guard.tick();
				}
			}
		}
		template<int D, int PL>
		__device__ __forceinline__ void f16Put( const F16Rows<D>& rg, int B, uint8_t* act, int warp, int lane )
		{
			using R = F16Rows<D>;
			constexpr int RS = Cfg<D>::RS;
#pragma unroll
			for( int q = 0; q < 2; q++ )
			{
				if( PL >= 0 && q != PL ) continue;
				const int c = PL >= 0 ? warp : warp + q * FL_WARPS;
				if( c >= B ) continue;
#pragma unroll
				for( int k = 0; k < R::NI; k++ )
				{
					const int i = k * 32 + lane;
					if( i < R::V8 ) *reinterpret_cast<uint4*>( act + (size_t)c * RS + i * 16 ) = rg.u[ q ][ k ];
				}
			}
		}

		enum { EP_QKV = 0, EP_RESID = 1, EP_QSCALE = 2, EP_GELU = 3, EP_LOGITS = 4 };
		// -----------------------------------------------------------------------------------------------------------
		// TIMED = the debug instantiation with the (id, %globaltimer) marks; the production instantiation carries none of that code
		// (about 700 SASS instructions: with them the kernel outgrows the 128 KB instruction cache and every phase slows down)
		template<int D, bool TIMED>
		__global__ void __launch_bounds__( FL_THREADS, 1 )
			decode_flow_kernel( const FlowArgs a )
		{
			using C = Cfg<D>;
			constexpr int RS = C::RS, SLOT = C::SLOT, CR = C::CR;
			extern __shared__ __align__( 128 ) uint8_t fl_smem[];
			const int NS = a.NS, ncols = a.ncols;
			const SmemLayout lay = smemLayout( SLOT, RS, NS, ncols );
			uint8_t* const ring = fl_smem;
			uint8_t* const act = fl_smem + lay.act;
			float* const red = reinterpret_cast<float*>( fl_smem + lay.red );
			float* const sp = reinterpret_cast<float*>( fl_smem + lay.sp );
			float* const sbias = reinterpret_cast<float*>( fl_smem + lay.bias );
			float* const xres = reinterpret_cast<float*>( fl_smem + lay.xres );
			float* const so = reinterpret_cast<float*>( fl_smem + lay.so );
			float* const sred = reinterpret_cast<float*>( fl_smem + lay.sred );
			uint8_t* const sqkv = fl_smem + lay.qkv;
			uint64_t* const full = reinterpret_cast<uint64_t*>( fl_smem + lay.bars );
			uint64_t* const empty = full + FL_NSMAX;

			const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
			const int cta = blockIdx.x, G = gridDim.x;
			if( tid == 0 )
			{
				for( int i = 0; i < NS; i++ )
				{
					ptx::mbar_init( full + i, 1 );
					ptx::mbar_init( empty + i, FL_WARPS );
				}

				ptx::fence_barrier_init();
			}
			__syncthreads();

			const unsigned epoch = *reinterpret_cast<const volatile unsigned*>( a.ctrl + 1 );
			const int set = (int)( epoch & 1u );
			const int B = a.B, H = a.H, T = a.T, L = a.L;
			int nPast = *a.dNPast;              // read once: the sampler advances it after this launch
			nPast = max( 0, min( nPast, a.nTextCtx - 1 ) );
			const int nkvOld = nPast;           // rows of earlier tokens in the self-KV cache
			const int parts = a.refThreads;
			const size_t colsD = (size_t)a.maxB * D;
			const size_t exLayer = colsD * 32;
			const FlowGeom& g = a.g;
			const int r1 = cta * g.R1, n1 = max( 0, min( g.R1, D - r1 ) );
			const int r3 = cta * g.R3, n3 = max( 0, min( g.R3, 3 * D - r3 ) );
			const int r4 = cta * g.R4, n4 = max( 0, min( g.R4, 4 * D - r4 ) );
			const int rv = cta * g.RV, nv = max( 0, min( g.RV, a.nVocab - rv ) );
			// V rows travel in (round, group) order: the four 64-thread groups of the consumers each own PG consecutive parts (one part
			// each up to 4 reference threads), and one slot carries RR rows of each of a group's parts
			const int NG = min( parts, 4 );
			const int PG = ( parts + NG - 1 ) / NG;
			const int RR = CR / PG;
			const int nKcSelf = ( nkvOld + CR - 1 ) / CR;
			const int dcSelf = ( nkvOld + 1 + parts - 1 ) / parts;
			const int roundsSelf = ( dcSelf + RR - 1 ) / RR;
			const int nKcCross = ( T + CR - 1 ) / CR;
			const int dcCross = ( T + parts - 1 ) / parts;
			const int roundsCross = ( dcCross + RR - 1 ) / RR;

			// =========================================================================================================
			// producer warp: everything that does not depend on this step, in consumption order, as far ahead as the ring allows
			// =========================================================================================================
			if( warp == FL_WARPS )
			{
				int pSlot = 0;
				uint32_t pPar = 0;
				bool wrapped = false;
				uint64_t* bar = nullptr;
				auto begin = [ & ]( uint32_t bytes ) -> uint8_t* {
					uint8_t* dst = ring + (size_t)pSlot * SLOT;
					bar = full + pSlot;
					if( lane == 0 )
					{
						if( wrapped ) mbarWaitLong( empty + pSlot, pPar ^ 1u );
						if( bytes ) ptx::mbar_expect_tx( bar, bytes );
						else ptx::mbar_arrive( bar );
					}
					__syncwarp();
					if( ++pSlot == NS ) { pSlot = 0; pPar ^= 1u; wrapped = true; }
					return dst;
				};
				// debug (TIMED): when the producer ISSUES selected loads, pairs 2000.. of the timing buffer, id = 100000 + 100 * layer + code
				int pMark = 0;
				auto pmark = [ & ]( int il, int code ) {
					if( !TIMED || !a.timing || cta != a.timingCta ) return;
					if( lane == 0 && pMark < 300 )
					{
						a.timing[ 2 * ( 2000 + pMark ) ] = (unsigned long long)( 100000 + 100 * il + code );
						a.timing[ 2 * ( 2000 + pMark ) + 1 ] = ptx::globaltimer();
					}
					pMark++;
				};
				auto sendParams = [ & ]( const float* gm, const float* bt, const float* slab, int slabFloats ) {
					uint8_t* dst = begin( (uint32_t)( 2 * D * 4 + slabFloats * 4 ) );
					if( lane == 0 ) ptx::bulk_load_1d( dst, gm, D * 4, bar );
					if( lane == 1 ) ptx::bulk_load_1d( dst + D * 4, bt, D * 4, bar );
					if( lane == 2 && slabFloats ) ptx::bulk_load_1d( dst + 2 * D * 4, slab, (uint32_t)slabFloats * 4, bar );
				};
				auto sendWeights = [ & ]( const __half* W, int K, int row0, int nRows, int kChunks ) {
					const int nUnits = ( nRows + 7 ) >> 3;
					for( int u0 = 0; u0 < nUnits; u0 += 4 )
					{
						const int nb = min( 4, nUnits - u0 );
						for( int kc = 0; kc < kChunks; kc++ )
							for( int u = 0; u < nb; u++ )
							{
								const int rows = min( 8, nRows - ( u0 + u ) * 8 );
								uint8_t* dst = begin( (uint32_t)rows * D * 2 );
								if( lane < rows )
									ptx::bulk_load_1d( dst + lane * RS, W + (size_t)( row0 + ( u0 + u ) * 8 + lane ) * K + (size_t)kc * D, D * 2, bar );
							}
					}
				};
				auto sendKv = [ & ]( const __half* base, int j0, int n ) {
					uint8_t* dst = begin( (uint32_t)( n > 0 ? n * 128 : 0 ) );
					if( lane == 0 && n > 0 ) ptx::bulk_load_1d( dst, base + (size_t)j0 * 64, (uint32_t)n * 128, bar );
				};
				// one slot of V rows for group q in round i: rows [pp*dc + i*RR, ...) of each of the group's parts pp, clipped to the part and to nOld
				auto sendV = [ & ]( const __half* base, int q, int i, int dc, int nOld ) {
					int myJ0 = 0, myN = 0, total = 0;
					for( int k = 0; k < PG; k++ )
					{
						const int pp = q * PG + k;
						const int j0 = pp * dc + i * RR;
						const int j1 = min( j0 + RR, min( ( pp + 1 ) * dc, nOld ) );
						const int n = ( pp < parts && j1 > j0 ) ? j1 - j0 : 0;
						total += n;
						if( k == lane ) { myJ0 = j0; myN = n; }
					}
					uint8_t* dst = begin( (uint32_t)total * 128 );
					if( myN > 0 ) ptx::bulk_load_1d( dst + (size_t)lane * RR * 128, base + (size_t)myJ0 * 64, (uint32_t)myN * 128, bar );
				};
				for( int il = 0; il < L; il++ )
				{
					const DecStepLayer& Lr = a.layers[ il ];
					sendParams( Lr.ln1g, Lr.ln1b, Lr.biasSlab + (size_t)cta * g.slabFloats, g.slabFloats );
					sendWeights( Lr.wqkv, D, r3, n3, 1 );
					for( int unit = cta; unit < B * H; unit += G )
					{
						const size_t hb = (size_t)unit * a.nTextCtx * 64;   // unit = b * H + h
						for( int ci = 0; ci < nKcSelf; ci++ ) sendKv( Lr.kCache + hb, ci * CR, min( CR, nkvOld - ci * CR ) );
						for( int i = 0; i < roundsSelf; i++ )
							for( int q = 0; q < NG; q++ ) sendV( Lr.vCache + hb, q, i, dcSelf, nkvOld );
					}
					pmark( il, 1 );
					sendWeights( Lr.wo, D, r1, n1, 1 );
					pmark( il, 2 );
					sendParams( Lr.lncg, Lr.lncb, nullptr, 0 );
					sendWeights( Lr.wcq, D, r1, n1, 1 );
					for( int unit = cta; unit < B * H; unit += G )
					{
						const size_t hb = (size_t)unit * T * 64;
						for( int ci = 0; ci < nKcCross; ci++ )
						{
							if( ci == 0 || ci == 4 || ci == 8 ) pmark( il, 3 + ci / 4 );
							sendKv( Lr.crossK + hb, ci * CR, min( CR, T - ci * CR ) );
						}
						pmark( il, 6 );
						for( int i = 0; i < roundsCross; i++ )
							for( int q = 0; q < NG; q++ ) sendV( Lr.crossV + hb, q, i, dcCross, T );
						pmark( il, 7 );
					}
					sendWeights( Lr.wco, D, r1, n1, 1 );
					pmark( il, 8 );
					sendParams( Lr.ln3g, Lr.ln3b, nullptr, 0 );
					sendWeights( Lr.w1, D, r4, n4, 1 );
					sendWeights( Lr.w2, 4 * D, r1, n1, 4 );
				}
				sendParams( a.lnfg, a.lnfb, nullptr, 0 );
				sendWeights( a.tokEmb, D, rv, nv, 1 );
				return;
			}

			// =========================================================================================================
			// consumer warps
			// =========================================================================================================
			int cSlot = 0;
			uint32_t cPar = 0;
			auto slotAt = [ & ]( int k, uint32_t& par ) -> int {
				int idx = cSlot + k;
				par = cPar;
				if( idx >= NS ) { idx -= NS; par ^= 1u; }
				return idx;
			};
			auto waitSlot = [ & ]( int k ) -> uint8_t* {
				uint32_t par;
				const int idx = slotAt( k, par );
				mbarWaitLong( full + idx, par );
				return ring + (size_t)idx * SLOT;
			};
			// Every consumer warp releases every slot exactly once, after its last read.  `observe`: this warp may not have waited for
			// the slot's data itself (V rows are read by the two warps of one chain only) — it does so now, so that every warp sees
			// every phase of every `full` barrier complete and a later parity wait can never match a phase it skipped.
			auto releaseSlots = [ & ]( int n, bool observe = false ) {
				__syncwarp();
				if( lane < n )   // lane k takes slot k (n <= 4): the waits and arrives of a V round overlap instead of queueing behind lane 0
				{
					uint32_t par;
					const int idx = slotAt( lane, par );
					if( observe ) mbarWaitLong( full + idx, par );
					ptx::mbar_arrive( empty + idx );
				}
				cSlot += n;
				if( cSlot >= NS ) { cSlot -= NS; cPar ^= 1u; }
			};
			// debug: (id, %globaltimer) pairs of one CTA.  ids: 0 = kernel start, 100 * (phase + 1) + sub for the sub-steps of a phase
			// (sub 0 = phase done; 1 = inputs arrived and staged; 2 = first weight slot landed; 3 = MMAs done; 4 = reduced + stored)
			int markIdx = 0;
			const int markCta = ( TIMED && a.timing ) ? a.timingCta : -1;
			auto markId = [ & ]( int id ) {
				if( !TIMED ) return;
				if( cta == markCta && tid == 0 && markIdx < 2000 )
				{
					a.timing[ 2 * markIdx ] = (unsigned long long)id;
					a.timing[ 2 * markIdx + 1 ] = ptx::globaltimer();
				}
				markIdx++;
			};
			int curPhase = 0;
			auto sub = [ & ]( int k ) { if( TIMED && markCta >= 0 ) markId( 100 * ( curPhase + 1 ) + k ); };
			auto mark = [ & ]() { if( TIMED ) { markId( 100 * ( curPhase + 1 ) ); curPhase++; } };
			markId( 0 );

			const int gq = lane >> 2, tq = lane & 3;
			const bool twoTiles = B > 8;
			const float qkScale = 0.35355339059327379f;   // 64^-1/4 (whisper.cpp:1588, 1595, 1700)

			// The step is ONE loop over (layer, phase) with a single copy of the weight-streaming GEMV code and a single copy of the
			// attention code; a switch only fills in their operands.  (The first version of this kernel instantiated the GEMV seven
			// times: 16 K SASS instructions = 256 KB, every phase started with a cold instruction cache.)
			enum { PH_QKV = 0, PH_SELF = 1, PH_O = 2, PH_CQ = 3, PH_CROSS = 4, PH_CO = 5, PH_FC1 = 6, PH_FC2 = 7, PH_COUNT = 8 };
#pragma unroll 1
			for( int il = 0; il <= L; il++ )
			{
				const bool last = il == L;                // final LayerNorm + logits (a17)
				const DecStepLayer& Lr = a.layers[ last ? L - 1 : il ];
				uint8_t* const exb = a.exch + ( (size_t)set * L + ( last ? L - 1 : il ) ) * exLayer;
				float* const x1 = reinterpret_cast<float*>( exb );
				float* const x2 = x1 + colsD;
				float* const x3 = x2 + colsD;
				__half* const hbase = reinterpret_cast<__half*>( exb + colsD * 12 );
				__half* const qh = hbase;
				__half* const knew = hbase + colsD;
				__half* const vnew = hbase + 2 * colsD;
				__half* const attn1 = hbase + 3 * colsD;
				__half* const cq = hbase + 4 * colsD;
				__half* const attn2 = hbase + 5 * colsD;
				__half* const hbuf = hbase + 6 * colsD;
				const float* xprev = nullptr;             // the previous layer's output (nullptr: embed on the spot)
				if( il > 0 && !last ) xprev = reinterpret_cast<const float*>( a.exch + ( (size_t)set * L + il - 1 ) * exLayer ) + 2 * colsD;

#pragma unroll 1
				for( int ph = 0; ph < PH_COUNT; ph++ )
				{
					if( ph == PH_SELF || ph == PH_CROSS )
					{
						// =====================================================================================================
						// attention of one new query per (chunk, head) over f16 K/V rows: the self-KV cache plus this step's own row
						// (a14), or the encoder's cross memories (a15).  K rows stream through the ring in runs of CR rows and are
						// scored as they land; V rows come in (round, part) order — part p of the reference's `parts` threads owns the
						// key range [p*dc, (p+1)*dc) and accumulates it in an f16 chain (ggml.c:4680-4722).
						// =====================================================================================================
						const bool self = ph == PH_SELF;
						const int nOld = self ? nkvOld : T;           // rows that come through the ring
						const int n = nOld + ( self ? 1 : 0 );
						const __half* qsrc = self ? qh : cq;
						__half* dst = self ? attn1 : attn2;
						const int nKc = ( nOld + CR - 1 ) / CR;
						const int dc = ( n + parts - 1 ) / parts;
						const int rounds = ( dc + RR - 1 ) / RR;
#pragma unroll 1
						for( int unit = cta; unit < B * H; unit += G )
						{
							const int b = unit / H, h = unit - b * H;
							const size_t vo = (size_t)b * D + h * 64;
							if( tid < ( self ? 24 : 8 ) )
							{
								const int arr = tid >> 3, piece = tid & 7;
								const __half* src = ( arr == 0 ? qsrc : arr == 1 ? knew : vnew ) + vo + piece * 8;
								uint4 u = ldPoll( src );
								SpinGuard guard;
								while( hasSent16( u ) ) { __nanosleep( 64 ); u = ldPoll( src ); guard.tick(); }
								reinterpret_cast<uint4*>( sqkv )[ tid ] = u;
							}
							consumerSync();
							sub( 1 );
							uint4 qf[ 2 ];    // this lane's two pieces of the (f16) query, in the order its K pieces come in (scorePiece)
							qf[ 0 ] = *reinterpret_cast<const uint4*>( sqkv + scorePiece( lane, 0 ) );
							qf[ 1 ] = *reinterpret_cast<const uint4*>( sqkv + scorePiece( lane, 1 ) );
							float lmax = -INFINITY;
							if( nKc <= 1 )
							{
								// one short slot (self-attention): its tiles spread over the warps
								for( int ci = 0; ci < nKc; ci++ )
								{
									const uint8_t* kc = waitSlot( 0 );
									lmax = scoreRows<1>( kc, min( CR, nOld - ci * CR ), ci * CR, qf, sp, warp, FL_WARPS, lane, lmax );
									releaseSlots( 1 );
								}
							}
							else
							{
								// a run of slots, eight at a time: warp w scores slot w of the group alone, then every warp releases all of them
								const int GS = min( FL_WARPS, NS );   // a group's slots are all in the ring at once
#pragma unroll 1
								for( int c0 = 0; c0 < nKc; c0 += GS )
								{
									const int ng = min( GS, nKc - c0 );
									if( warp < ng )
									{
										const uint8_t* kc = waitSlot( warp );
										lmax = scoreRows<4>( kc, min( CR, nOld - ( c0 + warp ) * CR ), ( c0 + warp ) * CR, qf, sp, 0, 1, lane, lmax );
									}
									releaseSlots( ng, true );
									if( TIMED && !self ) sub( 10 + c0 / GS );
								}
							}
							if( self ) lmax = scoreRows<1>( sqkv + 128, 1, nOld, qf, sp, warp, FL_WARPS, lane, lmax );   // this step's own K row
							sub( 2 );
							softmaxRow<consumerSync>( sp, n, lmax, sred, tid, warp, lane );
							sub( 3 );
							{
								const int q = tid >> 6, e = tid & 63;
								float y[ 4 ] = { 0.0f, 0.0f, 0.0f, 0.0f };
#pragma unroll 1
								for( int i = 0; i < rounds; i++ )
								{
									if( q < NG )
									{
										int j0[ 4 ], nk[ 4 ], nmax = 0;
#pragma unroll
										for( int k = 0; k < 4; k++ )
										{
											const int pp = q * PG + k;
											j0[ k ] = pp * dc + i * RR;
											const int j1 = min( j0[ k ] + RR, min( ( pp + 1 ) * dc, nOld ) );
											nk[ k ] = ( k < PG && pp < parts && j1 > j0[ k ] ) ? j1 - j0[ k ] : 0;
											nmax = max( nmax, nk[ k ] );
										}
										if( nmax > 0 )
										{
											const __half* vp = reinterpret_cast<const __half*>( waitSlot( q ) ) + e;
											if( PG == 1 ) y[ 0 ] = chainRows( y[ 0 ], sp + j0[ 0 ], vp, nk[ 0 ] );
											else chainSide( y, sp, vp, j0, nk, RR );
										}
									}
									releaseSlots( NG, true );
									if( TIMED && !self ) sub( 40 + i );
								}
								if( self )
								{
									// this step's own V row closes the chain of the part whose key range it falls into
									const int pOwn = nOld / dc;
									if( pOwn < parts && q == pOwn / PG )
									{
										const float x = __half2float( reinterpret_cast<const __half*>( sqkv + 256 )[ e ] );
										const float pj = sp[ nOld ];
										const int ko = pOwn - q * PG;
#pragma unroll
										for( int k = 0; k < 4; k++ )
											if( k == ko )
												y[ k ] = chainStep( y[ k ], x, pj );
									}
								}
#pragma unroll
								for( int k = 0; k < 4; k++ )
								{
									const int pp = q * PG + k;
									if( q < NG && k < PG && pp < parts ) so[ pp * 64 + e ] = y[ k ];
								}
							}
							sub( 4 );
							consumerSync();
							if( tid < 64 )
							{
								float acc = so[ tid ];
								for( int k = 1; k < parts; k++ ) acc += so[ k * 64 + tid ];
								stX16( dst + vo + tid, __float2half_rn( acc ) );
							}
							consumerSync();
						}
						mark();
						continue;
					}

					// =========================================================================================================
					// weight-streaming GEMV of this CTA's rows: out[col][n] = sum_k W[n][k] * act[col][k]
					// =========================================================================================================
					int epi = EP_RESID, row0 = r1, nRows = n1, KC = 1, ld = D, biasOff = 0;
					bool useLN = false;
					const float* lnSrc = nullptr;
					const __half* hSrc = nullptr;
					size_t hStride = D;
					float scale = 1.0f;
					float* outF32 = nullptr;
					__half* outF16 = nullptr;
					if( last )
					{
						epi = EP_LOGITS; row0 = rv; nRows = nv; useLN = true; lnSrc = x3; outF32 = a.logits; ld = a.nVocab; biasOff = -1;
					}
					else switch( ph )
					{
					case PH_QKV:    // LN1 + (Q | K | V): K/V rows appended to the f16 cache (a14)
						epi = EP_QKV; row0 = r3; nRows = n3; useLN = true; lnSrc = xprev; scale = qkScale; outF16 = qh; biasOff = g.oQkv;
						break;
					case PH_O:      // self-attention out projection + residual
						hSrc = attn1; outF32 = x1; biasOff = g.oO;
						break;
					case PH_CQ:     // LN + cross-attention query (a15)
						epi = EP_QSCALE; useLN = true; lnSrc = x1; scale = qkScale; outF16 = cq; biasOff = g.oCq;
						break;
					case PH_CO:     // cross-attention out projection + residual
						hSrc = attn2; outF32 = x2; biasOff = g.oCo;
						break;
					case PH_FC1:    // LN + fc1 + GELU (a16)
						epi = EP_GELU; row0 = r4; nRows = n4; useLN = true; lnSrc = x2; outF16 = hbuf; ld = 4 * D; biasOff = g.oFc1;
						break;
					default:        // PH_FC2: fc2 + residual, K = 4D walked in four D-wide chunks
						hSrc = hbuf; hStride = (size_t)4 * D; KC = 4; outF32 = x3; biasOff = g.oFc2;
						break;
					}
					const float* bias = biasOff >= 0 ? sbias + biasOff : nullptr;


					if( useLN )
					{
						// LayerNorm gamma | beta (| this layer's bias slab) arrive through the ring
						const uint8_t* pr = waitSlot( 0 );
						if( ph == PH_QKV && !last )
							for( int i = tid; i < g.slabFloats; i += FL_CONSUMERS ) sbias[ i ] = reinterpret_cast<const float*>( pr + 2 * D * 4 )[ i ];
						if( nRows > 0 )
						{
							const float* gamma = reinterpret_cast<const float*>( pr );
							const float* beta = gamma + D;
							const bool embed = !last && ph == PH_QKV && il == 0;
							for( int c = warp; c < B; c += FL_WARPS )
							{
								float4 v[ C::N4 ];
								if( embed ) embedRow<D>( a.tokEmb + (size_t)a.tokens[ c ] * D, a.decPos + (size_t)nPast * D, v, lane );
								else pollRowF32<D>( lnSrc + (size_t)c * D, v, lane );
								normRow<D>( v, gamma, beta, reinterpret_cast<__half*>( act + (size_t)c * RS ), xres + c * 16, r1, n1, lane );
							}
						}
						consumerSync();
						sub( 1 );
						releaseSlots( 1 );
					}
					F16Rows<D> hr;
					if( !useLN && nRows > 0 )
					{
						// (fc2: the first of its four K chunks; the others are fetched behind the MMAs below)
						f16Probe<D>( hSrc, hStride, B, warp, lane );
						f16Issue<D, -1>( hr, hSrc, hStride, B, warp, lane );
						f16Verify<D, -1>( hr, hSrc, hStride, B, warp, lane );
						f16Put<D, -1>( hr, B, act, warp, lane );
						consumerSync();
						sub( 1 );
					}

					const int nUnits = ( nRows + 7 ) >> 3;
#pragma unroll 1
					for( int u0 = 0; u0 < nUnits; u0 += 4 )
					{
						const int nb = min( 4, nUnits - u0 );
						float acc0[ 4 ][ 4 ], acc1[ 4 ][ 4 ];
#pragma unroll
						for( int u = 0; u < 4; u++ )
#pragma unroll
							for( int i = 0; i < 4; i++ ) { acc0[ u ][ i ] = 0.0f; acc1[ u ][ i ] = 0.0f; }
#pragma unroll 1
						for( int kc = 0; kc < KC; kc++ )
						{
							if( kc > 0 )
							{
								// this chunk's rows were requested before the previous chunk's MMAs
								f16Verify<D, -1>( hr, hSrc + (size_t)kc * D, hStride, B, warp, lane );
								consumerSync();   // the previous chunk's MMAs have read `act`
								f16Put<D, -1>( hr, B, act, warp, lane );
								consumerSync();
							}
							if( kc + 1 < KC ) f16Issue<D, -1>( hr, hSrc + (size_t)( kc + 1 ) * D, hStride, B, warp, lane );
#pragma unroll
							for( int u = 0; u < 4; u++ )
							{
								if( u < nb )
								{
									// (all units of a pass side by side — wait for their slots together, interleave their HMMA chains — is
									// slower: the weights of fc1 / fc2 arrive while the first units compute)
									const uint8_t* w = waitSlot( 0 );
									if( u == 0 && kc == 0 && u0 == 0 ) sub( 2 );
									const uint8_t* wb = w + (size_t)gq * RS + tq * 16;
									const uint8_t* xb0 = act + (size_t)gq * RS + tq * 16;
									const uint8_t* xb1 = act + (size_t)( gq + 8 ) * RS + tq * 16;
#pragma unroll
									for( int s = 0; s < C::SPW; s++ )
									{
										const int st = warp + FL_WARPS * s;
										if( st < C::STEPS )
										{
											const uint4 wv = *reinterpret_cast<const uint4*>( wb + st * 64 );
											const uint4 x0 = *reinterpret_cast<const uint4*>( xb0 + st * 64 );
											ptx::mma_m16n8k16_rows8( acc0[ u ], wv.x, wv.y, x0.x, x0.y );
											ptx::mma_m16n8k16_rows8( acc0[ u ], wv.z, wv.w, x0.z, x0.w );
											if( twoTiles )
											{
												const uint4 x1v = *reinterpret_cast<const uint4*>( xb1 + st * 64 );
												ptx::mma_m16n8k16_rows8( acc1[ u ], wv.x, wv.y, x1v.x, x1v.y );
												ptx::mma_m16n8k16_rows8( acc1[ u ], wv.z, wv.w, x1v.z, x1v.w );
											}
										}
									}
									releaseSlots( 1 );
								}
							}
						}
						if( u0 == 0 ) sub( 3 );
						// cross-warp reduction: red[u][warp][row g][col]
#pragma unroll
						for( int u = 0; u < 4; u++ )
						{
							if( u < nb )
							{
								float* my = red + ( ( u * FL_WARPS + warp ) * 8 + gq ) * ncols;
								my[ 2 * tq ] = acc0[ u ][ 0 ];
								my[ 2 * tq + 1 ] = acc0[ u ][ 1 ];
								if( twoTiles ) { my[ 8 + 2 * tq ] = acc1[ u ][ 0 ]; my[ 8 + 2 * tq + 1 ] = acc1[ u ][ 1 ]; }
							}
						}
						consumerSync();
						for( int idx = tid; idx < nb * B * 8; idx += FL_CONSUMERS )
						{
							const int u = idx / ( B * 8 );
							const int rem = idx - u * B * 8;
							const int c = rem >> 3, r = rem & 7;
							const int rl = ( u0 + u ) * 8 + r;     // row within this CTA's range
							if( rl >= nRows ) continue;
							const int nn0 = row0 + rl;
							float v = 0.0f;
#pragma unroll
							for( int w = 0; w < FL_WARPS; w++ ) v += red[ ( ( u * FL_WARPS + w ) * 8 + r ) * ncols + c ];
							const float bs = bias ? bias[ rl ] : 0.0f;
							switch( epi )
							{
							case EP_QKV:
							{
								const int which = nn0 / D;
								const int nn = nn0 - which * D;
								if( which == 0 ) stX16( outF16 + (size_t)c * D + nn, __float2half_rn( ( v + bs ) * scale ) );
								else
								{
									const int hh = nn >> 6, e = nn & 63;
									const size_t off = ( ( (size_t)c * H + hh ) * a.nTextCtx + nPast ) * 64 + e;
									if( which == 1 )
									{
										const __half kv = __float2half_rn( v * scale );
										Lr.kCache[ off ] = kv;
										stX16( knew + (size_t)c * D + nn, kv );
									}
									else
									{
										const __half vv = __float2half_rn( v + bs );
										Lr.vCache[ off ] = vv;
										stX16( vnew + (size_t)c * D + nn, vv );
									}
								}
								break;
							}
							case EP_RESID:
								stX32( outF32 + (size_t)c * D + nn0, v + bs + xres[ c * 16 + rl ] );
								break;
							case EP_QSCALE:
								stX16( outF16 + (size_t)c * D + nn0, __float2half_rn( ( v + bs ) * scale ) );
								break;
							case EP_GELU:
								stX16( outF16 + (size_t)c * ld + nn0, __float2half_rn( ptx::gelu_f16_semantics( v + bs ) ) );
								break;
							default:
								outF32[ (size_t)c * ld + nn0 ] = v;
								break;
							}
						}
						if( u0 == 0 ) sub( 4 );
						if( u0 + 4 < nUnits ) consumerSync();   // `red` is rewritten by the next batch
					}
					mark();
					if( last ) break;
				}
				if( last ) break;
				// ---- re-arm this layer's buffers of the idle set (their readers finished with the previous launch) ----
				{
					uint4* dst = reinterpret_cast<uint4*>( a.exch + ( (size_t)( set ^ 1 ) * L + il ) * exLayer );
					const size_t n16 = exLayer / 16;
					const size_t per = ( n16 + G - 1 ) / G;
					const size_t lo = (size_t)cta * per;
					for( size_t i = tid; i < per && lo + i < n16; i += FL_CONSUMERS ) dst[ lo + i ] = make_uint4( SENT32, SENT32, SENT32, SENT32 );
				}
			}
			// the last CTA to finish flips the exchange set for the next launch
			consumerSync();
			if( tid == 0 )
			{
				const unsigned old = atomicAdd( a.ctrl, 1u );
				if( old == (unsigned)G - 1u )
				{
					a.ctrl[ 0 ] = 0u;
					a.ctrl[ 1 ] = epoch + 1u;
				}
			}
		}

		__global__ void flow_bias_slab_kernel( float* slab, FlowGeom g, int d, const float* bqkv, const float* bo, const float* bcq, const float* bco,
			const float* b1, const float* b2 )
		{
			const int c = blockIdx.x;
			for( int i = threadIdx.x; i < g.slabFloats; i += blockDim.x )
			{
				const float* src;
				int r, R, nOut;
				if( i < g.oO ) { src = bqkv; r = i - g.oQkv; R = g.R3; nOut = 3 * d; }
				else if( i < g.oCq ) { src = bo; r = i - g.oO; R = g.R1; nOut = d; }
				else if( i < g.oCo ) { src = bcq; r = i - g.oCq; R = g.R1; nOut = d; }
				else if( i < g.oFc1 ) { src = bco; r = i - g.oCo; R = g.R1; nOut = d; }
				else if( i < g.oFc2 ) { src = b1; r = i - g.oFc1; R = g.R4; nOut = 4 * d; }
				else { src = b2; r = i - g.oFc2; R = g.R1; nOut = d; }
				const int n = c * R + r;
				slab[ (size_t)c * g.slabFloats + i ] = ( r < R && n < nOut ) ? src[ n ] : 0.0f;
			}
		}

		template<int D>
		int smemBytes( int ncols, int& ns )
		{
			using C = Cfg<D>;
			ns = ringSlots( C::SLOT, C::RS, ncols );
			return smemLayout( C::SLOT, C::RS, ns, ncols ).total;
		}
		template<int D>
		cudaError_t prepareD()
		{
			static PerDeviceMax attr;
			return attr.raise( FL_SMEM_MAX, []( size_t n ) {
				cudaError_t e = cudaFuncSetAttribute( decode_flow_kernel<D, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n );
				if( e != cudaSuccess ) return e;
				return cudaFuncSetAttribute( decode_flow_kernel<D, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)n );
			} );
		}
		template<int D>
		cudaError_t launchD( FlowArgs& a, int numSMs, cudaStream_t s )
		{
			a.ncols = a.B > 8 ? 16 : 8;
			int ns = 0;
			const int smem = smemBytes<D>( a.ncols, ns );
			a.NS = ns;
			cudaLaunchConfig_t cfg{};
			cfg.gridDim = dim3( (unsigned)numSMs );
			cfg.blockDim = dim3( FL_THREADS );
			cfg.dynamicSmemBytes = (size_t)smem;
			cfg.stream = s;
			cudaLaunchAttribute at[ 1 ];
			at[ 0 ].id = cudaLaunchAttributeCooperative;   // co-residency of all CTAs is a correctness requirement of the exchange
			at[ 0 ].val.cooperative = 1;
			cfg.attrs = at;
			cfg.numAttrs = 1;
			if( a.timing ) return cudaLaunchKernelEx( &cfg, decode_flow_kernel<D, true>, (const FlowArgs)a );
			return cudaLaunchKernelEx( &cfg, decode_flow_kernel<D, false>, (const FlowArgs)a );
		}
		inline int pad4( int x ) { return ( x + 3 ) & ~3; }

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

	FlowGeom flowGeometry( int d, int nVocab, int grid )
	{
		FlowGeom g;
		g.grid = grid;
		g.R1 = ( d + grid - 1 ) / grid;
		g.R3 = ( 3 * d + grid - 1 ) / grid;
		g.R4 = ( 4 * d + grid - 1 ) / grid;
		g.RV = ( nVocab + grid - 1 ) / grid;
		g.oQkv = 0;
		g.oO = g.oQkv + pad4( g.R3 );
		g.oCq = g.oO + pad4( g.R1 );
		g.oCo = g.oCq + pad4( g.R1 );
		g.oFc1 = g.oCo + pad4( g.R1 );
		g.oFc2 = g.oFc1 + pad4( g.R4 );
		g.slabFloats = g.oFc2 + pad4( g.R1 );
		return g;
	}

	bool flowSupported( int d, int B, int T, int H, int nTextCtx, int refThreads, const FlowGeom& g )
	{
		if( B < 1 || B > 16 || T > FL_MAXT || T < 1 || H * 64 != d || nTextCtx > FL_MAXT ) return false;
		if( refThreads < 1 || refThreads > kMaxRefThreads ) return false;
		if( g.R1 > 16 || g.slabFloats > 256 ) return false;
		const int ns = dispatchD( d, 0, [ & ]( auto D ) { int n = 0; smemBytes<decltype( D )::value>( B > 8 ? 16 : 8, n ); return n; } );
		return ns >= 4 + 1;   // a round of V slots (one per reference thread) is held at once
	}

	size_t flowExchangeBytes( int d, int maxB, int L ) { return (size_t)2 * L * maxB * d * 32; }

	cudaError_t flowPrepare( int d )
	{
		return dispatchD( d, cudaSuccess, []( auto D ) { return prepareD<decltype( D )::value>(); } );
	}

	cudaError_t flowBuildBiasSlab( float* slab, const FlowGeom& g, int d, const float* bqkv, const float* bo, const float* bcq, const float* bco,
		const float* b1, const float* b2, cudaStream_t s )
	{
		flow_bias_slab_kernel<<<g.grid, 128, 0, s>>>( slab, g, d, bqkv, bo, bcq, bco, b1, b2 );
		return cudaGetLastError();
	}

	cudaError_t decodeStepFlow( FlowArgs a, int d, int numSMs, cudaStream_t s )
	{
		return dispatchD( d, cudaErrorInvalidValue, [ & ]( auto D ) { return launchD<decltype( D )::value>( a, numSMs, s ); } );
	}
}

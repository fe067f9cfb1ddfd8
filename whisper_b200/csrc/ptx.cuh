// Thin inline-PTX layer for sm_90a: mbarrier, TMA (cp.async.bulk.tensor), wgmma (fence / mma_async / commit / wait) and the
// wgmma shared-memory descriptor; the decoder's mma.sync, streaming loads, cp.async, %globaltimer and warp reductions.
// Everything here is hand-written for H100; there is no other target.
//
// The descriptor bit layout follows the PTX ISA's "Matrix Descriptor Format" for wgmma — the layouts are hardware facts.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace ptx
{
	__device__ __forceinline__ uint32_t smem_u32( const void* p ) { return (uint32_t)__cvta_generic_to_shared( p ); }

	__device__ __forceinline__ bool elect_one()
	{
		uint32_t pred = 0;
		asm volatile(
			"{\n\t.reg .pred P;\n\telect.sync _|P, 0xffffffff;\n\tselp.u32 %0, 1, 0, P;\n\t}\n"
			: "=r"( pred ) );
		return pred != 0;
	}

	// ---------------------------------------------------------------------------------------------
	// mbarrier
	__device__ __forceinline__ void mbar_init( uint64_t* bar, uint32_t count )
	{
		asm volatile( "mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"( smem_u32( bar ) ), "r"( count ) : "memory" );
	}
	__device__ __forceinline__ void fence_barrier_init() { asm volatile( "fence.mbarrier_init.release.cluster;" ::: "memory" ); }
	__device__ __forceinline__ void fence_proxy_async() { asm volatile( "fence.proxy.async.shared::cta;" ::: "memory" ); }
	__device__ __forceinline__ void mbar_expect_tx( uint64_t* bar, uint32_t bytes )
	{
		asm volatile( "mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"( smem_u32( bar ) ), "r"( bytes ) : "memory" );
	}
	__device__ __forceinline__ void mbar_arrive( uint64_t* bar )
	{
		asm volatile( "mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"( smem_u32( bar ) ) : "memory" );
	}
	__device__ __forceinline__ bool mbar_try_wait( uint64_t* bar, uint32_t parity )
	{
		uint32_t ok;
		asm volatile(
			"{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}\n"
			: "=r"( ok )
			: "r"( smem_u32( bar ) ), "r"( parity )
			: "memory" );
		return ok != 0;
	}
	// Bounded wait: a protocol bug must surface as a trap (launch failure), never as a hung GPU.
	__device__ __forceinline__ void mbar_wait( uint64_t* bar, uint32_t parity )
	{
		uint32_t spins = 0;
		while( !mbar_try_wait( bar, parity ) )
		{
			if( ++spins > ( 1u << 22 ) )
				__trap();
		}
	}

	// ---------------------------------------------------------------------------------------------
	// TMA tile loads, completion signalled on an mbarrier (complete_tx::bytes)
	__device__ __forceinline__ void tma_load_2d( void* dst, const CUtensorMap* map, uint64_t* bar, int c0, int c1 )
	{
		asm volatile(
			"cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
			::"r"( smem_u32( dst ) ), "l"( map ), "r"( smem_u32( bar ) ), "r"( c0 ), "r"( c1 )
			: "memory" );
	}
	// 1-D bulk copy global -> shared by the TMA engine (no tensor map): one instruction moves up to the whole tile, completion is
	// counted in bytes on the mbarrier.  Addresses and size must be multiples of 16.
	__device__ __forceinline__ void bulk_load_1d( void* dst, const void* src, uint32_t bytes, uint64_t* bar )
	{
		asm volatile( "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"( smem_u32( dst ) ), "l"( src ),
			"r"( bytes ), "r"( smem_u32( bar ) )
			: "memory" );
	}
	__device__ __forceinline__ void prefetch_tensormap( const CUtensorMap* map )
	{
		asm volatile( "prefetch.tensormap [%0];" ::"l"( map ) : "memory" );
	}

	// ---------------------------------------------------------------------------------------------
	// wgmma: warpgroup MMA, f16 inputs, f32 accumulators in registers.  All 128 threads of a warpgroup issue each instruction.
	//
	// Accumulator layout of m64nNk16 (per warp w of the warpgroup, lane l, q = l & 3): d[4j + 0/1] = row 16w + l/4, columns
	// 8j + 2q + 0/1;  d[4j + 2/3] = row 16w + l/4 + 8, same columns.  A register A fragment of m64k16 has the same shape:
	// {a0, a1, a2, a3} = (row, k 2q..2q+1), (row + 8, k 2q..2q+1), (row, k 2q+8..2q+9), (row + 8, k 2q+8..2q+9), two f16 each.
	__device__ __forceinline__ void wgmma_fence() { asm volatile( "wgmma.fence.sync.aligned;" ::: "memory" ); }
	__device__ __forceinline__ void wgmma_commit() { asm volatile( "wgmma.commit_group.sync.aligned;" ::: "memory" ); }
	template<int N>
	__device__ __forceinline__ void wgmma_wait() { asm volatile( "wgmma.wait_group.sync.aligned %0;" ::"n"( N ) : "memory" ); }
	// keep the compiler from moving accumulator reads / writes across an in-flight wgmma
	template<int N>
	__device__ __forceinline__ void fence_regs( float* d )
	{
#pragma unroll
		for( int i = 0; i < N; i++ ) asm volatile( "" : "+f"( d[ i ] )::"memory" );
	}

	// D (+)= A * B^T, A = [64][16] and B = [N][16] K-major tiles in shared memory (descriptors below)
	__device__ __forceinline__ void wgmma_m64n128k16_ss( float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate )
	{
		asm volatile(
			"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
			"wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
			"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
			"%64, %65, p, 1, 1, 0, 0;\n\t}\n"
			: "+f"( d[ 0 ] ), "+f"( d[ 1 ] ), "+f"( d[ 2 ] ), "+f"( d[ 3 ] ), "+f"( d[ 4 ] ), "+f"( d[ 5 ] ), "+f"( d[ 6 ] ), "+f"( d[ 7 ] ), "+f"( d[ 8 ] ), "+f"( d[ 9 ] ), "+f"( d[ 10 ] ), "+f"( d[ 11 ] ), "+f"( d[ 12 ] ), "+f"( d[ 13 ] ), "+f"( d[ 14 ] ), "+f"( d[ 15 ] ), "+f"( d[ 16 ] ), "+f"( d[ 17 ] ), "+f"( d[ 18 ] ), "+f"( d[ 19 ] ), "+f"( d[ 20 ] ), "+f"( d[ 21 ] ), "+f"( d[ 22 ] ), "+f"( d[ 23 ] ), "+f"( d[ 24 ] ), "+f"( d[ 25 ] ), "+f"( d[ 26 ] ), "+f"( d[ 27 ] ), "+f"( d[ 28 ] ), "+f"( d[ 29 ] ), "+f"( d[ 30 ] ), "+f"( d[ 31 ] ), "+f"( d[ 32 ] ), "+f"( d[ 33 ] ), "+f"( d[ 34 ] ), "+f"( d[ 35 ] ), "+f"( d[ 36 ] ), "+f"( d[ 37 ] ), "+f"( d[ 38 ] ), "+f"( d[ 39 ] ), "+f"( d[ 40 ] ), "+f"( d[ 41 ] ), "+f"( d[ 42 ] ), "+f"( d[ 43 ] ), "+f"( d[ 44 ] ), "+f"( d[ 45 ] ), "+f"( d[ 46 ] ), "+f"( d[ 47 ] ), "+f"( d[ 48 ] ), "+f"( d[ 49 ] ), "+f"( d[ 50 ] ), "+f"( d[ 51 ] ), "+f"( d[ 52 ] ), "+f"( d[ 53 ] ), "+f"( d[ 54 ] ), "+f"( d[ 55 ] ), "+f"( d[ 56 ] ), "+f"( d[ 57 ] ), "+f"( d[ 58 ] ), "+f"( d[ 59 ] ), "+f"( d[ 60 ] ), "+f"( d[ 61 ] ), "+f"( d[ 62 ] ), "+f"( d[ 63 ] )
			: "l"( desc_a ), "l"( desc_b ), "r"( accumulate ) );
	}
	__device__ __forceinline__ void wgmma_m64n256k16_ss( float* d, uint64_t desc_a, uint64_t desc_b, uint32_t accumulate )
	{
		asm volatile(
			"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
			"wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 "
			"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, "
			"%128, %129, p, 1, 1, 0, 0;\n\t}\n"
			: "+f"( d[ 0 ] ), "+f"( d[ 1 ] ), "+f"( d[ 2 ] ), "+f"( d[ 3 ] ), "+f"( d[ 4 ] ), "+f"( d[ 5 ] ), "+f"( d[ 6 ] ), "+f"( d[ 7 ] ), "+f"( d[ 8 ] ), "+f"( d[ 9 ] ), "+f"( d[ 10 ] ), "+f"( d[ 11 ] ), "+f"( d[ 12 ] ), "+f"( d[ 13 ] ), "+f"( d[ 14 ] ), "+f"( d[ 15 ] ), "+f"( d[ 16 ] ), "+f"( d[ 17 ] ), "+f"( d[ 18 ] ), "+f"( d[ 19 ] ), "+f"( d[ 20 ] ), "+f"( d[ 21 ] ), "+f"( d[ 22 ] ), "+f"( d[ 23 ] ), "+f"( d[ 24 ] ), "+f"( d[ 25 ] ), "+f"( d[ 26 ] ), "+f"( d[ 27 ] ), "+f"( d[ 28 ] ), "+f"( d[ 29 ] ), "+f"( d[ 30 ] ), "+f"( d[ 31 ] ), "+f"( d[ 32 ] ), "+f"( d[ 33 ] ), "+f"( d[ 34 ] ), "+f"( d[ 35 ] ), "+f"( d[ 36 ] ), "+f"( d[ 37 ] ), "+f"( d[ 38 ] ), "+f"( d[ 39 ] ), "+f"( d[ 40 ] ), "+f"( d[ 41 ] ), "+f"( d[ 42 ] ), "+f"( d[ 43 ] ), "+f"( d[ 44 ] ), "+f"( d[ 45 ] ), "+f"( d[ 46 ] ), "+f"( d[ 47 ] ), "+f"( d[ 48 ] ), "+f"( d[ 49 ] ), "+f"( d[ 50 ] ), "+f"( d[ 51 ] ), "+f"( d[ 52 ] ), "+f"( d[ 53 ] ), "+f"( d[ 54 ] ), "+f"( d[ 55 ] ), "+f"( d[ 56 ] ), "+f"( d[ 57 ] ), "+f"( d[ 58 ] ), "+f"( d[ 59 ] ), "+f"( d[ 60 ] ), "+f"( d[ 61 ] ), "+f"( d[ 62 ] ), "+f"( d[ 63 ] ), "+f"( d[ 64 ] ), "+f"( d[ 65 ] ), "+f"( d[ 66 ] ), "+f"( d[ 67 ] ), "+f"( d[ 68 ] ), "+f"( d[ 69 ] ), "+f"( d[ 70 ] ), "+f"( d[ 71 ] ), "+f"( d[ 72 ] ), "+f"( d[ 73 ] ), "+f"( d[ 74 ] ), "+f"( d[ 75 ] ), "+f"( d[ 76 ] ), "+f"( d[ 77 ] ), "+f"( d[ 78 ] ), "+f"( d[ 79 ] ), "+f"( d[ 80 ] ), "+f"( d[ 81 ] ), "+f"( d[ 82 ] ), "+f"( d[ 83 ] ), "+f"( d[ 84 ] ), "+f"( d[ 85 ] ), "+f"( d[ 86 ] ), "+f"( d[ 87 ] ), "+f"( d[ 88 ] ), "+f"( d[ 89 ] ), "+f"( d[ 90 ] ), "+f"( d[ 91 ] ), "+f"( d[ 92 ] ), "+f"( d[ 93 ] ), "+f"( d[ 94 ] ), "+f"( d[ 95 ] ), "+f"( d[ 96 ] ), "+f"( d[ 97 ] ), "+f"( d[ 98 ] ), "+f"( d[ 99 ] ), "+f"( d[ 100 ] ), "+f"( d[ 101 ] ), "+f"( d[ 102 ] ), "+f"( d[ 103 ] ), "+f"( d[ 104 ] ), "+f"( d[ 105 ] ), "+f"( d[ 106 ] ), "+f"( d[ 107 ] ), "+f"( d[ 108 ] ), "+f"( d[ 109 ] ), "+f"( d[ 110 ] ), "+f"( d[ 111 ] ), "+f"( d[ 112 ] ), "+f"( d[ 113 ] ), "+f"( d[ 114 ] ), "+f"( d[ 115 ] ), "+f"( d[ 116 ] ), "+f"( d[ 117 ] ), "+f"( d[ 118 ] ), "+f"( d[ 119 ] ), "+f"( d[ 120 ] ), "+f"( d[ 121 ] ), "+f"( d[ 122 ] ), "+f"( d[ 123 ] ), "+f"( d[ 124 ] ), "+f"( d[ 125 ] ), "+f"( d[ 126 ] ), "+f"( d[ 127 ] )
			: "l"( desc_a ), "l"( desc_b ), "r"( accumulate ) );
	}
	// D (+)= A * B^T with A = [64][16] in registers (the fragment above), B = [64][16] K-major in shared memory
	__device__ __forceinline__ void wgmma_m64n64k16_rs( float* d, const uint32_t* a, uint64_t desc_b, uint32_t accumulate )
	{
		asm volatile(
			"{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %37, 0;\n\t"
			"wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 "
			"{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
			"{%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}\n"
			: "+f"( d[ 0 ] ), "+f"( d[ 1 ] ), "+f"( d[ 2 ] ), "+f"( d[ 3 ] ), "+f"( d[ 4 ] ), "+f"( d[ 5 ] ), "+f"( d[ 6 ] ), "+f"( d[ 7 ] ), "+f"( d[ 8 ] ), "+f"( d[ 9 ] ), "+f"( d[ 10 ] ), "+f"( d[ 11 ] ), "+f"( d[ 12 ] ), "+f"( d[ 13 ] ), "+f"( d[ 14 ] ), "+f"( d[ 15 ] ), "+f"( d[ 16 ] ), "+f"( d[ 17 ] ), "+f"( d[ 18 ] ), "+f"( d[ 19 ] ), "+f"( d[ 20 ] ), "+f"( d[ 21 ] ), "+f"( d[ 22 ] ), "+f"( d[ 23 ] ), "+f"( d[ 24 ] ), "+f"( d[ 25 ] ), "+f"( d[ 26 ] ), "+f"( d[ 27 ] ), "+f"( d[ 28 ] ), "+f"( d[ 29 ] ), "+f"( d[ 30 ] ), "+f"( d[ 31 ] )
			: "r"( a[ 0 ] ), "r"( a[ 1 ] ), "r"( a[ 2 ] ), "r"( a[ 3 ] ), "l"( desc_b ), "r"( accumulate ) );
	}

	// Named barrier over `count` threads (ids 1..15; 0 is __syncthreads)
	__device__ __forceinline__ void named_bar_sync( int id, int count ) { asm volatile( "bar.sync %0, %1;" ::"r"( id ), "r"( count ) : "memory" ); }

	// ---------------------------------------------------------------------------------------------
	// Shared-memory matrix descriptor (sm_90 wgmma) for a K-major operand tile stored as rows of 64 f16 (128 bytes) with the
	// 128-byte swizzle TMA writes (CU_TENSOR_MAP_SWIZZLE_128B): 8-row groups are 1024 bytes apart (stride byte offset), the
	// leading byte offset is unused for swizzled K-major (encoded 1), layout type 1 = SWIZZLE_128B.  Tiles start 1024-aligned;
	// the k-th 16-element slice of a row starts 32 bytes further: +2 in the (address >> 4) field.
	__device__ __forceinline__ uint64_t gmma_desc_sw128( uint32_t smem_addr )
	{
		uint64_t d = 0;
		d |= (uint64_t)( ( smem_addr & 0x3FFFF ) >> 4 );         // [0,14)  start address >> 4
		d |= (uint64_t)1 << 16;                                   // [16,30) leading byte offset >> 4 (ignored)
		d |= (uint64_t)( 1024 >> 4 ) << 32;                       // [32,46) stride byte offset >> 4
		d |= (uint64_t)1 << 62;                                   // [62,64) SWIZZLE_128B
		return d;
	}

	// Programmatic dependent launch: let the next kernel of the stream start its prologue (weight / KV prefetch) while this one runs,
	// and block until every kernel this one depends on has completed and flushed its writes.
	__device__ __forceinline__ void pdl_launch_dependents() { asm volatile( "griddepcontrol.launch_dependents;" ::: "memory" ); }
	__device__ __forceinline__ void pdl_wait() { asm volatile( "griddepcontrol.wait;" ::: "memory" ); }

	// ---------------------------------------------------------------------------------------------
	// Decoder building blocks
	//
	// Butterfly reductions over the 32 lanes of a warp (xor 16, 8, 4, 2, 1): every lane ends with the same value, and the order of
	// the additions is fixed, so results are bit-reproducible.
	template<class T>
	__device__ __forceinline__ T warp_sum( T v )
	{
		for( int o = 16; o > 0; o >>= 1 ) v += __shfl_xor_sync( 0xffffffffu, v, o );
		return v;
	}
	__device__ __forceinline__ float warp_max( float v )
	{
		for( int o = 16; o > 0; o >>= 1 ) v = fmaxf( v, __shfl_xor_sync( 0xffffffffu, v, o ) );
		return v;
	}

	// D += A * B, mma.sync m16n8k16 with f16 inputs and f32 accumulators: A fragment {a0, a1, a2, a3}, B fragment {b0, b1}
	__device__ __forceinline__ void mma_m16n8k16( float* c, uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0, uint32_t b1 )
	{
		asm volatile(
			"mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
			: "+f"( c[ 0 ] ), "+f"( c[ 1 ] ), "+f"( c[ 2 ] ), "+f"( c[ 3 ] )
			: "r"( a0 ), "r"( a1 ), "r"( a2 ), "r"( a3 ), "r"( b0 ), "r"( b1 ) );
	}
	// the same with rows 8..15 of A zero (registers a1, a3): a unit of 8 weight rows
	__device__ __forceinline__ void mma_m16n8k16_rows8( float* c, uint32_t a0, uint32_t a2, uint32_t b0, uint32_t b1 )
	{
		mma_m16n8k16( c, a0, 0u, a2, 0u, b0, b1 );
	}

	// 16-byte load of read-only data that is used once (weights): non-coherent path, not kept in L1
	__device__ __forceinline__ uint4 ldg_stream( const uint4* p )
	{
		uint4 r;
		asm volatile( "ld.global.nc.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"( r.x ), "=r"( r.y ), "=r"( r.z ), "=r"( r.w ) : "l"( p ) );
		return r;
	}

	// 16-byte asynchronous copy global -> shared (bypassing L1), its commit and the wait for every committed group
	__device__ __forceinline__ void cp_async16( void* smemDst, const void* gmemSrc )
	{
		asm volatile( "cp.async.cg.shared.global [%0], [%1], 16;" ::"r"( smem_u32( smemDst ) ), "l"( gmemSrc ) : "memory" );
	}
	// the same with only the first srcBytes (0..16) read and the rest of the 16 bytes zero-filled
	__device__ __forceinline__ void cp_async16_zfill( void* smemDst, const void* gmemSrc, uint32_t srcBytes )
	{
		asm volatile( "cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"( smem_u32( smemDst ) ), "l"( gmemSrc ), "r"( srcBytes ) : "memory" );
	}
	__device__ __forceinline__ void cp_async_commit() { asm volatile( "cp.async.commit_group;" ::: "memory" ); }
	__device__ __forceinline__ void cp_async_wait_all() { asm volatile( "cp.async.wait_group 0;" ::: "memory" ); }
	template<int N> __device__ __forceinline__ void cp_async_wait() { asm volatile( "cp.async.wait_group %0;" ::"n"( N ) : "memory" ); }

	// nanoseconds of the global timer (debug marks, and the time limit of spin waits)
	__device__ __forceinline__ unsigned long long globaltimer()
	{
		unsigned long long t;
		asm volatile( "mov.u64 %0, %globaltimer;" : "=l"( t ) );
		return t;
	}

	__device__ __forceinline__ float gelu_f16_semantics( float x )
	{
		// Oracle: y = f32( T[f16(x)] ), T[i] = f16( gelu( f32(i) ) ) evaluated in double (ggml.c:999-1021, table init :1372-1383).
		// Both roundings are reproduced; the table is replaced by evaluating the same function as v * sigmoid(2u),
		// u = sqrt(2/pi) * v * (1 + 0.044715 v^2)  ==  0.5 v (1 + tanh(u)), with ex2/rcp (relative error ~1e-6, i.e. the f16 result
		// differs from the table only on near-ties).  This form costs ~10 instructions instead of tanhf's ~30: the fc1 epilogue
		// evaluates it 49 M times per encoder layer.
		const float v = __half2float( __float2half_rn( x ) );
		const float u2 = -1.5957691216057308f * v * ( 1.0f + 0.044715f * v * v );   // -2u
		const float y = __fdividef( v, 1.0f + __expf( u2 ) );
		return __half2float( __float2half_rn( y ) );
	}
}

// Issue rate of the conversion instructions the decoder's f16 V^T*P chains are made of (HADD2.F32 = f16 -> f32, F2FP.F16.F32.PACK_AB =
// f32 -> f16) against FFMA, per SM: 8 warps x 8 independent streams per thread, so that latency is hidden and only the pipe counts.
// build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o cvt_rate cvt_rate.cu ; run on an H100
#include <cstdio>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

template<int MODE>
__global__ void k( float* out, int iters, long long* cyc )
{
	float a[ 8 ];
	for( int i = 0; i < 8; i++ ) a[ i ] = 1.0f + threadIdx.x * 1e-3f + i;
	__syncthreads();
	const long long t0 = clock64();
	for( int it = 0; it < iters; it++ )
	{
#pragma unroll
		for( int i = 0; i < 8; i++ )
		{
			if( MODE == 0 ) a[ i ] = __fmaf_rn( a[ i ], 1.0000001f, 1e-7f );                       // FFMA
			if( MODE == 1 ) a[ i ] = __half2float( __float2half_rn( a[ i ] ) ) + 0.0f;            // F2FP + HADD2.F32 (the compiler may fold +0)
			if( MODE == 2 ) { __half h = __float2half_rn( a[ i ] ); a[ i ] = __half2float( h ); }    // F2FP + HADD2.F32
			if( MODE == 3 ) { __half h = __float2half_rn( a[ i ] ); a[ i ] = __fmaf_rn( __half2float( h ), 1.0000001f, 1e-7f ); }   // one chain step
			if( MODE == 4 )
			{
				unsigned short hb;
				asm volatile( "cvt.rn.f16.f32 %0, %1;" : "=h"( hb ) : "f"( a[ i ] ) );            // f32 -> f16 only
				a[ i ] = __uint_as_float( 0x3f800000u | hb );
			}
			if( MODE == 5 )
			{
				unsigned short hb = (unsigned short)( __float_as_uint( a[ i ] ) >> 13 );
				float f;
				asm volatile( "cvt.f32.f16 %0, %1;" : "=f"( f ) : "h"( hb ) );                     // f16 -> f32 only
				a[ i ] = f + 1.0f;
			}
		}
	}
	const long long t1 = clock64();
	float s = 0;
	for( int i = 0; i < 8; i++ ) s += a[ i ];
	out[ blockIdx.x * blockDim.x + threadIdx.x ] = s;
	if( threadIdx.x == 0 && blockIdx.x == 0 ) *cyc = t1 - t0;
}

template<int MODE>
void run( const char* name, float* out, long long* cyc )
{
	const int iters = 4096;
	k<MODE><<<132, 256>>>( out, iters, cyc );
	k<MODE><<<132, 256>>>( out, iters, cyc );
	cudaDeviceSynchronize();
	long long c;
	cudaMemcpy( &c, cyc, 8, cudaMemcpyDeviceToHost );
	const double ops = 256.0 * 8 * iters;
	printf( "%-44s %8.1f thread-iterations per cycle per SM (%lld cycles)\n", name, ops / c, c );
}
int main()
{
	float* out; long long* cyc;
	cudaMalloc( &out, 132 * 256 * 4 ); cudaMalloc( &cyc, 8 );
	run<0>( "FFMA", out, cyc );
	run<2>( "f32->f16->f32 (F2FP + HADD2.F32)", out, cyc );
	run<3>( "chain step (F2FP + HADD2.F32 + FFMA)", out, cyc );
	run<4>( "cvt.rn.f16.f32 (+ LOP)", out, cyc );
	run<5>( "cvt.f32.f16 (+ SHF + FADD)", out, cyc );
	return 0;
}

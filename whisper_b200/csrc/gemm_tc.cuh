// Persistent, warp-specialised wgmma GEMM for sm_90a:  D[M,N] = A[M,K] * B[N,K]^T  (both operands f16, K-major; f32 accumulate)
//
// Replaces the reference's mulMatTiled.hlsl (43 % of its GPU time, ComputeShaders/mulMatTiled.hlsl:203-274, host call
// Whisper/ML/MlContext.cpp:132-147) and the ggml CPU path ggml_compute_forward_mul_mat_f16_f32 (Whisper/source/ggml.c:4447-4749),
// whose arithmetic — activation rounded to f16, f16 x f16 products, f32 accumulation — is exactly what wgmma .f32.f16.f16 does.
//
//   warpgroup 0    : TMA producer   (one thread: cp.async.bulk.tensor 2D, 128B swizzle, mbarrier complete_tx)
//   warpgroups 1-2 : consumers      (wgmma.mma_async m64nBNk16, rows [0,64) and [64,128) of the 128 x BN tile, accumulators in
//                                    registers; then the fused epilogue through a 64 x 64 shared-memory staging tile)
//
// Pipeline: smem full/empty mbarriers between the producer and the consumers (one k-block of wgmma kept in flight), and a static
// persistent tile schedule (grid = #SMs), so the producer already streams the next tile while the consumers run the epilogue.
//
// The fused epilogues are the reference's element-wise shaders folded in: addRepeat / addRepeatScale / addRepeatGelu /
// addRepeatEx / copyConvert / copyTranspose (SURVEY.md §2.2), writing head-major f16 Q/K, transposed V and the f16
// cross-attention KV memories directly.
#pragma once
#include "ptx.cuh"

namespace gemm
{
	constexpr int BM = 128;
	constexpr int BK = 64;

	enum EpiMode : int
	{
		EPI_F32 = 0,          // out_f32[m][n] = acc (+ bias[n])                                  (the wsp_test_gemm hook only)
		EPI_CONV1 = 1,        // f16 out[(m+1)][n] = gelu(acc + bias[n]), rows of padded time axis, halos zeroed (a3)
		EPI_CONV2 = 2,        // f32 out[b*T+j][n] = gelu(acc + bias[n]) + pos[j][n]                (a4)
		EPI_QKV = 3,          // Q,K head-major f16, V transposed f16                               (a6, a7)
		EPI_BIAS_RESID = 4,   // f32 out[m][n] = acc + bias[n] + resid[m][n]                        (a9, a10)
		EPI_BIAS_GELU_F16 = 5,// f16 out[m][n] = gelu(acc + bias[n])                                (a10)
		EPI_CROSSKV = 6,      // f16 cross K (scaled) / cross V (+bias) memories for all layers     (a12)
	};

	// A-operand addressing of the producer
	enum AMode : int
	{
		A_PLAIN = 0,   // A is a plain [M][K] matrix
		A_CONV_S1 = 1, // K = 3 taps x Kt: tap k reads rows (m + k) of the zero-padded time-major input   (conv1d stride 1)
		A_CONV_S2 = 2, // tap 0: even rows view [m], tap 1: odd rows view [m], tap 2: even rows view [m+1] (conv1d stride 2)
	};

	struct EpiParams
	{
		int M = 0;                 // valid output rows (guard)
		int N = 0;                 // valid output columns (guard)
		int ld = 0;                // leading dimension (elements) of row-major outputs
		const float* bias = nullptr;
		const float* resid = nullptr;  // may alias out_f32
		const float* pos = nullptr;
		float* out_f32 = nullptr;
		__half* out_a = nullptr;   // Q | conv1 out | gelu out | cross K
		__half* out_b = nullptr;   // K | cross V
		__half* out_c = nullptr;   // V^T
		int T = 0;                 // time steps per chunk (audio_ctx, 1500 by default)
		int Tp = 0;                // padded row length of V^T
		int H = 0;                 // heads
		int d = 0;                 // model width
		int rows_per_chunk = 0;    // conv: padded rows per chunk in the flattened A row space
		int valid_per_chunk = 0;   // conv: valid output rows per chunk
		int nchunks = 0;
		size_t layer_stride = 0;   // EPI_CROSSKV: elements between two decoder layers' memories
		float scale = 1.0f;
	};

	struct Launch
	{
		CUtensorMap mapA;
		CUtensorMap mapA2;  // A_CONV_S2 only: odd-row view
		CUtensorMap mapB;
		int M = 0, N = 0, K = 0; // K = total reduction length (taps included), multiple handling via TMA zero fill
		int kTap = 0;           // A_CONV_*: K-blocks (of 64) per tap
		EpiParams ep;
	};

	// Host side: 2D f16 tensor map, 128B swizzle, box = {64, boxRows}.  rowStrideBytes must be a multiple of 16.
	bool makeMap2D( CUtensorMap* map, const void* base, uint64_t inner, uint64_t rows, uint64_t rowStrideBytes, uint32_t boxRows );

	// Launch on `stream`.  bn selects the N tile (128 or 256).
	cudaError_t launch( const Launch& L, EpiMode epi, AMode amode, int bn, int numSMs, cudaStream_t stream );
}

// Encoder flash attention (wgmma) — see attn_enc.cu.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>

namespace attn
{
	struct EncParams
	{
		int T = 0;            // keys / queries per (chunk, head): n_audio_ctx
		int H = 0;            // heads
		int nBH = 0;          // chunks * heads
		int d = 0;            // model width = H * 64
		float scale_log2 = 0; // (1/sqrt(64)) * log2(e)
		__half* out = nullptr;// [chunk][T][d] f16, heads merged
	};
	// mapQ / mapK: 2D f16 [(nBH*T)][64], box {64,128};  mapVt: 2D f16 [(nBH*64)][Tp], box {64,64}; all 128B-swizzled.
	cudaError_t launchEnc( const CUtensorMap& mapQ, const CUtensorMap& mapK, const CUtensorMap& mapVt, const EncParams& p, cudaStream_t stream );
}

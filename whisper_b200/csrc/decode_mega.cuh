// Persistent decoder-step kernel — see decode_mega.cu.
#pragma once
#include "decode_step.cuh"

namespace kern
{
	struct MegaArgs : DecStepArgs       // timing: marks of CTA 0 around every barrier
	{
		float* x = nullptr;                 // [B][d] residual stream
		float* q = nullptr;                 // [B][d]
		__half* attn = nullptr;             // [B][d]
		__half* h = nullptr;                // [B][4d]
		unsigned* barrier = nullptr;        // grid barrier counter (zeroed by the launcher)
	};
	bool megaSupported( int d, int B, int T );
	cudaError_t megaPrepare( int d );   // function attributes, outside any stream capture
	// one single-token decoder step for B chunks: embedding -> L layers -> final LN -> logits (sampling is a separate kernel)
	cudaError_t decodeStepMega( const MegaArgs& a, int d, int numSMs, cudaStream_t s );
}

// Dataflow decoder-step kernel — see decode_flow.cu.
#pragma once
#include "decode_step.cuh"

namespace kern
{
	// how the output rows of every weight-streaming phase are split over the CTAs: CTA c owns rows [c*R, min((c+1)*R, nOut))
	struct FlowGeom
	{
		int grid = 0;
		int R1 = 0, R3 = 0, R4 = 0, RV = 0;                        // rows per CTA for nOut = d, 3d, 4d, n_vocab
		int oQkv = 0, oO = 0, oCq = 0, oCo = 0, oFc1 = 0, oFc2 = 0;   // float offsets of the sections in a bias slab
		int slabFloats = 0;
	};
	FlowGeom flowGeometry( int d, int nVocab, int grid );

	struct FlowArgs : DecStepArgs       // timing: (id, %globaltimer) marks of CTA `timingCta`
	{
		uint8_t* exch = nullptr;            // exchange buffers: 2 sets x L layers x (maxB * d * 32) bytes, all 0xFF when idle
		unsigned* ctrl = nullptr;           // [0] CTAs finished, [1] launch epoch (selects the exchange set)
		int timingCta = 0;
		FlowGeom g;
		int NS = 0;                         // ring slots
		int ncols = 8;                      // activation columns staged: 8 (B <= 8) or 16
	};
	// g: the context's geometry (flowGeometry); the limits checked on it do not depend on the vocabulary, so neither does the answer
	bool flowSupported( int d, int B, int T, int H, int nTextCtx, int refThreads, const FlowGeom& g );
	size_t flowExchangeBytes( int d, int maxB, int L );
	cudaError_t flowPrepare( int d );   // function attributes for the current device, outside any stream capture
	// regroup one layer's biases per CTA: slab[c] = (qkv rows of c | o | cq | co | fc1 | fc2), zero padded
	cudaError_t flowBuildBiasSlab( float* slab, const FlowGeom& g, int d, const float* bqkv, const float* bo, const float* bcq, const float* bco,
		const float* b1, const float* b2, cudaStream_t s );
	// one single-token decoder step for B chunks: embedding -> L layers -> final LN -> logits (sampling is a separate kernel)
	cudaError_t decodeStepFlow( FlowArgs a, int d, int numSMs, cudaStream_t s );
}

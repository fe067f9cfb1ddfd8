// What the two N = 1 decoder-step kernels (decode_flow.cu, decode_mega.cu) are handed alike: the per-layer pointer table and
// the shared part of their arguments.  Each kernel reads only the fields it needs.
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace kern
{
	struct DecStepLayer
	{
		const float *ln1g, *ln1b, *lncg, *lncb, *ln3g, *ln3b;
		const __half *wqkv, *wo, *wcq, *wco, *w1, *w2;
		const float *bqkv, *bo, *bcq, *bco, *b1, *b2;   // raw biases (barrier kernel)
		const float* biasSlab;              // [grid][slabFloats]: the same biases regrouped per CTA (flowBuildBiasSlab; dataflow kernel)
		__half *kCache, *vCache;            // [maxB][H][nTextCtx][64] of this layer (head-major: a head's rows are contiguous)
		const __half *crossK, *crossV;      // [maxB][H][T][64] of this layer
	};
	struct DecStepArgs
	{
		const DecStepLayer* layers = nullptr;   // device array [L]
		int L = 0, B = 0, H = 0, nTextCtx = 0, T = 0, nVocab = 0, refThreads = 4, maxB = 0;   // maxB last: ahead of H it changes how the barrier kernel pairs its constant loads, and that kernel spills (step +4.6 % on H100)
		const __half* tokEmb = nullptr;
		const float* decPos = nullptr;
		const float* lnfg = nullptr;
		const float* lnfb = nullptr;
		const int* tokens = nullptr;        // [B] (device)
		const int* dNPast = nullptr;
		float* logits = nullptr;            // [B][nVocab]
		unsigned long long* timing = nullptr;   // optional: %globaltimer marks of one CTA (debug)
	};
}

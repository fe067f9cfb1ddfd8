// iContext::detectSpeaker's rule (Whisper/Whisper/ContextImpl.diarize.cpp:17-108, Spectrogram.cpp:142-168), once, for the host and the
// device: which stereo frames a segment covers, the per-channel sums of |sample| in the reference's SSE lane order, and the 1.1
// decision.  iContext::detectSpeaker (com_shell.cpp, built by g++) and wsp_test_speakers run it on the host; speaker_kernel
// (kernels_frontend.cu) folds the same lanes and decides with the same code for a whole batch of segments.
#pragma once
#include "../../include/whisper_b200.h"
#include <math.h>
#include <stdint.h>

#if !defined( WSP_HOST_DEVICE )
#if defined( __CUDACC__ )
#define WSP_HOST_DEVICE __host__ __device__
#else
#define WSP_HOST_DEVICE
#endif
#endif

namespace wsp
{
	constexpr int kSpeakerHop = 160;      // stereo frames per 10 ms unit (FFT_STEP)
	constexpr int kSpeakerSums = -2;      // speakerSpan: the answer needs the channel sums of frames [first, first + count)

	// The part of detectSpeaker before any sample is read, for a segment [t0, t1) in 10 ms units over nFrames stereo frames (0: the
	// clip has none, as the reference's empty stereo buffer).  Returns WSP_SPEAKER_UNSURE for an empty or reversed interval,
	// WSP_SPEAKER_NO_STEREO without stereo, WSP_SPEAKER_OUT_OF_RANGE when the first frame lies outside the clip (copyStereoPcm's
	// E_BOUNDS), else kSpeakerSums with count = (t1 - t0) * 160 frames cut at the end of the clip (the zero fill past it adds nothing).
	WSP_HOST_DEVICE inline int speakerSpan( int64_t t0, int64_t t1, int64_t nFrames, int64_t& first, int64_t& count )
	{
		if( t1 <= t0 ) return WSP_SPEAKER_UNSURE;
		if( nFrames <= 0 ) return WSP_SPEAKER_NO_STEREO;
		if( t0 < 0 || t0 >= ( nFrames + kSpeakerHop - 1 ) / kSpeakerHop ) return WSP_SPEAKER_OUT_OF_RANGE;   // t0 * 160 >= nFrames
		first = t0 * kSpeakerHop;
		const int64_t rest = nFrames - first;
		count = t1 - t0 >= ( rest + kSpeakerHop - 1 ) / kSpeakerHop ? rest : ( t1 - t0 ) * kSpeakerHop;
		return kSpeakerSums;
	}

	// One step of a lane's chain.  The reference adds two frames per step into four f32 lanes { |L even|, |R even|, |L odd|, |R odd| }
	// (computeChannelsEnergy); each lane is a chain in frame order, and an odd last frame leaves the odd lanes as they are.
	WSP_HOST_DEVICE inline float speakerFold( float acc, float x ) { return acc + fabsf( x ); }

	// produceResult (ContextImpl.diarize.cpp:54-70) over the four lanes: left = lane 0 + lane 2, right = lane 1 + lane 3, and a channel
	// wins when it exceeds 1.1 times the other
	WSP_HOST_DEVICE inline int speakerDecide( float lEven, float rEven, float lOdd, float rOdd )
	{
		const float left = lEven + lOdd, right = rEven + rOdd;
		return ( left > right * 1.1f ? WSP_SPEAKER_LEFT : 0 ) | ( right > left * 1.1f ? WSP_SPEAKER_RIGHT : 0 );
	}

	// the whole rule on the host: interleaved lr[nFrames][2]
	inline int speakerOfSegment( const float* lr, int64_t nFrames, int64_t t0, int64_t t1 )
	{
		int64_t first = 0, count = 0;
		const int r = speakerSpan( t0, t1, nFrames, first, count );
		if( r != kSpeakerSums ) return r;
		float acc[ 4 ] = { 0.0f, 0.0f, 0.0f, 0.0f };
		const float* p = lr + 2 * first;
		for( int64_t i = 0; i < count; i++ )
		{
			acc[ 2 * ( i & 1 ) ] = speakerFold( acc[ 2 * ( i & 1 ) ], p[ 2 * i ] );
			acc[ 2 * ( i & 1 ) + 1 ] = speakerFold( acc[ 2 * ( i & 1 ) + 1 ], p[ 2 * i + 1 ] );
		}
		return speakerDecide( acc[ 0 ], acc[ 1 ], acc[ 2 ], acc[ 3 ] );
	}
}

// whisper_full's window rule (Whisper/source/whisper.cpp:2926-3003), once, for the host and the device: which sampled token ends a
// window, how many of its tokens are its result and how far the window advances.  iContext::runFull (com_shell.cpp, built by g++) runs
// it per token on the host; wsp_run_chunks_window runs it per row in the sampler's epilogue (kernels_decode.cu).
#pragma once

#if defined( __CUDACC__ )
#define WSP_HOST_DEVICE __host__ __device__
#else
#define WSP_HOST_DEVICE
#endif

namespace wsp
{
	constexpr int kWindowFrames = 100 * 30;   // 100 * WHISPER_CHUNK_SIZE: a window's length in 10 ms mel frames

	struct WindowRule
	{
		int tokEot, tokBeg;
		int maxTokens;        // whisper_full_params::max_tokens (<= 0: no limit)
		int singleSegment;
		int nMax;             // n_text_ctx / 2 - 4: the most tokens a window samples
	};

	// one window's state; wsp_window_result reports seekDelta, resultLen and failed
	struct WindowState
	{
		int hasTs;            // a timestamp token above tokBeg has been sampled
		int seekDelta;        // frames the window advances by
		int resultLen;        // tokens of the window's result
		int failed;           // no usable timestamp: whisper_full drops the window's tokens
		int ended;
	};

	WSP_HOST_DEVICE inline WindowState windowStart() { return WindowState{ 0, kWindowFrames, 0, 0, 0 }; }

	// Token `id`, sampled at step i (0 = the window's first sampled token) of the window at `seek` over a clip of seekEnd frames.
	// Returns whether the window has ended.  A token that goes back in time ends the window without being part of it.
	WSP_HOST_DEVICE inline bool windowStep( WindowState& s, const WindowRule& r, int seek, int seekEnd, int i, int id )
	{
		if( s.ended ) return true;
		if( id > r.tokBeg )                                                                          // :2946-2957
		{
			const int seekDeltaNew = 2 * ( id - r.tokBeg );
			if( s.hasTs && s.seekDelta > seekDeltaNew && s.resultLen < i )
			{
				s.ended = 1;
				return true;
			}
			s.seekDelta = seekDeltaNew;
			s.resultLen = i + 1;
			s.hasTs = 1;
		}
		if( id == r.tokEot || ( r.maxTokens > 0 && i >= r.maxTokens ) || ( s.hasTs && seek + s.seekDelta + 100 >= seekEnd ) )   // :2969-2988
		{
			s.ended = 1;
			if( s.resultLen == 0 )
			{
				if( seek + s.seekDelta + 100 >= seekEnd ) s.resultLen = i + 1;
				else
				{
					s.failed = 1;
					return true;
				}
			}
			if( r.singleSegment )
			{
				s.resultLen = i + 1;
				s.seekDelta = kWindowFrames;
			}
			return true;
		}
		if( i >= r.nMax - 1 )                                                                        // :3000-3003, and the loop's end
		{
			s.ended = 1;
			if( s.resultLen == 0 || s.seekDelta < kWindowFrames / 2 ) s.failed = 1;
		}
		return s.ended != 0;
	}
}

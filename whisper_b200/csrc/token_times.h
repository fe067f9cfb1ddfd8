// whisper_full's token-level timestamps and segment wrapping (Whisper/source/whisper.cpp:3320-3600, 2713-2763), once, on plain
// arrays: iContext::runFull (com_shell.cpp, built by g++) runs them per segment of its loop, wsp_window_token_times (c_api.cu) per
// segment of one batch window.  The signal energy they read is computed on the device (signal_energy_kernel, kernels_frontend.cu).
#pragma once
#include "../../include/whisper_b200.h"
#include <algorithm>
#include <stdint.h>

namespace wsp
{
	// what whisper_context carries from one segment to the next (t_beg / t_last / tid_last, whisper.cpp:425-431); whisper_full zeroes
	// it at the start of a call (:2803-2808)
	struct TokenTimeState
	{
		int64_t tBeg = 0, tLast = 0;
		int tidLast = 0;
	};

	// voice_length (whisper.cpp:3330-3353): a cost that is high for text that takes longer to pronounce
	inline float voiceLength( const char* text )
	{
		float res = 0.0f;
		for( const char* p = text ? text : ""; *p; p++ )
		{
			const char c = *p;
			if( c == ' ' ) res += 0.01f;
			else if( c == ',' ) res += 2.00f;
			else if( c == '.' || c == '!' || c == '?' ) res += 3.00f;
			else if( c >= '0' && c <= '9' ) res += 3.00f;
			else res += 1.00f;
		}
		return res;
	}

	// :3320-3322, clamped before the narrowing so that a span's times past 2^31 samples (offsets beyond 37 h) clamp as well
	inline int timestampToSample( int64_t t, int nSamples ) { return (int)std::max<int64_t>( 0, std::min<int64_t>( nSamples - 1, ( t * 16000 ) / 100 ) ); }
	inline int64_t sampleToTimestamp( int iSample ) { return ( 100 * (int64_t)iSample ) / 16000; }   // :3324-3326

	// whisper_exp_compute_token_level_timestamps (whisper.cpp:3374-3600) for one segment of n tokens over [t0, t1] (10 ms units):
	// timestamps from confident timestamp tokens, the gaps split in proportion to the voice lengths vlen[n], then every token grown or
	// shrunk against the signal energy[nSamples].  times[n] holds the tokens' times on entry (-1 where none) and on return.
	// Returns false, changing nothing, when there is no energy (the reference's "no signal data available").
	inline bool computeTokenTimes( const wsp_token_data* tokens, const float* vlen, wsp_token_time* times, int n, int64_t t0, int64_t t1,
		int tokBeg, int tokEot, const float* energy, int nSamples, float tholdPt, float tholdPtsum, TokenTimeState& st )
	{
		if( nSamples <= 0 ) return false;
		if( n == 0 ) return true;
		if( n == 1 ) { times[ 0 ].t0 = t0; times[ 0 ].t1 = t1; return true; }
		for( int j = 0; j < n; ++j )
		{
			const wsp_token_data& token = tokens[ j ];
			if( j == 0 )
			{
				if( token.id == tokBeg )
				{
					times[ j ].t0 = t0;
					times[ j ].t1 = t0;
					times[ j + 1 ].t0 = t0;
					st.tBeg = t0; st.tLast = t0; st.tidLast = tokBeg;
				}
				else times[ j ].t0 = st.tLast;
			}
			const int64_t tt = st.tBeg + 2 * ( (int64_t)token.tid - tokBeg );
			times[ j ].vlen = vlen[ j ];
			if( token.pt > tholdPt && token.ptsum > tholdPtsum && token.tid > st.tidLast && tt <= t1 )
			{
				if( j > 0 ) times[ j - 1 ].t1 = tt;
				times[ j ].t0 = tt;
				st.tidLast = token.tid;
			}
		}
		times[ n - 2 ].t1 = t1;
		times[ n - 1 ].t0 = t1;
		times[ n - 1 ].t1 = t1;
		st.tLast = t1;
		// intervals of tokens with unknown timestamps: split proportionally to the voice lengths
		{
			int p0 = 0, p1 = 0;
			while( true )
			{
				while( p1 < n && times[ p1 ].t1 < 0 ) p1++;
				if( p1 >= n ) p1--;
				if( p1 > p0 )
				{
					double psum = 0.0;
					for( int j = p0; j <= p1; j++ ) psum += times[ j ].vlen;
					const double dt = (double)( times[ p1 ].t1 - times[ p0 ].t0 );
					for( int j = p0 + 1; j <= p1; j++ )
					{
						const double ct = times[ j - 1 ].t0 + dt * times[ j - 1 ].vlen / psum;
						times[ j - 1 ].t1 = (int64_t)ct;
						times[ j ].t0 = (int64_t)ct;
					}
				}
				p1++;
				p0 = p1;
				if( p1 >= n ) break;
			}
		}
		// fix up (just in case)
		for( int j = 0; j < n - 1; j++ )
		{
			if( times[ j ].t1 < 0 ) times[ j + 1 ].t0 = times[ j ].t1;
			if( j > 0 && times[ j - 1 ].t1 > times[ j ].t0 )
			{
				times[ j ].t0 = times[ j - 1 ].t1;
				times[ j ].t1 = std::max( times[ j ].t0, times[ j ].t1 );
			}
		}
		// VAD: expand or contract tokens based on voice activity
		const int hw = 16000 / 8;
		for( int j = 0; j < n; j++ )
		{
			if( tokens[ j ].id >= tokEot ) continue;
			int s0 = timestampToSample( times[ j ].t0, nSamples );
			int s1 = timestampToSample( times[ j ].t1, nSamples );
			const int ss0 = std::max( s0 - hw, 0 );
			const int ss1 = std::min( s1 + hw, nSamples );
			const int ns = ss1 - ss0;
			float sum = 0.0f;
			for( int k = ss0; k < ss1; k++ ) sum += energy[ k ];
			const float thold = (float)( 0.5 * sum / ns );
			{
				int k = s0;
				if( energy[ k ] > thold && j > 0 )
				{
					while( k > 0 && energy[ k ] > thold ) k--;
					times[ j ].t0 = sampleToTimestamp( k );
					if( times[ j ].t0 < times[ j - 1 ].t1 ) times[ j ].t0 = times[ j - 1 ].t1;
					else s0 = k;
				}
				else
				{
					while( energy[ k ] < thold && k < s1 ) k++;
					s0 = k;
					times[ j ].t0 = sampleToTimestamp( k );
				}
			}
			{
				int k = s1;
				if( energy[ k ] > thold )
				{
					while( k < nSamples - 1 && energy[ k ] > thold ) k++;
					times[ j ].t1 = sampleToTimestamp( k );
					// (the reference tests `j < ns - 1` and then reads tokens[j + 1]: past the end for the last token of a segment
					// that does not close with a timestamp — undefined there, skipped here)
					if( j < ns - 1 && j + 1 < n && times[ j ].t1 > times[ j + 1 ].t0 ) times[ j ].t1 = times[ j + 1 ].t0;
					else s1 = k;
				}
				else
				{
					while( energy[ k ] < thold && k > s0 ) k--;
					s1 = k;
					times[ j ].t1 = sampleToTimestamp( k );
				}
			}
		}
		return true;
	}

	// whisper_wrap_segment (whisper.cpp:2713-2763) for a segment of tokens [i0, i1) over [t0, t1]: a new segment starts at the first
	// token whose text would take the current one past maxLen characters (special tokens, id >= tokEot, count nothing); it takes the
	// token's t0 as its start and the end of the current one.  textLen[i] = strlen of token i's text.  Writes the first `cap` pieces to
	// out and returns how many there are (at least one).  A piece's text is that of its non-special tokens.
	inline int wrapSegment( const wsp_token_data* tokens, const wsp_token_time* times, const int* textLen, int i0, int i1, int64_t t0, int64_t t1,
		int tokEot, int maxLen, wsp_segment* out, int cap )
	{
		int n = 0, start = i0, acc = 0;
		int64_t begin = t0;
		for( int k = i0; k < i1; k++ )
		{
			if( tokens[ k ].id >= tokEot ) continue;
			const int cur = textLen[ k ];
			if( acc + cur > maxLen && k > start )
			{
				// split here; the new segment's loop restarts at this token, where it cannot split again
				if( n < cap ) out[ n ] = wsp_segment{ begin, times[ k ].t0, start, k };
				n++;
				begin = times[ k ].t0;
				start = k;
				acc = cur;
			}
			else acc += cur;
		}
		if( n < cap ) out[ n ] = wsp_segment{ begin, t1, start, i1 };
		return n + 1;
	}
}

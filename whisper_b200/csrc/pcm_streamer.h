// Host side of iContext::runStreamed: the PCM queue between an audio source that delivers samples in stream order and the
// transcription loop that asks for 30 s windows at increasing offsets.
//
// Reference: Whisper/Whisper/MelStreamer.{h,cpp} + Whisper/MF/PcmReader.{h,cpp}.  There the queue holds 10 ms PCM chunks AND their
// mel columns, computed on the CPU either on demand (MelStreamerSimple) or ahead of time by a background thread that keeps 2 x 3000
// columns ready (MelStreamerThread, prebufferChunks).  Here a window's log-mel is a fraction of a millisecond of GPU time (mel_power_batch_kernel), so only
// the PCM is queued and the window is transformed when the loop asks for it; what the background thread buys is the SOURCE's
// latency (file reads, decoding, a live feed), and it keeps the same 60 s ahead.  Semantics kept from the reference:
//   * forward only: a window that starts before the previous one fails (MelStreamer.cpp:176-180 "doesn't support backwards seeks");
//   * samples before the current window's start are dropped (dropOldChunks :12-22);
//   * a window of `len` frames needs len*160 + 240 samples so that its last frame sees all 400 of its samples
//     (ensurePcmChunks asks for len + FFT_SIZE/FFT_STEP chunks, :31); at the end of the stream it gets what is left and the
//     transform pads with zeros (PcmReader::readChunk pads the last chunk, PcmReader.cpp:417-423).
// No CUDA in here: tests/boundary/streamer_test.cpp exercises this class on the CPU.
#pragma once
#include <condition_variable>
#include <deque>
#include <functional>
#include <mutex>
#include <stddef.h>
#include <stdint.h>
#include <string.h>
#include <thread>
#include <vector>

namespace wsp
{
	class PcmStreamer
	{
	public:
		// Pull up to `capacity` samples of 16 kHz mono PCM into dst; *written == 0 means end of stream.  Negative return = failure (an HRESULT).
		using ReadFn = std::function<int32_t( float* dst, uint32_t capacity, uint32_t* written )>;

		static constexpr size_t kHop = 160, kFft = 400;
		static constexpr size_t kBlock = 16000;                  // samples asked of the source per call (1 s)
		static constexpr size_t kPrebuffer = 2 * 3000 * kHop;    // the background thread stays this far ahead (MelStreamer.cpp: prebufferChunks)

		PcmStreamer( ReadFn readFn, size_t lengthFrames, bool background ) : read( std::move( readFn ) ), nFrames( lengthFrames )
		{
			if( background ) worker = std::thread( [ this ]() { threadMain(); } );
		}
		~PcmStreamer()
		{
			if( worker.joinable() )
			{
				{
					std::lock_guard<std::mutex> lk( mtx );
					shuttingDown = true;
				}
				wakeWorker.notify_all();
				worker.join();
			}
		}
		PcmStreamer( const PcmStreamer& ) = delete;
		PcmStreamer& operator=( const PcmStreamer& ) = delete;

		// length of the stream in mel frames, as announced by the source (iSpectrogram::getLength)
		size_t length() const { return nFrames; }
		// first frame still held
		size_t startFrame() const { return baseFrame; }

		// PCM for frames [off, off+len): *pcm points at sample off*160, *nSamples <= len*160 + 240 (less only at the end of the stream).
		// The pointer stays valid until the next call.  Returns 0, or a negative HRESULT (0x8000FFFF E_UNEXPECTED for a backward seek).
		int32_t window( size_t off, size_t len, const float** pcm, size_t* nSamples )
		{
			if( off < baseFrame ) return (int32_t)0x8000FFFF;
			const size_t want = len * kHop + ( kFft - kHop );
			// skipping ahead of what has been read so far simply consumes the stream up to there, a few blocks at a time
			size_t drop = ( off - baseFrame ) * kHop;
			while( drop > 0 )
			{
				const int32_t hr = fill( drop < 8 * kBlock ? drop : 8 * kBlock );
				if( hr < 0 ) return hr;
				if( held.empty() ) break;   // the stream ended before `off`
				const size_t n = drop < held.size() ? drop : held.size();
				held.erase( held.begin(), held.begin() + (ptrdiff_t)n );
				drop -= n;
			}
			baseFrame = off;
			const int32_t hr = fill( want );
			if( hr < 0 ) return hr;
			*pcm = held.data();
			*nSamples = held.size() < want ? held.size() : want;
			return 0;
		}

	private:
		ReadFn read;
		const size_t nFrames;
		std::vector<float> held;          // samples from frame `baseFrame` on, contiguous
		size_t baseFrame = 0;
		bool sourceEnded = false;

		// background reader
		std::thread worker;
		std::mutex mtx;
		std::condition_variable wakeWorker, wakeMain;
		std::deque<std::vector<float>> ready;
		size_t readySamples = 0;
		bool shuttingDown = false, workerEnded = false;
		int32_t workerStatus = 0;

		int32_t readBlock( std::vector<float>& blk )
		{
			blk.resize( kBlock );
			uint32_t got = 0;
			const int32_t hr = read( blk.data(), (uint32_t)kBlock, &got );
			if( hr < 0 ) { blk.clear(); return hr; }
			blk.resize( got <= kBlock ? got : kBlock );
			return 0;
		}

		// make `held` at least `samples` long, or as long as the stream allows
		int32_t fill( size_t samples )
		{
			while( held.size() < samples && !sourceEnded )
			{
				std::vector<float> blk;
				if( worker.joinable() )
				{
					std::unique_lock<std::mutex> lk( mtx );
					wakeMain.wait( lk, [ this ]() { return !ready.empty() || workerEnded; } );
					if( ready.empty() )
					{
						if( workerStatus < 0 ) return workerStatus;
						sourceEnded = true;
						break;
					}
					blk = std::move( ready.front() );
					ready.pop_front();
					readySamples -= blk.size();
					lk.unlock();
					wakeWorker.notify_one();
				}
				else
				{
					const int32_t hr = readBlock( blk );
					if( hr < 0 ) return hr;
					if( blk.empty() ) { sourceEnded = true; break; }
				}
				held.insert( held.end(), blk.begin(), blk.end() );
			}
			return 0;
		}

		void threadMain()
		{
			while( true )
			{
				{
					std::unique_lock<std::mutex> lk( mtx );
					wakeWorker.wait( lk, [ this ]() { return shuttingDown || readySamples < kPrebuffer; } );
					if( shuttingDown ) break;
				}
				std::vector<float> blk;
				const int32_t hr = readBlock( blk );
				std::lock_guard<std::mutex> lk( mtx );
				if( hr < 0 || blk.empty() )
				{
					workerStatus = hr;
					break;
				}
				readySamples += blk.size();
				ready.push_back( std::move( blk ) );
				wakeMain.notify_one();
			}
			{
				std::lock_guard<std::mutex> lk( mtx );
				workerEnded = true;
			}
			wakeMain.notify_all();
		}
	};
}

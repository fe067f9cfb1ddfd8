#!/usr/bin/env python
"""Cost of stereo chunks and per-segment speakers on the batch path (wsp_upload_pcm_stereo, wsp_chunk_speakers).

medium-sc (bench.py's model), batch 8, 30 s stereo chunks 0..7 with the 2 s left / right / balanced gain pattern of the tests.
- downmix_kernel: downmix_stereo_kernel's device time per chunk (torch.profiler with CUDA activities, mean over the launches of
  --steps uploads of the batch), with the bytes it must move (12 per frame: 8 read, 4 written) over the data sheet's 3.35 TB/s;
  and the host wall time of one wsp_upload_pcm_stereo, copy included;
- speaker_kernel: speaker_kernel's device time per call for three segment lists over the same 8 chunks: one 0..3000 segment per
  chunk; the segments of the window fixtures (tests/golden/chunks_window.npz, chunk b's list on stereo chunk b); the segments
  wsp_run_chunks_window returns for these chunks.  Also the host wall time of the whole wsp_chunk_speakers call;
- host_rule: the same answers from csrc/speaker.h on one host core (wsp_test_speakers), which the device answers must equal.
The first line names the card and its power limit, read in the same run with a read-only nvidia-smi query.

    python tools/speakers_sweep.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.audio_ctx_sweep import card  # noqa: E402
from whisper_b200 import capi, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


def gains_stereo(mono, rotate):
    t = np.arange(mono.size) / 16000.0
    g = np.choose(((t // 2).astype(np.int64) + rotate) % 3, [1.6, 0.4, 1.0]).astype(np.float32)
    return np.stack([mono * g, mono * (np.float32(2.0) - g)], axis=1).astype(np.float32)


def stats(xs):
    s = np.array(xs, np.float64)
    return round(float(np.median(s)), 3), [round(float(s.min()), 3), round(float(s.max()), 3)]


def kernel_us(fn, name, steps):
    """mean device time (us) of the kernels whose name contains `name`, over `steps` calls of fn, from torch.profiler"""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    total, count = 0.0, 0
    for ev in prof.events():
        if name in ev.name and ev.device_type.name == "CUDA":
            total += ev.time_range.elapsed_us()
            count += 1
    if count == 0:
        raise RuntimeError("the profiler recorded no %s launch" % name)
    return total / count, count


def window_fixture_segments(batch):
    g = np.load(os.path.join(ROOT, "tests", "golden", "chunks_window.npz"))
    lists = []
    for name in ("micro_en", "micro_ml"):
        segs = g[name + "_t4_segments"]
        for b in range(segs.shape[0]):
            lists.append([(int(s[0]), int(s[1])) for s in segs[b] if s[0] >= 0])
    return (lists * batch)[:batch]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="medium-sc")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    m = capi.Model(synth.model_path(a.model))
    e = capi.Engine(m, 0)
    c = capi.Context(e, a.batch)
    lrs = [gains_stereo(np.ascontiguousarray(synth.synth_pcm(i), np.float32), i) for i in range(a.batch)]
    frames = sum(x.shape[0] for x in lrs)
    print(json.dumps(dict(card(), model=a.model, batch=a.batch, frames=frames, steps=a.steps, warmup=a.warmup)), flush=True)

    def upload_all():
        for b, lr in enumerate(lrs):
            c.upload_pcm_stereo(b, lr)

    for _ in range(a.warmup):
        upload_all()
    wall = []
    for _ in range(a.steps):
        t = time.perf_counter()
        upload_all()
        wall.append((time.perf_counter() - t) * 1e3 / a.batch)
    us, n = kernel_us(upload_all, "downmix_stereo_kernel", a.steps)
    per_chunk = frames / a.batch
    bound_us = 12.0 * per_chunk / HBM_BYTES_PER_S * 1e6
    print(json.dumps({"leg": "downmix_kernel", "us_per_chunk": round(us, 2), "launches": n, "frames_per_chunk": per_chunk,
                      "hbm_bound_us": round(bound_us, 2), "share_of_bound": round(bound_us / us, 3),
                      "upload_wall_ms_per_chunk": stats(wall)[0], "upload_wall_ms_min_max": stats(wall)[1],
                      "what": "downmix_stereo_kernel device time (torch.profiler); host wall time of wsp_upload_pcm_stereo with its copy"}),
          flush=True)

    out, _ = c.run_chunks_window(None, m.prompt_init(), batch=a.batch, speakers=True)
    lists = {
        "one_30s_segment": [[(0, 3000)] for _ in range(a.batch)],
        "window_fixture_segments": window_fixture_segments(a.batch),
        "own_window_segments": [[(s["t0"], s["t1"]) for s in o["segments"]] for o in out],
    }
    for name, segs in lists.items():
        dsegs = [[dict(t0=t0, t1=t1) for t0, t1 in s] for s in segs]
        for _ in range(a.warmup):
            got = c.chunk_speakers(dsegs)
        wall = []
        for _ in range(a.steps):
            t = time.perf_counter()
            c.chunk_speakers(dsegs)
            wall.append((time.perf_counter() - t) * 1e3)
        us, n = kernel_us(lambda: c.chunk_speakers(dsegs), "speaker_kernel", a.steps)
        host = []
        for _ in range(max(3, a.steps // 4)):
            t = time.perf_counter()
            want = [capi.test_speakers(lr, s) for lr, s in zip(lrs, segs)]
            host.append((time.perf_counter() - t) * 1e3)
        assert got == want, name
        n_segs = sum(len(s) for s in segs)
        summed = sum(min(t1 - t0, 3000 - max(t0, 0)) * 160 for s in segs for t0, t1 in s if 0 <= t0 < 3000 and t1 > t0)
        longest = max((min(t1, 3000) - t0) * 160 for s in segs for t0, t1 in s) if n_segs else 0
        print(json.dumps({"leg": "speaker_kernel", "segments": name, "n_segments": n_segs, "frames_summed": summed,
                          "longest_segment_frames": longest, "kernel_us": round(us, 2), "launches": n,
                          "call_wall_ms": stats(wall)[0], "call_wall_ms_min_max": stats(wall)[1],
                          "answers": {str(k): int(sum(x == k for s in got for x in s)) for k in sorted({x for s in got for x in s})},
                          "what": "speaker_kernel device time (torch.profiler); host wall time of wsp_chunk_speakers"}), flush=True)
        print(json.dumps({"leg": "host_rule", "segments": name, "ms": stats(host)[0], "ms_min_max": stats(host)[1],
                          "what": "csrc/speaker.h on one host core (wsp_test_speakers) over the same segments; equal answers"}), flush=True)
    c.close()
    e.close()


if __name__ == "__main__":
    main()

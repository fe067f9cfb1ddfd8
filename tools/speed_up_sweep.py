#!/usr/bin/env python
"""Throughput of the measured path with speed-up (the 2x phase-vocoder log-mel, wsp_set_speed_up) against the default.

medium-sc (bench.py's model), batch 8, PCM resident in HBM (wsp_upload_pcm + wsp_run_chunks_resident), 100 greedy tokens per chunk.
Two legs in one process, alternated step by step after their warm-up: 30 s chunks with speed-up off, and 60 s chunks with speed-up on
(one 3000-frame encoder window each).  Per leg: one JSON line with the median mel / encode / decode stage milliseconds (CUDA events on
the library's stream) and audio-s/s counted in real audio seconds (batch x clip length / step time).  The first line names the card
and its power limit, read in the same run with a read-only nvidia-smi query.

    python tools/speed_up_sweep.py [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.audio_ctx_sweep import card  # noqa: E402
from whisper_b200 import capi, synth  # noqa: E402

LEGS = {"off_30s": (0, 480000), "on_60s": (1, 960000)}   # name: (speed-up, samples per chunk)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="medium-sc")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--n-decode", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    print(json.dumps(dict(card(), model=a.model, batch=a.batch, n_decode=a.n_decode, steps=a.steps, warmup=a.warmup)), flush=True)

    m = capi.Model(synth.model_path(a.model))
    e = capi.Engine(m, 0)
    prompt = m.prompt_init()
    ctxs = {}
    for name, (on, n) in LEGS.items():
        c = capi.Context(e, a.batch)
        c.set_reference_threads(16)            # bench.py's arithmetic
        c.set_speed_up(on)
        for i in range(a.batch):
            c.upload_pcm(i, synth.synth_pcm(i, n))
        for _ in range(max(1, a.warmup)):
            c.run_chunks_resident(a.batch, prompt, a.n_decode)
        ctxs[name] = c
    st = {name: [] for name in LEGS}
    for _ in range(a.steps):
        for name, c in ctxs.items():
            st[name].append(c.run_chunks_resident(a.batch, prompt, a.n_decode)[1])
    for name, (on, n) in LEGS.items():
        s = np.array(st[name], np.float64)
        med = np.median(s, axis=0)
        audio_s = a.batch * n / 16000.0
        print(json.dumps({"leg": name, "speed_up": on, "clip_s": n / 16000.0, "mel_ms": round(float(med[0]), 3), "encode_ms": round(float(med[1]), 3),
                          "decode_ms": round(float(med[2]), 3), "step_ms": round(float(med.sum()), 3),
                          "step_ms_min_max": [round(float(s.sum(1).min()), 3), round(float(s.sum(1).max()), 3)],
                          "audio_s_per_s": round(audio_s / (float(med.sum()) / 1000.0), 1)}), flush=True)
    for c in ctxs.values():
        c.close()
    e.close()


if __name__ == "__main__":
    main()

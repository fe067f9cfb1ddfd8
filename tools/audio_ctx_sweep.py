#!/usr/bin/env python
"""Stage times of the measured path at a shortened encoder context (sFullParams::audio_ctx, wsp_set_audio_ctx).

medium-sc (bench.py's model), batch 8, PCM resident in HBM (wsp_upload_pcm + wsp_run_chunks_resident), 100 greedy tokens per chunk,
at audio_ctx n in {1500, 1000, 750, 500, 250}.  Per n: warm-up steps, then --steps timed steps; one JSON line with the median mel /
encode / decode stage milliseconds (CUDA events on the library's stream) and the decoder step's algorithmic bytes, computed from
shapes: decoder weights (read once per step) + B x (cross-KV of n rows + self-KV rows of prompt + n_decode tokens).  The first line
names the card and its power limit, read in the same run with a read-only nvidia-smi query.

    python tools/audio_ctx_sweep.py [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from whisper_b200 import capi, synth  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, limit = [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")]
        return {"gpu": name, "power_limit": limit}
    except Exception as ex:     # the numbers still stand; they just lack their card
        return {"gpu": None, "power_limit": None, "error": str(ex)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="medium-sc")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--n-decode", type=int, default=100)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--audio-ctx", default="1500,1000,750,500,250")
    a = ap.parse_args()
    print(json.dumps(dict(card(), model=a.model, batch=a.batch, n_decode=a.n_decode, steps=a.steps, warmup=a.warmup)), flush=True)

    m = capi.Model(synth.model_path(a.model))
    e = capi.Engine(m, 0)
    c = capi.Context(e, a.batch)
    c.set_reference_threads(16)            # bench.py's arithmetic
    prompt = m.prompt_init()
    for i in range(a.batch):
        c.upload_pcm(i, synth.synth_pcm(i))
    d, L = m.n_text_state, m.n_text_layer
    weights = L * 14 * d * d * 2 + m.n_vocab * d * 2
    self_kv = L * 2 * (len(prompt) + a.n_decode) * d * 2
    for n in [int(x) for x in a.audio_ctx.split(",")]:
        c.set_audio_ctx(n)
        for _ in range(max(1, a.warmup)):
            c.run_chunks_resident(a.batch, prompt, a.n_decode)
        st = np.array([c.run_chunks_resident(a.batch, prompt, a.n_decode)[1] for _ in range(a.steps)], np.float64)
        cross_kv = L * 2 * n * d * 2
        step_bytes = weights + a.batch * (cross_kv + self_kv)
        med = np.median(st, axis=0)
        print(json.dumps({"audio_ctx": n, "mel_ms": round(float(med[0]), 3), "encode_ms": round(float(med[1]), 3), "decode_ms": round(float(med[2]), 3),
                          "step_ms": round(float(med.sum()), 3), "decode_ms_per_token": round(float(med[2]) / a.n_decode, 4),
                          "encode_ms_min_max": [round(float(st[:, 1].min()), 3), round(float(st[:, 1].max()), 3)],
                          "decode_ms_min_max": [round(float(st[:, 2].min()), 3), round(float(st[:, 2].max()), 3)],
                          "decode_step_bytes": step_bytes, "decode_step_gb": round(step_bytes / 1e9, 3)}), flush=True)
    c.close()
    e.close()


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Decode time of a batch stopped at end of text (wsp_run_chunks_until_eot) against the fixed-length batch at the ceiling
(wsp_run_chunks with n_decode = n_text_ctx - n_prompt), on the same inputs, alternated call by call in one process.

medium-sc (bench.py's model), batch 8, host PCM, reference threads 4.  Two batches:
- script_30s: chunks 0..7 of 30 s each; the scripted model ends each of them with EOT after about 45 tokens.
- mixed: 30 s clips and clips of 27.5, 26.25 and 25 s, zero-padded to the window; the padded ones leave the script, and a chunk
  that never samples EOT keeps the batch running to the ceiling (then the difference is the cost of the end-of-text log itself).
Per batch and call form: one JSON line with the median decode stage milliseconds (CUDA events on the library's stream), the min / max,
and the decoder steps run.  The first line names the card and its power limit, read in the same run with a read-only nvidia-smi query.

    python tools/eot_sweep.py [--steps 5] [--warmup 2]
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

MIXED_LENGTHS = (480000, 440000, 420000, 400000)   # 30 s and zero-padded clips (tests/test_gpu_chunks_eot.py's GPU-only batches)


def batches(n):
    return {"script_30s": [synth.synth_pcm(i) for i in range(n)],
            "mixed": [synth.synth_pcm(i, MIXED_LENGTHS[i % len(MIXED_LENGTHS)]) for i in range(n)]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="medium-sc")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    m = capi.Model(synth.model_path(a.model))
    e = capi.Engine(m, 0)
    c = capi.Context(e, a.batch)
    prompt = m.prompt_init()
    ceiling = m.n_text_ctx - len(prompt)
    print(json.dumps(dict(card(), model=a.model, batch=a.batch, max_decode=ceiling, steps=a.steps, warmup=a.warmup)), flush=True)

    def fixed(pcms):
        return c.run_chunks(pcms, prompt, ceiling)[1][2]

    def until_eot(pcms):
        return c.run_chunks_until_eot(pcms, prompt, ceiling)[1][2]

    forms = {"run_chunks": fixed, "until_eot": until_eot}
    for bname, pcms in batches(a.batch).items():
        ms = {f: [] for f in forms}
        steps = {}
        for i in range(a.warmup + a.steps):
            for f, call in forms.items():
                c.timings(reset=True)
                t = call(pcms)
                steps[f] = int(c.timings()[1][2])
                if i >= a.warmup:
                    ms[f].append(t)
        lens = [len(t) for t in c.run_chunks_until_eot(pcms, prompt, ceiling)[0]]
        for f in forms:
            s = np.array(ms[f], np.float64)
            print(json.dumps({"batch": bname, "call": f, "decode_ms": round(float(np.median(s)), 3),
                              "decode_ms_min_max": [round(float(s.min()), 3), round(float(s.max()), 3)],
                              "steps_run": steps[f], "n_out": lens}), flush=True)
    c.close()
    e.close()


if __name__ == "__main__":
    main()

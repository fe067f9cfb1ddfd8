#!/usr/bin/env python
"""Cost of per-chunk language detection on the batch path: wsp_run_chunks_until_eot with [sot, WSP_TOKEN_LANGUAGE_AUTO, transcribe]
against the same call with the language fixed, on the same inputs, alternated call by call in one process.  The fixed prompt holds the
language one auto call detects for most chunks; when it is every chunk's, both prompts decode the same tokens, so the difference is
the detection pass alone.

medium-sc (bench.py's model), batch 8, resident PCM (wsp_upload_pcm), reference threads 4, max_decode = n_text_ctx - 3, scripted 30 s
chunks 0..7.  Per prompt: one JSON line with the median decode stage milliseconds (CUDA events on the library's stream; the detection
pass is part of it), min / max, the decoder steps run and the milliseconds per step.  The last line gives the difference of the
medians and whether the two prompts gave the same tokens.  The first line names the card and its power
limit, read in the same run with a read-only nvidia-smi query.

    python tools/lang_sweep.py [--steps 5] [--warmup 2]
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
    for b in range(a.batch):
        c.upload_pcm(b, synth.synth_pcm(b))
    auto = m.prompt_init("auto")
    ceiling = m.n_text_ctx - len(auto)
    auto_toks, _ = c.run_chunks_until_eot(None, auto, ceiling, batch=a.batch)
    langs = c.chunk_languages(a.batch)[0].tolist()
    fixed_lang = max(set(langs), key=langs.count)
    prompts = {"fixed": m.prompt_init(fixed_lang), "auto": auto}
    fixed_toks, _ = c.run_chunks_until_eot(None, prompts["fixed"], ceiling, batch=a.batch)
    same_tokens = [t.tolist() for t in auto_toks] == [t.tolist() for t in fixed_toks]
    print(json.dumps(dict(card(), model=a.model, batch=a.batch, max_decode=ceiling, steps=a.steps, warmup=a.warmup,
                          languages=langs, fixed_language=fixed_lang)), flush=True)
    ms = {p: [] for p in prompts}
    steps = {}
    for i in range(a.warmup + a.steps):
        for p, prompt in prompts.items():
            c.timings(reset=True)
            _toks, st = c.run_chunks_until_eot(None, prompt, ceiling, batch=a.batch)
            steps[p] = int(c.timings()[1][2])
            if i >= a.warmup:
                ms[p].append(float(st[2]))
    med = {}
    for p in prompts:
        s = np.array(ms[p], np.float64)
        med[p] = float(np.median(s))
        print(json.dumps({"prompt": p, "decode_ms": round(med[p], 3), "decode_ms_min_max": [round(float(s.min()), 3), round(float(s.max()), 3)],
                          "steps_run": steps[p], "ms_per_step": round(med[p] / steps[p], 4)}), flush=True)
    print(json.dumps({"detect_ms": round(med["auto"] - med["fixed"], 3), "same_steps": steps["auto"] == steps["fixed"],
                      "same_tokens": same_tokens}), flush=True)
    c.close()
    e.close()


if __name__ == "__main__":
    main()

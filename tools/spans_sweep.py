#!/usr/bin/env python
"""Cost of span windows over one long resident source (wsp_run_spans_window).

medium-sc (bench.py's model), B = 8 windows of one 5-minute source at offsets 0, 30, ..., 210 s (duration 0), three ways:
- shared: one spans call, every row on slot 0 (the source's log-mel computed once);
- copies: one spans call over the source uploaded to 8 slots, row b on slot b (8 log-mels in one mel launch triple);
- sequential: 8 spans calls at B = 1 on slot 0 (the log-mel computed 8 times).
Each is run --steps times after --warmup runs; reported per way: the median (and range) of the mel, encode and decode stage times
(CUDA events, stage_ms), of the host wall time around the whole call(s), the kernel launches per run, and wsp_context_device_bytes.
The rows' results must be identical across the three ways.  The first line names the card and its power limit, read in the same run
with a read-only nvidia-smi query.

    python tools/spans_sweep.py [--steps 5] [--warmup 1]
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


def stats(xs):
    s = np.array(xs, np.float64)
    return round(float(np.median(s)), 3), [round(float(s.min()), 3), round(float(s.max()), 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="medium-sc")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--seconds", type=int, default=300)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    L = capi.lib()
    if L.wsp_device_count() < 1:
        raise SystemExit("spans_sweep: no CUDA device")
    print(json.dumps(card()), flush=True)
    m = capi.Model(synth.model_path(a.model))
    e = capi.Engine(m, 0)
    # a 5-minute source from 30 s pieces of the clip family the scripted models were calibrated on
    pcm = np.concatenate([synth.synth_pcm(k, 480000) for k in range(a.seconds // 30)]).astype(np.float32)
    offs = [30000 * k for k in range(a.batch)]
    prompt = m.prompt_init()
    ways = {
        "shared": (1, lambda c: [c.run_spans_window([(0, o, 0) for o in offs], prompt)]),
        "copies": (a.batch, lambda c: [c.run_spans_window([(b, o, 0) for b, o in enumerate(offs)], prompt)]),
        "sequential": (1, lambda c: [c.run_spans_window([(0, o, 0)], prompt) for o in offs]),
    }
    results = {}
    for name, (slots, run) in ways.items():
        c = capi.Context(e, a.batch)
        for s in range(slots):
            c.upload_pcm(s, pcm)
        for _ in range(a.warmup):
            run(c)
        mel, enc, dec, wall, launches = [], [], [], [], []
        for _ in range(a.steps):
            before = L.wsp_launch_count()
            t0 = time.perf_counter()
            outs = run(c)
            wall.append((time.perf_counter() - t0) * 1e3)
            launches.append(int(L.wsp_launch_count() - before))
            st = np.sum([o[1] for o in outs], axis=0)
            mel.append(st[0]); enc.append(st[1]); dec.append(st[2])
        rows = [r for o in outs for r in o[0]]
        results[name] = [(r["result"], [t["id"] for t in r["tokens"]]) for r in rows]
        print(json.dumps(dict(way=name, model=a.model, batch=a.batch, source_s=pcm.size / 16000, mel_ms=stats(mel), encode_ms=stats(enc),
                              decode_ms=stats(dec), wall_ms=stats(wall), launches=stats(launches)[0],
                              device_bytes=int(L.wsp_context_device_bytes(c.h)))), flush=True)
        c.close()
    same = results["shared"] == results["copies"] == results["sequential"]
    print(json.dumps(dict(identical_rows=same)), flush=True)
    if not same:
        raise SystemExit("spans_sweep: the three ways disagree")


if __name__ == "__main__":
    main()

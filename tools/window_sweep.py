#!/usr/bin/env python
"""Cost of whisper_full's window rule and token-data log on the batch path, and what the batch path saves over one clip at a time.

medium-sc (bench.py's model), batch 8, host PCM, reference threads 4, chunks 0..7 of 30 s (the scripted model ends each with EOT after
about 45 tokens).  Three calls on the same clips, alternated call by call in one process:
- window: wsp_run_chunks_window (max_tokens 0), decode stage milliseconds from CUDA events;
- until_eot: wsp_run_chunks_until_eot with max_decode = n_max on the same chunks, the same decode stage;
- run_full: the clips one after another through iContext::runFull (the COM layer, tests/boundary's shim), host wall time of the B
  calls, which includes their mel and encode and every later window of each clip.
One JSON line per call with the median and min / max over --steps, and the steps the batch ran.  The first line names the card and its
power limit, read in the same run with a read-only nvidia-smi query.

    python tools/window_sweep.py [--steps 5] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.audio_ctx_sweep import card  # noqa: E402
from whisper_b200 import capi, synth  # noqa: E402

# the flat helpers over the COM vtables that __graft_entry__.build() compiles (ctypes cannot call vtables)
COM_HELPERS = os.path.join(ROOT, "tests", "boundary", "_build", "libwspc_test.so")


def com_session(model):
    """(library, session) of one iModel + iContext on device 0, driven through wspc_open / wspc_run_full"""
    capi.lib()                       # the helpers link against the product library
    L = C.CDLL(COM_HELPERS)
    vp, i32 = C.c_void_p, C.c_int32
    L.wspc_open.restype = i32
    L.wspc_open.argtypes = [C.c_char_p, i32, C.POINTER(vp)]
    L.wspc_close.argtypes = [vp]
    L.wspc_run_full.restype = i32
    L.wspc_run_full.argtypes = [vp, C.POINTER(C.c_float), i32, C.c_uint32, C.c_char_p, i32, i32, i32, i32, C.POINTER(i32), i32]
    h = C.c_void_p()
    hr = L.wspc_open(synth.model_path(model).encode(), 0, C.byref(h))
    assert hr == 0, hex(hr & 0xFFFFFFFF)
    return L, h


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
    n_max = m.n_text_ctx // 2 - 4
    pcms = [synth.synth_pcm(i) for i in range(a.batch)]
    print(json.dumps(dict(card(), model=a.model, batch=a.batch, n_max=n_max, steps=a.steps, warmup=a.warmup)), flush=True)

    L, h = com_session(a.model)

    def window():
        c.timings(reset=True)
        st = c.run_chunks_window(pcms, prompt)[1]
        return st[2], int(c.timings()[1][2])

    def until_eot():
        c.timings(reset=True)
        st = c.run_chunks_until_eot(pcms, prompt, n_max)[1]
        return st[2], int(c.timings()[1][2])

    def run_full():
        t = time.perf_counter()
        for p in pcms:
            arr = np.ascontiguousarray(p, np.float32)
            hr = L.wspc_run_full(h, arr.ctypes.data_as(C.POINTER(C.c_float)), arr.size, 0, b"en", 0, 4, 0, 0, None, 0)
            assert hr == 0, hex(hr & 0xFFFFFFFF)
        return (time.perf_counter() - t) * 1e3, None

    forms = {"window": window, "until_eot": until_eot, "run_full": run_full}
    ms = {f: [] for f in forms}
    steps = {}
    for i in range(a.warmup + a.steps):
        for f, call in forms.items():
            t, s = call()
            steps[f] = s
            if i >= a.warmup:
                ms[f].append(t)
    out, _ = c.run_chunks_window(pcms, prompt)
    for f in forms:
        s = np.array(ms[f], np.float64)
        print(json.dumps({"call": f, "ms": round(float(np.median(s)), 3), "ms_min_max": [round(float(s.min()), 3), round(float(s.max()), 3)],
                          "what": "host wall time of B runFull calls" if f == "run_full" else "decode stage (CUDA events)",
                          "steps_run": steps[f], "n_sampled": [o["result"]["n_sampled"] for o in out] if f == "window" else None}), flush=True)
    L.wspc_close(h)
    c.close()
    e.close()


if __name__ == "__main__":
    main()

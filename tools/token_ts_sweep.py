#!/usr/bin/env python
"""Cost of token-level timestamps on the batch path: the signal energy on the device and whisper_full's token times on the host.

medium-sc (bench.py's model), batch 8, host PCM, reference threads 4, chunks 0..7 of 30 s.  wsp_run_chunks_window runs alternately
on two contexts of the same engine, one with token timestamps off and one with them on, call by call in one process; --warmup calls
of each first, then the median (min / max) of --steps.  Per leg: the three stage times (CUDA events) and the call's host wall time.
Then, for the same clips:
- energy_kernel: signal_energy_kernel alone over the batch (wsp_test_signal_energy), CUDA events around 20 launches, with the bytes
  it must move (8 per sample: one f32 read, one written) over the data sheet's 3.35 TB/s as its lower bound;
- token_times: host wall time of wsp_window_token_times over the 8 chunks, at max_len 0 and 12;
- host_energy: the reference's get_signal_energy loop (whisper.cpp:3356-3372) compiled with gcc -O2 into a temporary directory,
  over the same 8 clips on one host core: what computing the energy on the host would cost.
The first line names the card and its power limit, read in the same run with a read-only nvidia-smi query.

    python tools/token_ts_sweep.py [--steps 5] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.audio_ctx_sweep import card  # noqa: E402
from whisper_b200 import capi, synth  # noqa: E402

HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet

# get_signal_energy as the reference writes it, for the host comparison
HOST_ENERGY_C = r"""
#include <math.h>
void signal_energy( const float* signal, int n_samples, int hw, float* result )
{
	for( int i = 0; i < n_samples; i++ )
	{
		float sum = 0;
		for( int j = -hw; j <= hw; j++ )
			if( i + j >= 0 && i + j < n_samples ) sum += fabsf( signal[ i + j ] );
		result[ i ] = sum / ( 2 * hw + 1 );
	}
}
"""


def host_energy_lib(tmp):
    src, so = os.path.join(tmp, "energy.c"), os.path.join(tmp, "libenergy.so")
    with open(src, "w") as f:
        f.write(HOST_ENERGY_C)
    subprocess.run(["gcc", "-O2", "-shared", "-fPIC", src, "-o", so], check=True)
    L = C.CDLL(so)
    L.signal_energy.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.POINTER(C.c_float)]
    return L


def stats(xs):
    s = np.array(xs, np.float64)
    return round(float(np.median(s)), 3), [round(float(s.min()), 3), round(float(s.max()), 3)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="medium-sc")
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    m = capi.Model(synth.model_path(a.model))
    e = capi.Engine(m, 0)
    ctx = {"off": capi.Context(e, a.batch), "on": capi.Context(e, a.batch)}
    ctx["on"].set_token_timestamps(1)
    prompt = m.prompt_init()
    pcms = [np.ascontiguousarray(synth.synth_pcm(i), np.float32) for i in range(a.batch)]
    samples = sum(p.size for p in pcms)
    print(json.dumps(dict(card(), model=a.model, batch=a.batch, samples=samples, steps=a.steps, warmup=a.warmup)), flush=True)

    stage, wall = {k: [] for k in ctx}, {k: [] for k in ctx}
    for i in range(a.warmup + a.steps):
        for leg, c in ctx.items():
            t = time.perf_counter()
            _out, st = c.run_chunks_window(pcms, prompt)
            w = (time.perf_counter() - t) * 1e3
            if i >= a.warmup:
                stage[leg].append(st.tolist())
                wall[leg].append(w)
    for leg in ctx:
        st = np.array(stage[leg])
        print(json.dumps({"leg": "energy " + leg, "stage_ms": [stats(st[:, k])[0] for k in range(3)],
                          "mel_stage_ms_min_max": stats(st[:, 0])[1], "wall_ms": stats(wall[leg])[0], "wall_ms_min_max": stats(wall[leg])[1],
                          "what": "wsp_run_chunks_window: {mel (+ energy), encode, decode} from CUDA events; host wall time of the call"}), flush=True)

    energies, ms = capi.test_signal_energy(pcms, iters=20)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(energies, [ctx["on"].get_tensor("energy", b) for b in range(a.batch)]))
    bound_us = 8.0 * samples / HBM_BYTES_PER_S * 1e6
    print(json.dumps({"leg": "energy_kernel", "us": round(ms * 1e3, 2), "bytes": 8 * samples, "hbm_bound_us": round(bound_us, 2),
                      "share_of_bound": round(bound_us / (ms * 1e3), 3),
                      "what": "signal_energy_kernel over the batch, mean of 20 launches between CUDA events"}), flush=True)

    # token times on the host, from the "on" context's last window call
    c = ctx["on"]
    out, _ = c.run_chunks_window(pcms, prompt)
    L = capi.lib()
    cap = m.n_text_ctx // 2 - 4
    data = []
    for b, o in enumerate(out):
        toks = (capi.TokenData * cap)(*[capi.TokenData(t["id"], t["tid"], t["p"], t["pt"], t["ptsum"]) for t in o["tokens"]])
        r = o["result"]
        data.append((toks, capi.WindowResult(r["n_sampled"], r["n_tokens"], r["seek_delta"], r["failed"]), (capi.TokenTime * cap)(),
                     (capi.Segment * (4 * cap))()))
    n_segs = np.zeros(1, np.int32)
    for max_len in (0, 12):
        prm = capi.TokenTimeParams(0.01, 0.01, max_len)
        ts = []
        for i in range(a.warmup + a.steps):
            t = time.perf_counter()
            for b, (toks, res, times, segs) in enumerate(data):
                capi.check(L.wsp_window_token_times(c.h, b, toks, C.byref(res), 0, C.byref(prm), segs, len(segs), capi._i(n_segs), times))
            if i >= a.warmup:
                ts.append((time.perf_counter() - t) * 1e3)
        med, mm = stats(ts)
        print(json.dumps({"leg": "token_times", "max_len": max_len, "ms": med, "ms_min_max": mm,
                          "tokens": sum(o["result"]["n_tokens"] for o in out),
                          "what": "host wall time of wsp_window_token_times over the %d chunks" % a.batch}), flush=True)

    with tempfile.TemporaryDirectory() as tmp:
        H = host_energy_lib(tmp)
        dst = [np.empty_like(p) for p in pcms]
        ts = []
        for i in range(1 + a.steps):
            t = time.perf_counter()
            for p, d in zip(pcms, dst):
                H.signal_energy(capi._f(p), p.size, 32, capi._f(d))
            if i >= 1:
                ts.append((time.perf_counter() - t) * 1e3)
        assert all(x.tobytes() == y.tobytes() for x, y in zip(dst, energies))
        med, mm = stats(ts)
        print(json.dumps({"leg": "host_energy", "ms": med, "ms_min_max": mm,
                          "what": "get_signal_energy's loop, gcc -O2, one host core, over the %d clips" % a.batch}), flush=True)
    for c in ctx.values():
        c.close()
    e.close()


if __name__ == "__main__":
    main()

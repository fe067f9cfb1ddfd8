#!/usr/bin/env python
"""bench.py against two builds of libwhisper_b200.so on the same card in one run, alternating A, B, A, B, ...

bench.py loads whisper_b200/libwhisper_b200.so; this driver copies each candidate over it in turn, runs bench.py in a process of
its own, and puts the library it found back when it is done.  Per build: every run's value (audio-s/s), mel / encode / decode stage
milliseconds per step and decoder-step-kernel milliseconds per launch, then their medians and spread (min .. max).  The first line
names the card and its power limit, read in the same run with a read-only nvidia-smi query.

    python tools/ab_bench.py --a old/libwhisper_b200.so --b new/libwhisper_b200.so [--rounds 3] [-- <bench.py arguments>]
"""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tools.audio_ctx_sweep import card  # noqa: E402

LIB = os.path.join(ROOT, "whisper_b200", "libwhisper_b200.so")


def run_bench(lib, bench_args):
    shutil.copyfile(lib, LIB)
    out = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py")] + bench_args, cwd=ROOT, capture_output=True, text=True)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith("{")]
    if out.returncode != 0 or not lines:
        raise RuntimeError("bench.py failed with %s:\n%s" % (lib, out.stderr[-2000:]))
    r = json.loads(lines[-1])
    st = r["stage_ms_per_step"]
    return {"value": r["value"], "mel_ms": st["mel"], "encode_ms": st["encode"], "decode_ms": st["decode"],
            "step_kernel_ms_per_launch": r["roofline"]["ms_per_launch"], "tokens_match_reference_fixture": r["tokens_match_reference_fixture"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True)
    ap.add_argument("--b", required=True)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("bench_args", nargs="*", default=[])
    a = ap.parse_args()
    bench_args = a.bench_args or ["--gpus", "1", "--steps", "5", "--warmup", "2", "--no-cpu-baseline"]
    print(json.dumps(card()), flush=True)
    runs = {"a": [], "b": []}
    with tempfile.TemporaryDirectory() as tmp:
        keep = os.path.join(tmp, "lib.so")
        shutil.copyfile(LIB, keep)
        try:
            for i in range(a.rounds):
                for leg, lib in (("a", a.a), ("b", a.b)):
                    r = run_bench(os.path.abspath(lib), bench_args)
                    runs[leg].append(r)
                    print(json.dumps({"leg": leg, "round": i, **r}), flush=True)
        finally:
            shutil.copyfile(keep, LIB)
    for leg in ("a", "b"):
        summary = {"leg": leg, "runs": len(runs[leg])}
        for k in ("value", "mel_ms", "encode_ms", "decode_ms", "step_kernel_ms_per_launch"):
            v = np.array([r[k] for r in runs[leg]])
            summary[k] = {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}
        print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()

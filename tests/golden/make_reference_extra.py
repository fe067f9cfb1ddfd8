"""TEST INFRASTRUCTURE — golden vectors for the tests that used to call the reference live.

Generates tests/golden/reference_extra.npz from oracle/_ref (the reference's own CPU code, built by oracle/Makefile) so that
those comparisons run wherever the repository is checked out:
  * tiny_*: log-mel, cross-attention K memory (every CROSS_T_STEP-th time step) and 20 greedy tokens of the tiny.en-sc model on
    synth_pcm(5), a chunk with no other fixture (tests/test_gpu_parity.py::test_reference_tiny_chunk);
  * vad_s<seed>: the reference detector's detect() results for seeds 100..129 (tests/test_vad.py);
  * sampler_*: the reference sampler's decision on every row of tests/test_gpu_sampler.make_rows (ties included), with the
    probabilities given by the restated f16-table softmax (oracle/whisper_np.softmax_rows).

    python tests/golden/make_reference_extra.py
"""
import ctypes as C
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

TINY_MODEL, TINY_CHUNK, TINY_STEPS = "tiny.en-sc", 5, 20
CROSS_T_STEP = 30
VAD_SEEDS = range(100, 130)
SAMPLER_MODEL = "micro.en"


def main():
    from oracle import ref
    from oracle import whisper_np as wn
    from tests.golden.make_golden import MEL_STEP
    from tests.golden.make_vad_golden import drive
    from tests.test_gpu_sampler import BEG, make_rows
    from whisper_b200 import capi, synth

    out = {}
    o = ref.RefOracle(synth.model_path(TINY_MODEL), threads=4)
    pcm = synth.synth_pcm(TINY_CHUNK)
    out["tiny_mel"] = o.pcm_to_mel(pcm)[:, ::MEL_STEP].astype(np.float32)
    o.encode(0)
    ck, _ = o.cross_kv()
    out["tiny_cross_k"] = ck[:, ::CROSS_T_STEP, :].astype(np.float32)
    m = capi.Model(synth.model_path(TINY_MODEL))
    prompt = m.prompt_init()
    _, toks, _ = o.bench_chunk(pcm, prompt, TINY_STEPS)
    out["tiny_prompt"] = np.asarray(prompt, np.int32)
    out["tiny_tokens"] = np.asarray(toks, np.int32)

    vad = C.CDLL(os.path.join(ROOT, "oracle", "_ref", "liboracle_vad.so"))
    for seed in VAD_SEEDS:
        out["vad_s%d" % seed] = np.asarray(drive(vad, "ora_vad", seed), np.int64)

    so = ref.RefOracle(synth.model_path(SAMPLER_MODEL), threads=1)
    res = []
    for lg, force_ts, initial, label in make_rows():
        for r in range(lg.shape[0]):
            s = so.sample_from_probs(wn.softmax_rows(lg[r]), force_ts, initial)
            res.append([s["id"], s["tid"], s["p"], s["pt"], s["ptsum"]])
    res = np.asarray(res, np.float64)
    out["sampler_ids"] = res[:, :2].astype(np.int64)
    out["sampler_p_pt_ptsum"] = res[:, 2:]
    print("tiny tokens", out["tiny_tokens"].tolist(), "| sampler rows", len(res), "| ts decisions", int((out["sampler_ids"][:, 0] >= BEG).sum()))
    np.savez_compressed(os.path.join(HERE, "reference_extra.npz"), **out)


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Generate tests/golden/audio_ctx.npz from oracle/_ref — the reference's own CPU implementation — for sFullParams::audio_ctx, the
shortened encoder context (whisper.cpp:1092-1167, 1479-1480, 1528, 2836): the encoder reads mel frames [offset, offset + 2n), the
cross-K/V memories hold n rows per layer and the decoder cross-attends over n keys.

Encode / decode-level cases: for micro.en-sc and micro-sc at every n of AUDIO_CTX — the encoder input window and encoder trace
points, the cross-K/V memories, the prompt and teacher-forced step logits and the greedy tokens at reference threads 1, 4 and 16
(the reference's f16 V^T*P chains are split over its threads, ggml.c:4680-4722: at n = 16 each of 16 threads owns one key, at
n = 100 the 16th owns none).
The PCM chunk is searched the way make_golden.make() does (GAP_SAFE, MIN_DISTINCT).  A shortened context may throw the scripted
decoder off its script; where none of the tried chunks is clean, the case pins its tensors and logits only: its "<key>_tokens_pinned"
entry is 0 and the tests then compare logits step by step under teacher forcing but not the free-running tokens.

whisper_full runs on the -sc1 models over the 78 s clip of make_golden.full_pcm: .en at audio_ctx 750; .en at 384 with an offset and
max_tokens; the multilingual model with language "de" and 750 followed, on the same context, by a second call with "auto" and 0 —
whisper_full detects the language BEFORE it overwrites exp_n_audio_ctx (:2789-2801, then :2836), so that detection still runs at 750.

The oracle build exports no setter for exp_n_audio_ctx; `set_audio_ctx` below reaches it through whisper_full itself: a call on one
second of silence with duration_ms = 1000 passes the 1 s check (:2814), overwrites exp_n_audio_ctx (:2836) and leaves the seek loop
before its first encode (:2871).  It also replaces the context's mel, so it is called before set_mel.

    python tests/golden/make_audio_ctx_golden.py        # rewrites tests/golden/audio_ctx.npz
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from oracle.ref import RefOracle  # noqa: E402
from tests.golden.make_golden import (FULL_MODEL, FULL_MODEL_ML, GAP_SAFE, LOGIT_STEP, MIN_DISTINCT, full_pcm, greedy,  # noqa: E402
                                      logits_sample, prompt_of)
from whisper_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "audio_ctx.npz")

AUDIO_CTX = (1499, 750, 129, 128, 100, 16)   # just under the default, half, both sides of one 128-key tile, short ones
MODELS = {"en": ("micro.en-sc", 0), "ml": ("micro-sc", 3)}   # key: (model, first PCM chunk id tried)
THREADS = (1, 4, 16)
N_STEPS = 24           # greedy steps stored per case
CHUNK_TRIES = 12
ROWS_KEPT = 24         # time rows kept of every [n][d] / [2n][.] tensor ...
COL_STEP = 8           # ... and every 8th channel of those rows
LOGIT_THIN = 8         # logits: every 8th entry of make_golden's sub-sample, i.e. every 488th vocabulary entry


def rows_of(n: int) -> np.ndarray:
    """Sub-sampled time rows of an n-row tensor: evenly spaced, always including the first and the last (the padded edge)."""
    return np.unique(np.linspace(0, n - 1, min(n, ROWS_KEPT)).round().astype(np.int64))


def set_audio_ctx(o: RefOracle, n: int):
    """exp_n_audio_ctx = n through whisper_full (see the module docstring); replaces the oracle's mel."""
    silence = np.zeros(16000, np.float32)
    rc = o.L.ora_full_ex(o.ctx, silence.ctypes.data_as(C.POINTER(C.c_float)), silence.size, o.threads, 2, b"en", 0, n, 0, 1000)
    assert rc == 0


def cross_kv(o: RefOracle, n: int):
    """The cross-K/V memories of the last encode: n rows per layer, packed (whisper.cpp:1479-1480) -> [L][n][d] each."""
    k, v = o.cross_kv()
    L, d = o.n_text_layer, o.n_text_state
    return (a.reshape(-1)[: L * n * d].reshape(L, n, d) for a in (k, v))


def run_case(model: str, mel: np.ndarray, n: int, th: int):
    o = RefOracle(synth.model_path(model), threads=th)
    set_audio_ctx(o, n)
    o.set_mel(mel)
    o.encode(0)
    return o, greedy(o, prompt_of(o), N_STEPS, keep_logits=True)


def make_case(key: str, model: str, chunk0: int, n: int, out: dict):
    first = None
    for chunk in range(chunk0, chunk0 + CHUNK_TRIES):
        o1 = RefOracle(synth.model_path(model), threads=1)
        mel = o1.pcm_to_mel(synth.synth_pcm(chunk, 480000))
        # the cheap thread counts first: 16 spin-waiting reference threads are slow on a small host
        runs = {}
        for th in THREADS:
            runs[th] = run_case(model, mel, n, th)[1]
            worst = min(float(r["gap"].min()) for r in runs.values())
            distinct = min(len(set(r["tokens"].tolist())) for r in runs.values())
            if first is not None and not (worst >= GAP_SAFE and distinct >= MIN_DISTINCT):
                break
        print("  %s n=%d chunk %d: min gap %.3f, distinct %d" % (key, n, chunk, worst, distinct), flush=True)
        if first is None:
            first = (chunk, mel, runs)
        if len(runs) == len(THREADS) and worst >= GAP_SAFE and distinct >= MIN_DISTINCT:
            pinned = True
            break
    else:
        chunk, mel, runs = first
        pinned = False
        print("  %s n=%d: no clean chunk in %d tries — tensors and logits only" % (key, n, CHUNK_TRIES), flush=True)
    p = "%s_n%d_" % (key, n)
    out[p + "chunk"] = np.int32(chunk)
    out[p + "tokens_pinned"] = np.int32(pinned)
    o = RefOracle(synth.model_path(model), threads=1)
    set_audio_ctx(o, n)
    o.set_mel(mel)
    o.trace(True)
    o.encode(0)
    tr = o.trace_items()
    o.trace(False)
    d = o.n_audio_state
    r1, r2 = rows_of(n), rows_of(2 * n)
    out[p + "enc_input"] = tr["enc.input"].reshape(o.n_mels, 2 * n).T[r2, ::COL_STEP].astype(np.float32)
    out[p + "enc_temp1"] = tr["enc.temp1"].reshape(d, 2 * n).T[r2, ::COL_STEP].astype(np.float32)
    out[p + "enc_layer0_in"] = tr["enc.layer[ 0 ].in"].reshape(n, d)[r1, ::COL_STEP].astype(np.float32)
    out[p + "encode_out"] = tr["encode-out"].reshape(n, d)[r1, ::COL_STEP].astype(np.float32)
    ck, cv = cross_kv(o, n)
    out[p + "cross_k"] = ck[:, r1, ::COL_STEP].astype(np.float16)
    out[p + "cross_v"] = cv[:, r1, ::COL_STEP].astype(np.float16)
    for th, r in runs.items():
        out[p + "t%d_prompt_logits" % th] = logits_sample(r["prompt_logits"])[..., ::LOGIT_THIN]
        out[p + "t%d_tokens" % th] = r["tokens"]
        out[p + "t%d_step_logits" % th] = r["step_logits"][..., ::LOGIT_THIN]
        out[p + "t%d_gap" % th] = r["gap"]


# whisper_full runs: name -> (model, flags, max_tokens, offset_ms, duration_ms, [(language, audio_ctx) per call]); the last call is stored
FULL_SECONDS_USED = 64000
FULL_RUNS = {
    "full_en_750": (FULL_MODEL, 0, 0, 0, FULL_SECONDS_USED, [("en", 750)]),
    "full_en_384_offset_max": (FULL_MODEL, 8 | 2, 24, 10000, 40000, [("en", 384)]),
    "full_ml_de_then_auto": (FULL_MODEL_ML, 0, 0, 0, FULL_SECONDS_USED, [("de", 750), ("auto", 0)]),
}


def run_full(model, pcm, flags, max_tokens, off, dur, calls):
    o = RefOracle(synth.model_path(model), threads=4, log_level=0)
    L = o.L
    o.gap_log(True)
    for lang, actx in calls:
        lg = b"" if lang == "auto" else lang.encode()
        rc = L.ora_full_ex(o.ctx, pcm.ctypes.data_as(C.POINTER(C.c_float)), pcm.size, 4, flags, lg, max_tokens, actx, off, dur)
        assert rc == 0
    gaps = o.gap_log()
    o.gap_log(False)
    segs = []
    for i in range(L.ora_full_n_segments(o.ctx)):
        toks = [L.ora_full_token_id(o.ctx, i, j) for j in range(L.ora_full_n_tokens(o.ctx, i))]
        segs.append((L.ora_full_segment_t0(o.ctx, i), L.ora_full_segment_t1(o.ctx, i), toks))
    return segs, gaps


def make_full(out: dict):
    for name, (model, flags, max_tokens, off, dur, calls) in FULL_RUNS.items():
        for base in range(10, 410, 10):
            pcm = full_pcm(base)
            segs, gaps = run_full(model, pcm, flags, max_tokens, off, dur, calls)
            if gaps.size and gaps.min() >= GAP_SAFE and gaps.size <= 80 * len(calls) * 5:
                break
        else:
            raise RuntimeError("no clean PCM for " + name)
        out[name + "_pcm_base"] = np.int32(base)
        out[name + "_t"] = np.array([[s[0], s[1]] for s in segs], np.int64).reshape(-1, 2)
        out[name + "_ntok"] = np.array([len(s[2]) for s in segs], np.int32)
        out[name + "_tokens"] = np.array([t for s in segs for t in s[2]], np.int32)
        out[name + "_min_gap"] = np.float32(gaps.min())
        print("  %s: pcm base %d, %d segments, %d tokens (%d distinct), %d decoder calls, min gap %.3f" % (
            name, base, len(segs), out[name + "_tokens"].size, len(set(out[name + "_tokens"].tolist())), gaps.size, gaps.min()), flush=True)


def make() -> dict:
    out = {"audio_ctx": np.array(AUDIO_CTX, np.int32), "threads": np.array(THREADS, np.int32), "n_steps": np.int32(N_STEPS),
           "logit_step": np.int32(LOGIT_STEP * LOGIT_THIN), "col_step": np.int32(COL_STEP)}
    for key, (model, chunk0) in MODELS.items():
        o = RefOracle(synth.model_path(model), threads=1)
        out[key + "_prompt"] = np.array(prompt_of(o), np.int32)
        for n in AUDIO_CTX:
            make_case(key, model, chunk0, n, out)
    make_full(out)
    return out


if __name__ == "__main__":
    data = make()
    np.savez_compressed(OUT, **data)
    print("audio_ctx.npz %.0f KB" % (os.path.getsize(OUT) / 1024), flush=True)

#!/usr/bin/env python
"""Generate tests/golden/speed_up.npz from oracle/_ref — the reference's own CPU implementation — for speed-up, the 2x phase-vocoder
log-mel of whisper_pcm_to_mel_phase_vocoder (whisper.cpp:2299-2311; log_mel_spectrogram :2060-2181 with fft_size 800, hop 320,
speed_up = true) that whisper_full_params::speed_up selects (:2776-2786).  Its frames hold twice the audio of the default mel, so one
3000-frame encoder window covers 60 s.

The oracle wrapper (oracle/ref_wrap.cpp) is unchanged: whisper.h does not declare whisper_pcm_to_mel_phase_vocoder, but the function
has external linkage in liboracle_ref.so, so `vocoder_mel` below binds it by its (C++) symbol.

Contents:
- mel only: clips of 0, 319, 320, 799, 800 and 12 345 samples (n_len = n // 320: 0, 0, 1, 2, 2, 38 frames) and a 10 s signal of two
  tones just under 8 kHz (HF_TONES), whose energy lies in the 800-point bins 397-401: the edge of the reference's fold (bin 400 single,
  bin 401 = |X399|^2 left unfolded) reaches the top band of the synthetic filter bank, which weighs averaged bin 200.
- decode cases on micro.en-sc and micro-sc (CLIPS): a 60 s clip, a 45.7 s clip (window zero-padded past frame 2285), a 75 s clip (the
  first 3000 of its 3750 frames) and an 80 s clip encoded from mel offset 1000.  Each stores every 50th mel frame, encode-out and the
  cross-K/V memories (sub-sampled), the prompt and teacher-forced step logits and 40 greedy tokens at reference threads 1, 4 and 16.
  PCM chunk ids are redrawn as make_golden.make() does until every step's top-2 margin is >= GAP_SAFE at all three thread counts.
  Where none of CHUNK_TRIES chunks is clean — the 45.7 s clips, whose window is zero-padded: a random encoder's response to silence
  throws the scripted decoder off its script — the case pins mel, tensors and logits only ("<key>_<clip>_tokens_pinned" = 0).
- one case at audio_ctx = 750 (micro.en-sc, 60 s), set the way make_audio_ctx_golden.py sets it.
- whisper_lang_auto_detect (whisper.cpp:2428-2495) on the vocoder mel of three 60 s clips (micro-sc).
- mel_spread: the largest |oracle - numpy restatement| over every mel this generator computes.  The restatement (log_mel_raw below)
  evaluates the DFT in double, so the spread is the reference's own f32 FFT round-off; the tests' TOL_MEL is derived from it.

    python tests/golden/make_speed_up_golden.py        # rewrites tests/golden/speed_up.npz
"""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden import GAP_SAFE, LOGIT_STEP, MIN_DISTINCT, greedy, logits_sample, prompt_of  # noqa: E402
from whisper_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "speed_up.npz")

F32 = np.float32
HOP, FFT = 320, 800
MEL_LENGTHS = (0, 319, 320, 799, 800, 12345)
HF_TONES = (7950.0, 7990.0)   # Hz; bins of 20 Hz: 397.5 and 399.5
HF_SAMPLES = 160000
MODELS = {"en": ("micro.en-sc", 0), "ml": ("micro-sc", 3)}   # key: (model, first PCM chunk id tried)
CLIPS = {"s60": (960000, 0), "s45": (731200, 0), "s75": (1200000, 0), "off1000": (1280000, 1000)}   # name: (samples, mel offset)
AUDIO_CTX_CASE = ("en", "s60", 750)
LANG_CHUNKS = (3, 5, 8)
THREADS = (1, 4, 16)
N_STEPS = 40
CHUNK_TRIES = 24
MEL_KEEP = 50          # every 50th mel frame of a decode case
ROW_STEP = 25          # every 25th audio position ...
COL_STEP = 8           # ... and every 8th channel of encode-out and cross-K/V
LOGIT_THIN = 8         # logits: every 8th entry of make_golden's sub-sample


# ---------------------------------------------------------------------------------------------------------------------
# numpy restatement of the phase-vocoder log-mel (whisper.cpp:2060-2181 with fft_size 800, fft_step 320, speed_up)
def vocoder_power(pcm, n_len=None):
    """|X[k]|^2 in f32 of the 800-point Hann-windowed frames, k = 0..401, [n_len][402].  The DFT is evaluated in double (pocketfft),
    i.e. exact up to the final f32 rounding of re / im; bin 401 is |X399|^2 (X401 = conj X399 for a real frame)."""
    pcm = np.asarray(pcm, F32)
    if n_len is None:
        n_len = pcm.size // HOP                                          # :2080
    hann = (0.5 * (1.0 - np.cos(2.0 * np.pi * np.arange(FFT) / FFT))).astype(F32)   # :2076
    padded = np.concatenate([pcm, np.zeros(n_len * HOP + FFT, F32)])
    idx = np.arange(n_len)[:, None] * HOP + np.arange(FFT)[None, :]
    frames = hann[None, :] * padded[idx]                                  # f32 product, zero past the end (:2104-2110)
    X = np.fft.rfft(frames.astype(np.float64), axis=1)                    # bins 0..400
    re, im = X.real.astype(F32), X.imag.astype(F32)
    pw = re * re + im * im                                                # :2115-2117
    return np.concatenate([pw, pw[:, FFT // 2 - 1:FFT // 2]], axis=1)


def fold_average(pw, fold_401=False, double_400=False):
    """The reference's fold over bins 1..399 (:2118-2123) and the average of bin pairs onto 201 bins, f32 sum halved in double
    (:2130-2135).  fold_401 / double_400 are the two misreadings of the fold's edge the tests must tell apart."""
    P = pw.copy()
    P[:, 1:FFT // 2] = P[:, 1:FFT // 2] + P[:, 1:FFT // 2]
    if double_400:
        P[:, FFT // 2] = P[:, FFT // 2] + P[:, FFT // 2]
    if fold_401:
        P[:, FFT // 2 + 1] = P[:, FFT // 2 + 1] + P[:, FFT // 2 + 1]
    return (0.5 * (P[:, 0::2] + P[:, 1::2]).astype(np.float64)).astype(F32)   # [n_len][201]


def log_mel_raw(pcm, filters, **misread):
    """log10 mel power before normalisation, [80][n_len]"""
    Pa = fold_average(vocoder_power(pcm), **misread)
    out = np.empty((Pa.shape[0], filters.shape[0]), F32)
    for i in range(0, Pa.shape[0], 512):
        prod = Pa[i:i + 512, None, :] * filters[None, :, :]               # float products (:2142)
        s = np.maximum(prod.astype(np.float64).sum(-1), 1e-10)            # double accumulate, floor (:2139-2147)
        out[i:i + 512] = np.log10(s).astype(F32)
    return out.T.copy()


def log_mel(pcm, filters, **misread):
    """the normalised log-mel: clip-wide maximum - 8 as the floor, (x + 4) / 4 in double (:2155-2177)"""
    mel = log_mel_raw(pcm, filters, **misread)
    if mel.size == 0:
        return mel
    mmax = float(mel.max()) - 8.0
    mel = np.where(mel.astype(np.float64) < mmax, F32(mmax), mel)
    return ((mel.astype(np.float64) + 4.0) / 4.0).astype(F32)


def mel_pcm(n: int):
    """the mel-only clip of n samples: the first n of one synthetic clip"""
    return synth.synth_pcm(0, max(MEL_LENGTHS))[:n]


def hf_pcm():
    i = np.arange(HF_SAMPLES, dtype=np.float64)
    return sum(0.25 * np.sin(2 * np.pi * f * i / 16000.0) for f in HF_TONES).astype(F32)


# ---------------------------------------------------------------------------------------------------------------------
# oracle
def vocoder_mel(o, pcm):
    """whisper_pcm_to_mel_phase_vocoder of the reference on `pcm` into o's context; returns the mel [80][n // 320]"""
    fn = getattr(o.L, "_Z32whisper_pcm_to_mel_phase_vocoderP15whisper_contextPKfii")
    fn.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int, C.c_int]
    fn.restype = C.c_int
    pcm = np.ascontiguousarray(pcm, F32)
    assert fn(o.ctx, pcm.ctypes.data_as(C.POINTER(C.c_float)), pcm.size, o.threads) == 0
    return o.get_mel()


def case_pcm(chunk: int, name: str):
    return synth.synth_pcm(chunk, CLIPS[name][0])


def run_case(model: str, mel, offset: int, th: int, audio_ctx: int = 0):
    from oracle.ref import RefOracle
    from tests.golden.make_audio_ctx_golden import set_audio_ctx
    o = RefOracle(synth.model_path(model), threads=th)
    if audio_ctx:
        set_audio_ctx(o, audio_ctx)
    o.set_mel(mel)
    o.encode(offset)
    return o, greedy(o, prompt_of(o), N_STEPS, keep_logits=True)


def clean(r):
    return float(r["gap"].min()) >= GAP_SAFE and len(set(r["tokens"].tolist())) >= MIN_DISTINCT


def make_case(key: str, name: str, out: dict, spread: list, audio_ctx: int = 0):
    from oracle.ref import RefOracle
    model, chunk0 = MODELS[key]
    offset = CLIPS[name][1]
    first = None
    for chunk in range(chunk0, chunk0 + CHUNK_TRIES):
        o1 = RefOracle(synth.model_path(model), threads=1)
        pcm = case_pcm(chunk, name)
        mel = vocoder_mel(o1, pcm)
        runs = {}
        for th in THREADS:   # 16 spin-waiting reference threads are slow on a small host: only where 1 and 4 are clean
            runs[th] = run_case(model, mel, offset, th, audio_ctx)[1]
            if not clean(runs[th]):
                break
        ok = len(runs) == len(THREADS) and all(clean(r) for r in runs.values())
        print("  %s/%s chunk %d: min gaps %s %s" % (key, name, chunk, [round(float(r["gap"].min()), 3) for r in runs.values()],
                                                  "keep" if ok else "skip"), flush=True)
        if first is None:
            first = (chunk, pcm, mel)
        if ok:
            pinned = True
            break
    else:
        chunk, pcm, mel = first
        runs = {th: run_case(model, mel, offset, th, audio_ctx)[1] for th in THREADS}
        pinned = False
        print("  %s/%s: no clean chunk in %d tries — tensors and logits only" % (key, name, CHUNK_TRIES), flush=True)
    spread.append(float(np.abs(log_mel(pcm, o1_filters(model)) - mel).max()))
    p = "%s_%s_" % (key, name) if not audio_ctx else "%s_%s_n%d_" % (key, name, audio_ctx)
    out[p + "chunk"] = np.int32(chunk)
    out[p + "tokens_pinned"] = np.int32(pinned)
    out[p + "mel_shape"] = np.array(mel.shape, np.int32)
    out[p + "mel"] = mel[:, ::MEL_KEEP].astype(F32)
    o, _ = run_case(model, mel, offset, 1, audio_ctx)
    o.trace(True)
    o.encode(offset)
    tr = o.trace_items()
    o.trace(False)
    n = audio_ctx or o.n_audio_ctx
    d, L = o.n_audio_state, o.n_text_layer
    out[p + "encode_out"] = tr["encode-out"].reshape(n, d)[::ROW_STEP, ::COL_STEP].astype(F32)
    k, v = o.cross_kv()
    k, v = (a.reshape(-1)[: L * n * d].reshape(L, n, d) for a in (k, v))   # n rows per layer, packed (whisper.cpp:1479-1480)
    out[p + "cross_k"] = k[:, ::ROW_STEP, ::COL_STEP].astype(np.float16)
    out[p + "cross_v"] = v[:, ::ROW_STEP, ::COL_STEP].astype(np.float16)
    for th, r in runs.items():
        out[p + "t%d_prompt_logits" % th] = logits_sample(r["prompt_logits"])[..., ::LOGIT_THIN]
        out[p + "t%d_step_logits" % th] = r["step_logits"][..., ::LOGIT_THIN]
        out[p + "t%d_tokens" % th] = r["tokens"]
        out[p + "t%d_gap" % th] = r["gap"]


_filters = {}


def o1_filters(model):
    if model not in _filters:
        from oracle.whisper_np import NpModel
        _filters[model] = NpModel(synth.model_path(model)).filters
    return _filters[model]


def make_mels(out: dict, spread: list):
    from oracle.ref import RefOracle
    o = RefOracle(synth.model_path("micro.en-sc"), threads=4)
    filters = o1_filters("micro.en-sc")
    for n in MEL_LENGTHS:
        pcm = mel_pcm(n)
        mel = vocoder_mel(o, pcm)
        assert mel.shape == (80, n // HOP)
        out["mel_len%d" % n] = mel
        if mel.size:
            spread.append(float(np.abs(log_mel(pcm, filters) - mel).max()))
    mel = vocoder_mel(o, hf_pcm())
    out["mel_hf"] = mel
    spread.append(float(np.abs(log_mel(hf_pcm(), filters) - mel).max()))
    return mel


def make_lang(out: dict):
    from oracle.ref import RefOracle
    o = RefOracle(synth.model_path("micro-sc"), threads=4)
    ids, probs = [], []
    for ch in LANG_CHUNKS:
        vocoder_mel(o, synth.synth_pcm(ch, 960000))
        lid, pr = o.lang_auto_detect(0)
        ids.append(lid); probs.append(pr)
        print("  lang/chunk %d: id %d p %.4f (runner-up %.4f)" % (ch, lid, np.sort(pr)[-1], np.sort(pr)[-2]), flush=True)
    out["lang_chunks"] = np.array(LANG_CHUNKS, np.int32)
    out["lang_id"] = np.array(ids, np.int32)
    out["lang_probs"] = np.array(probs, F32)


def make() -> dict:
    from oracle.ref import RefOracle
    out = {"threads": np.array(THREADS, np.int32), "n_steps": np.int32(N_STEPS), "logit_step": np.int32(LOGIT_STEP * LOGIT_THIN),
           "row_step": np.int32(ROW_STEP), "col_step": np.int32(COL_STEP), "mel_keep": np.int32(MEL_KEEP)}
    spread = []
    hf = make_mels(out, spread)
    # the edge of the fold must be visible in the committed high-frequency mel
    filters = o1_filters("micro.en-sc")
    for kw in ({"fold_401": True}, {"double_400": True}):
        print("  hf misreading %s: max diff %.3g" % (kw, np.abs(log_mel(hf_pcm(), filters, **kw) - hf).max()), flush=True)
    make_lang(out)
    for key, (model, _c) in MODELS.items():
        out[key + "_prompt"] = np.array(prompt_of(RefOracle(synth.model_path(model))), np.int32)
        for name in CLIPS:
            make_case(key, name, out, spread)
    key, name, n = AUDIO_CTX_CASE
    make_case(key, name, out, spread, audio_ctx=n)
    out["mel_spread"] = np.float32(max(spread))
    print("  mel spread (oracle vs numpy, f64 DFT): %.3g" % max(spread), flush=True)
    return out


if __name__ == "__main__":
    data = make()
    np.savez_compressed(OUT, **data)
    print("speed_up.npz %.0f KB" % (os.path.getsize(OUT) / 1024), flush=True)

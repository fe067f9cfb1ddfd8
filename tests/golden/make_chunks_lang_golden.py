#!/usr/bin/env python
"""Generate tests/golden/chunks_lang.npz from oracle/_ref — the reference's own CPU implementation — for the language sentinel of the
batch path (WSP_TOKEN_LANGUAGE_AUTO): every chunk's language detected from its own window, then its greedy decode with that language
in the prompt.

Each chunk runs through the reference on its own: whisper_pcm_to_mel, then whisper_lang_auto_detect at offset 0 (the language id and its 99 probabilities), then make_chunks_eot_golden's greedy loop with the
prompt [sot, sot + 1 + id, transcribe] until EOT or CAP tokens.  The same loop is also run with the other active language in the
prompt; those tokens are stored as "other_tokens".

micro-sc is the multilingual scripted model: after [sot] it chooses between en (id 0) and de (id 2) from the audio
(whisper_b200/synth.py).  A candidate (PCM chunk id, clip length) is kept when, at every thread count of the case, its top-2
language-probability gap is >= LANG_GAP_SAFE (10x the 2e-4 tolerance of the GPU's probabilities, so there is no top tie) and its
decoding margin is >= GAP_SAFE at every step.  A batch must hold both languages and at least one chunk that decodes differently
under the other language's prompt; the generator fails instead of writing a weaker batch.

Cases, each a batch of 4 at 1 and 4 reference threads: one at the full audio context, and one at audio_ctx 750 (set through
whisper_full, make_audio_ctx_golden.set_audio_ctx), where the 15 s window of clips of 240000 samples (16 kHz) is detected as de and
that of zero-padded clips of 185000 samples as en.  There is no speed-up case: the phase-vocoder mels of the clips tried (chunk ids
0-7, 13, 15 and 30 at 500000-960000 samples) come out en or without a clear gap, so no speed-up batch holds both languages.
tests/test_gpu_chunks_lang.py checks speed-up against the GPU's single-clip path instead.

    python tests/golden/make_chunks_lang_golden.py [case ...]   # rewrites tests/golden/chunks_lang.npz (a few minutes)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_chunks_eot_golden import until_eot  # noqa: E402
from tests.golden.make_golden import GAP_SAFE  # noqa: E402
from whisper_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "chunks_lang.npz")

MODEL = "micro-sc"
CAP = 72                                 # max_decode of every case
LANG_TOL = 2e-4                          # the GPU's language probabilities against the reference's
LANG_GAP_SAFE = 10 * LANG_TOL
ACTIVE = (0, 2)                          # en, de: the language tokens the scripted model uses
CHUNK_TRIES = 24
CASES = {
    # name: (reference threads, batch, audio_ctx, first chunk id tried, clip lengths tried per chunk id)
    # at the full audio context only chunk ids 13..15 (mod 16) are detected as en with a clear gap (at 370000 samples)
    "base": ((1, 4), 4, 0, 12, (440000, 370000, 480000, 400000)),
    "actx750": ((1, 4), 4, 750, 0, (240000, 185000)),
}


def lang_gap(probs):
    s = np.sort(probs)
    return float(s[-1] - s[-2])


def run_chunk(o, pcm):
    """o: a RefOracle.  Returns (lang id, lang probs, tokens, gaps, other-language tokens)."""
    o.pcm_to_mel(pcm)
    lid, probs = o.lang_auto_detect(0)
    sot, task = o.special["sot"], o.special["transcribe"]
    toks, gaps = until_eot(o, [sot, sot + 1 + lid, task], CAP)
    other = ACTIVE[1] if lid == ACTIVE[0] else ACTIVE[0]
    otoks, _ = until_eot(o, [sot, sot + 1 + other, task], CAP)
    return lid, probs, toks, gaps, otoks


def clean(r):
    lid, probs, _toks, gaps, _o = r
    return lid in ACTIVE and lang_gap(probs) >= LANG_GAP_SAFE and (gaps.size == 0 or float(gaps.min()) >= GAP_SAFE)


def differs(r):
    return r[2].tolist() != r[4].tolist()


def choose(kept, batch, th):
    """one chunk per language and one that decodes differently under the other language first, the rest in the order found"""
    picked = []
    for want in (lambda r: r[0] == ACTIVE[0], lambda r: r[0] == ACTIVE[1], differs):
        for k in kept:
            if want(k[2][th]) and not any(k is p for p in picked):
                picked.append(k)
                break
    picked += [k for k in kept if not any(k is p for p in picked)][:batch - len(picked)]
    if len(picked) < batch:
        return None
    rs = [k[2][th] for k in picked]
    if {r[0] for r in rs} != set(ACTIVE) or not any(differs(r) for r in rs):
        return None
    return picked


def make_case(name):
    from oracle.ref import RefOracle
    from tests.golden.make_audio_ctx_golden import set_audio_ctx
    threads, batch, audio_ctx, first, lengths = CASES[name]
    oracles = {}
    for th in threads:
        oracles[th] = RefOracle(synth.model_path(MODEL), threads=th)
        if audio_ctx:
            set_audio_ctx(oracles[th], audio_ctx)
    kept, chosen = [], None          # (chunk, n_samples, {th: run})
    for ch in range(first, first + CHUNK_TRIES):
        for n in lengths:
            pcm = synth.synth_pcm(ch, n)
            rs = {th: run_chunk(o, pcm) for th, o in oracles.items()}
            ok = all(clean(r) for r in rs.values()) and len({r[0] for r in rs.values()}) == 1
            r = rs[threads[0]]
            print("  %s chunk %d, %d samples: lang %d (gap %.4f), n_out %d, min gap %.3f, %s, %s" % (
                name, ch, n, r[0], lang_gap(r[1]), r[2].size, float(r[3].min()) if r[3].size else 0.0,
                "differs" if differs(r) else "same", "keep" if ok else "skip"), flush=True)
            if ok:
                kept.append((ch, n, rs))
            chosen = choose(kept, batch, threads[0])
            if chosen:
                break
        if chosen:
            break
    else:
        raise RuntimeError("%s: no batch of %d clean chunks with both languages and a language-dependent decode" % (name, batch))
    sot = oracles[threads[0]].special["sot"]
    out = {name + "_chunks": np.array([c[0] for c in chosen], np.int32),
           name + "_n_samples": np.array([c[1] for c in chosen], np.int32),
           name + "_prompt": np.array([sot, -1, oracles[threads[0]].special["transcribe"]], np.int32),
           name + "_threads": np.array(threads, np.int32), name + "_audio_ctx": np.int32(audio_ctx), name + "_cap": np.int32(CAP)}
    for th in threads:
        pre = "%s_t%d_" % (name, th)
        ids = np.zeros(batch, np.int32)
        probs = np.zeros((batch, chosen[0][2][th][1].size), np.float32)
        toks, otoks = np.full((batch, CAP), -1, np.int32), np.full((batch, CAP), -1, np.int32)
        gaps = np.full((batch, CAP - 1), np.nan, np.float32)
        n_out, o_n_out = np.zeros(batch, np.int32), np.zeros(batch, np.int32)
        for b, (_ch, _n, rs) in enumerate(chosen):
            lid, pr, t, g, ot = rs[th]
            ids[b], probs[b] = lid, pr
            toks[b, :t.size], gaps[b, :g.size], n_out[b] = t, g, t.size
            otoks[b, :ot.size], o_n_out[b] = ot, ot.size
        out[pre + "lang_id"], out[pre + "lang_probs"] = ids, probs
        out[pre + "tokens"], out[pre + "gap"], out[pre + "n_out"] = toks, gaps, n_out
        out[pre + "other_tokens"], out[pre + "other_n_out"] = otoks, o_n_out
    return out


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)       # a subset of the cases is merged into the existing file
    new = {}
    for nm in names:
        new.update(make_case(nm))
    data = dict(np.load(OUT)) if os.path.exists(OUT) and len(names) < len(CASES) else {}
    data.update(new)
    np.savez_compressed(OUT, **data)
    print("chunks_lang %.0f KB" % (os.path.getsize(OUT) / 1024), flush=True)

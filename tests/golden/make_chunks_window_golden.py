#!/usr/bin/env python
"""Generate tests/golden/chunks_window.npz from oracle/_ref — the reference's own CPU implementation — for wsp_run_chunks_window: every
chunk of a batch decoded as whisper_full decodes its first window, then cut into whisper_full's segments.

Per chunk, window() restates whisper_full's window loop (Whisper/source/whisper.cpp:2910-3003) over the reference's whisper_decode,
whisper_sample_timestamp(initial) and whisper_sample_best, at seek 0 over the clip's whole mel, with the prompt of prompt_of();
segments() restates the segment loop (:3026-3119).  Stored per chunk: every sampled token's id, tid, p, pt and ptsum, the window's
result (n_sampled, result_len, seek_delta, failed), its segments (t0, t1, token range, text) and the reference's top-2 logit margin at
every step but the forced first one.  For every window that did not fail, the generator checks that its segments are the first
segments of the reference's own whisper_full on the same clip, with no past prompt: whisper_full emits window 1's segments before
any later window runs, so this ties the restatement to whisper_full itself.

Coverage: the cases' batches together hold windows ended by EOT, by the end of the audio (a clip of just over 1 s, whose first
timestamp already reaches its end), by a timestamp that goes back in time, by max_tokens and under single_segment, a window that
fails at n_max (the scripted models' off-script repetition loops), and a clip under 1 s (no window).  Candidates are (PCM chunk id,
clip length) pairs in a fixed order; one is kept when it adds a kind its case still lacks (or, once it lacks none, to fill the batch
with windows of more than one token from chunk ids not kept yet) and its margin is >= GAP_SAFE at every step at every thread count
of its case.  The generator fails instead of writing a batch that lacks a kind.  The oracle's whisper_full has no speed-up switch, so no speed-up batch is pinned;
tests/test_gpu_chunks_window.py checks speed-up against the GPU's own run without it, including a window that ends at the end of a
phase-vocoder mel.

    python tests/golden/make_chunks_window_golden.py [case ...]   # rewrites tests/golden/chunks_window.npz
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden import GAP_SAFE, prompt_of, top2_gap  # noqa: E402
from whisper_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "chunks_window.npz")

SHORT = 12000                     # samples of the clip under 1 s (75 frames: no window)
# 16160 samples = 101 frames: the window ends at its first timestamp, which already reaches the end of the audio (seek_delta + 100 >= 101)
LENGTHS = (16160, 480000, 160000, 440000, 240000, 420000, 320000, 400000, 200000, 360000, 120000, 280000, 460000)
CHUNK_TRIES = 16
CASES = {
    # name: (model, reference threads, batch, max_tokens, single_segment, kinds the batch must hold)
    "micro_en": ("micro.en-sc", (1, 4), 5, 0, 0, ("eot", "audio_end", "back_in_time", "n_max", "short")),
    "micro_ml": ("micro-sc", (1, 4), 4, 12, 1, ("max_tokens", "single_segment", "short")),
}
MAX_SEGS = 16


def n_max_of(o):
    return o.n_text_ctx // 2 - 4


def rule(ids, eot, beg, max_tokens, single_segment, n_max, seek, seek_end):
    """whisper.cpp:2926-3003 over a token sequence from step 0: (result dict, kind of end, tokens consumed).  The result holds
    has_ts, seek_delta, result_len, failed; kind is one of eot, audio_end, max_tokens, back_in_time, n_max, or None (not ended)."""
    has_ts, seek_delta, result_len = False, 100 * 30, 0

    def out(failed, kind, i):
        return dict(has_ts=int(has_ts), seek_delta=seek_delta, result_len=result_len, failed=int(failed)), kind, i + 1

    for i, tid in enumerate(ids):
        if tid > beg:
            new = 2 * (tid - beg)
            if has_ts and seek_delta > new and result_len < i:
                return out(False, "back_in_time", i)
            seek_delta, result_len, has_ts = new, i + 1, True
        if tid == eot or (max_tokens > 0 and i >= max_tokens) or (has_ts and seek + seek_delta + 100 >= seek_end):
            kind = "eot" if tid == eot else "max_tokens" if max_tokens > 0 and i >= max_tokens else "audio_end"
            if result_len == 0:
                if seek + seek_delta + 100 >= seek_end:
                    result_len = i + 1
                else:
                    return out(True, kind, i)
            if single_segment:
                result_len, seek_delta = i + 1, 100 * 30
            return out(False, kind, i)
        if i == n_max - 1:
            return out(result_len == 0 or seek_delta < 100 * 30 // 2, "n_max", i)
    return dict(has_ts=int(has_ts), seek_delta=seek_delta, result_len=result_len, failed=0), None, len(ids)


def segments(tokens, result, seek, eot, beg, text_of, single_segment=False, print_special=False, speed_up=False):
    """whisper.cpp:3026-3119: tokens = list of dicts with id and tid; result = dict with n_tokens, seek_delta, failed"""
    if result["failed"] or result["n_tokens"] == 0:
        return []
    cur = tokens[:result["n_tokens"]]
    sc = 2 if speed_up else 1
    segs, i0, t0, text, i = [], 0, seek + 2 * (cur[0]["tid"] - beg), "", 0
    while i < len(cur):
        tid = cur[i]["id"]
        if print_special or tid < eot:
            text += text_of(tid)
        if tid > beg and not single_segment:
            t1 = seek + 2 * (cur[i]["tid"] - beg)
            if text:
                segs.append(dict(t0=sc * t0, t1=sc * t1, i0=i0, i1=i + 1, text=text))
            text = ""
            while i < len(cur) and cur[i]["id"] > beg:
                i += 1
            i -= 1
            t0, i0 = t1, i + 1
        i += 1
    if text:
        segs.append(dict(t0=sc * t0, t1=sc * (seek + result["seek_delta"]), i0=i0, i1=len(cur), text=text))
    return segs


def window(o, prompt, n_samples, max_tokens, single_segment):
    """o: a RefOracle with the chunk's mel set and encoded.  Returns (tokens, result, kind, gaps)."""
    eot, beg, n_max = o.special["eot"], o.special["beg"], n_max_of(o)
    seek_end = o.L.ora_mel_len(o.ctx)
    if seek_end <= 100:                                                   # whisper.cpp:2871
        return [], dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0), "short", []
    o.decode(prompt, 0)
    toks, gaps = [o.sample(initial=True, force_timestamp=True)], []
    while True:
        r, kind, used = rule([t["id"] for t in toks], eot, beg, max_tokens, single_segment, n_max, 0, seek_end)
        if kind is not None:
            break
        lg, _ = o.decode([toks[-1]["id"]], len(prompt) + len(toks) - 1)
        gaps.append(top2_gap(lg[0]))
        toks.append(o.sample())
    assert used == len(toks)
    if single_segment and not r["failed"] and kind != "back_in_time":
        kind = (kind, "single_segment")
    res = dict(n_sampled=len(toks), n_tokens=r["result_len"], seek_delta=r["seek_delta"], failed=r["failed"])
    return toks, res, kind, gaps


def kinds_of(kind):
    return set(kind) if isinstance(kind, tuple) else {kind}


def full_check(o, pcm, toks, segs, max_tokens, single_segment, language):
    """the window's segments must be the first segments of the reference's whisper_full on the same clip, no past prompt"""
    o.clear_prompt_past()
    rc, full = o.full(pcm, flags=2 | (4 if single_segment else 0), language=language, max_tokens=max_tokens)
    assert rc == 0
    got = [(s["t0"], s["t1"], s["text"], [t["id"] for t in toks[s["i0"]:s["i1"]]]) for s in segs]
    want = [(f["t0"], f["t1"], f["text"], f["tokens"]) for f in full[:len(segs)]]
    assert got == want, (got, want)


def make_case(name):
    from oracle.ref import RefOracle
    from whisper_b200 import capi
    model, threads, batch, max_tokens, single, need = CASES[name]
    path = synth.model_path(model)
    vocab = capi.Model(path)
    oracles = {th: RefOracle(path, threads=th) for th in threads}
    o0 = oracles[threads[0]]
    eot, beg, prompt = o0.special["eot"], o0.special["beg"], prompt_of(o0)
    text_of = lambda i: vocab.token_text(i) or ""
    kept = []        # (chunk, n_samples, kinds, {th: (tokens, result, segments, gaps)})

    def run(ch, n):
        pcm = synth.synth_pcm(ch, n)
        mel = o0.pcm_to_mel(pcm)
        rs, kinds = {}, set()
        for th, o in oracles.items():
            o.set_mel(mel)
            o.encode(0)
            toks, res, kind, gaps = window(o, prompt, n, max_tokens, single)
            segs = segments(toks, res, 0, eot, beg, text_of, single_segment=bool(single))
            rs[th] = (toks, res, segs, gaps)
            kinds |= kinds_of(kind)
        gap = min([min(g) for _t, _r, _s, g in rs.values() if g] or [np.inf])
        return rs, kinds, gap

    def covered():
        return set().union(*[k[2] for k in kept]) & set(need)

    rs, kinds, _gap = run(0, SHORT)
    kept.append((0, SHORT, kinds, rs))
    for ch in range(CHUNK_TRIES):
        for n in LENGTHS:
            if covered() == set(need) and len(kept) >= batch:
                break
            rs, kinds, gap = run(ch, n)
            fill = (covered() == set(need) and ch not in [k[0] for k in kept if k[1] != SHORT]
                    and rs[threads[0]][1]["n_sampled"] > 1)
            take = gap >= GAP_SAFE and (bool(kinds & set(need) - covered()) or fill)
            print("  %s chunk %d, %d samples: %s, n_sampled %d, min gap %.3f %s" % (
                name, ch, n, sorted(kinds), rs[threads[0]][1]["n_sampled"], gap, "keep" if take else "skip"), flush=True)
            if take:
                pcm = synth.synth_pcm(ch, n)
                for th, o in oracles.items():
                    toks, res, segs, _g = rs[th]
                    if not res["failed"]:
                        full_check(o, pcm, toks, segs, max_tokens, single, "en")
                kept.append((ch, n, kinds, rs))
    have = set().union(*[k[2] for k in kept])
    if not set(need) <= have or len(kept) < batch:
        raise RuntimeError("%s: batch lacks %s" % (name, sorted(set(need) - have)))
    kept = kept[:batch]
    out = {name + "_chunks": np.array([k[0] for k in kept], np.int32),
           name + "_n_samples": np.array([k[1] for k in kept], np.int32),
           name + "_prompt": np.array(prompt, np.int32), name + "_threads": np.array(threads, np.int32),
           name + "_params": np.array([max_tokens, single], np.int32),
           name + "_kinds": np.array([",".join(sorted(k[2])) for k in kept])}
    nm = n_max_of(o0)
    for th in threads:
        tok = np.full((batch, nm, 2), -1, np.int32)             # id, tid
        prob = np.full((batch, nm, 3), np.nan, np.float32)      # p, pt, ptsum
        gaps = np.full((batch, nm), np.nan, np.float32)
        res = np.zeros((batch, 4), np.int32)                    # n_sampled, n_tokens, seek_delta, failed
        segs = np.full((batch, MAX_SEGS, 4), -1, np.int64)      # t0, t1, i0, i1
        texts = np.full((batch, MAX_SEGS), "", dtype=object)
        for b, (_ch, _n, _k, rs) in enumerate(kept):
            toks, r, sg, g = rs[th]
            for i, t in enumerate(toks):
                tok[b, i] = (t["id"], t["tid"])
                prob[b, i] = (t["p"], t["pt"], t["ptsum"])
            gaps[b, :len(g)] = g
            res[b] = (r["n_sampled"], r["n_tokens"], r["seek_delta"], r["failed"])
            assert len(sg) <= MAX_SEGS
            for j, s in enumerate(sg):
                segs[b, j] = (s["t0"], s["t1"], s["i0"], s["i1"])
                texts[b, j] = s["text"]
        pre = "%s_t%d_" % (name, th)
        out[pre + "tokens"], out[pre + "probs"], out[pre + "gap"], out[pre + "result"] = tok, prob, gaps, res
        out[pre + "segments"], out[pre + "texts"] = segs, texts.astype(str)
    return out


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)       # a subset of the cases is merged into the existing file
    new = {}
    for nm in names:
        new.update(make_case(nm))
    data = dict(np.load(OUT)) if os.path.exists(OUT) and len(names) < len(CASES) else {}
    data.update(new)
    np.savez_compressed(OUT, **data)
    print("chunks_window %.0f KB" % (os.path.getsize(OUT) / 1024), flush=True)

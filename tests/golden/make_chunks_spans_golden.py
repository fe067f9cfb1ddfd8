#!/usr/bin/env python
"""Generate tests/golden/chunks_spans.npz from oracle/_ref — the reference's own CPU implementation — for wsp_run_spans_window: every
row of a batch decoded as the first window of whisper_full( clip of its source, offset_ms, duration_ms ).

A case holds a few source clips (slots; each a concatenation of synth_pcm pieces) and a batch of spans (slot, offset_ms, duration_ms).
Per span, span_window() restates whisper_full's window loop (Whisper/source/whisper.cpp:2810-2818, 2910-3003) at seek_start =
offset_ms / 10 and seek_end = seek_start + (duration_ms == 0 ? n_len : duration_ms / 10) over the reference's whisper_encode at
seek_start on the source's whole-clip log-mel, its whisper_decode and its samplers, with make_chunks_window_golden's rule(); segments
come from its segments() at that seek, so they are absolute in the clip.  With the language sentinel in the prompt each row's
language is whisper_lang_auto_detect( offset_ms ).  Every row's token times (max_len 0 and 12) are restated over the source's whole
signal energy from t_beg = t_last = 0 (make_chunks_token_ts_golden).  For every window that did not fail the generator checks that
its segments, token times included, are the first segments of the reference's own whisper_full( offset_ms, duration_ms ) with
token_timestamps on, in the row's language, on the whole clip: that ties the restatement to whisper_full itself.

A candidate span is kept only if, at every thread count, every decoding margin is >= GAP_SAFE, every result token's pt and ptsum lie
more than P_TOL from their thresholds, no segment takes the branch in which the reference reads past a segment's end and, with the
sentinel, the top-2 language-probability gap is >= LANG_GAP_SAFE.  Each of a case's NEEDS lists candidates in order; the first that
clears the margins and shows the kind is kept, and the generator fails instead of writing a case that lacks one.

Two kinds the spans cannot have as first worded:
  - an offset within 1 s of the clip's end runs a window: seek_end counts n_len frames from the offset (:2811), not to the clip's
    end, so only a short duration (short_span) or a negative one gives no window there;
  - the sentinel cannot sit on a row whose offset is at or past the clip's end (whisper_lang_auto_detect's -2), so the window over
    zero frames (past_end) is pinned in the case without the sentinel.

    python tests/golden/make_chunks_spans_golden.py [case ...]   # rewrites tests/golden/chunks_spans.npz
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden import make_chunks_token_ts_golden as mkt  # noqa: E402
from tests.golden.make_chunks_window_golden import rule, segments  # noqa: E402
from tests.golden.make_golden import GAP_SAFE, top2_gap  # noqa: E402
from whisper_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "chunks_spans.npz")

P_TOL = mkt.P_TOL
LANG_GAP_SAFE = 2e-3                    # 10x the GPU's language-probability tolerance
MAX_LENS = (0, 12)
MAX_SEGS = 48
# kinds a case keeps only when a candidate clears the margins (the scripted models are calibrated on 30 s synthetic clips, not on
# windows cut out of longer ones): over the zeros past a clip's end they loop with top-2 margins below GAP_SAFE; every clean window
# of micro.en-sc tried at a non-zero offset opens with beg; micro-sc's windows at odd offsets tried fall below the margins
OPTIONAL = ("near_end", "past_end", "nonbeg_first", "odd_offset")
# cases whose token times are pinned: the scripted multilingual model's max_tokens windows hold tokens whose pt lies within P_TOL of
# thold_pt, where the GPU's probabilities could flip the reference's decision, so micro_ml pins windows, segments and languages only
TOKEN_TIMES = {"micro_en": True, "micro_ml": False}
LANG_CODE = {0: "en", 2: "de"}          # the scripted multilingual model's two active languages

# NEEDS: kind -> candidate spans (slot, offset_ms, duration_ms) tried in order.  Kinds:
#   zero_span      { slot, 0, 0 }
#   past_30s       a window at an offset past 30 s of a source longer than 30 s
#   odd_offset     a window at an offset that is not a multiple of 10 ms
#   audio_end      a window with duration_ms > 0 ended by the end-of-audio rule (before its EOT)
#   short_span     0 < duration_ms < 1 s: no window
#   neg_duration   duration_ms < 0: no window
#   near_end       an offset within 1 s of the clip's end (a window over its last frames and the zeros after)
#   past_end       an offset past the clip's end with duration 0: a window over zero frames
#   nonbeg_first   a window at a non-zero offset whose first segment does not open with beg (token times read energy before it)
#   lang_diff      two rows of one slot detected as different languages
#   max_tokens     a window ended by max_tokens
CASES = {
    # name: (model, reference threads, sentinel, max_tokens, single_segment, sources, needs, shared slot)
    "micro_en": ("micro.en-sc", (1, 4), False, 0, 0,
                 [[(1, 480000), (2, 320000), (3, 420000)], [(5, 480000)], [(0, 440000)]],
                 {"zero_span": [(0, 0, 0), (2, 0, 0)],
                  "past_30s": [(0, 30000, 0), (0, 50000, 0), (0, 31000, 0), (0, 36000, 0), (0, 42000, 0), (0, 48000, 0)],
                  "odd_offset": [(0, 12345, 0), (0, 30007, 0), (2, 3333, 0), (0, 50003, 0), (0, 7771, 0)],
                  "audio_end": [(0, 5000, 6000), (0, 10000, 4000), (2, 0, 5000), (0, 45000, 8000), (2, 4000, 9000), (0, 2000, 3000)],
                  "short_span": [(0, 7000, 800)],
                  "neg_duration": [(0, 1000, -500)],
                  "near_end": [(2, 27000, 0), (2, 26800, 0), (0, 75300, 0), (0, 75100, 0), (2, 26500, 0)],
                  "past_end": [(2, 30000, 0), (2, 27500, 0), (0, 77000, 0), (0, 76250, 0), (0, 90000, 0)],
                  "nonbeg_first": [(0, t, 0) for t in range(500, 76000, 1500)] + [(2, t, 0) for t in range(1000, 27000, 1000)]},
                 0),
    "micro_ml": ("micro-sc", (1, 4), True, 12, 1,
                 [[(13, 370000), (6, 480000)], [(5, 480000)], [(14, 370000)]],
                 {"zero_span": [(2, 0, 0), (0, 0, 0)],
                  "past_30s": [(0, t, 0) for t in range(30000, 52000, 1500)],
                  "odd_offset": [(2, 3333, 0), (0, 4321, 0), (0, 26007, 0), (2, 1234, 0), (0, 33333, 0)],
                  "lang_diff": [(0, t, 0) for t in range(0, 52000, 2000)],
                  "max_tokens": [(2, 0, 0), (0, 0, 0), (2, 5000, 0), (2, 10000, 0)] + [(0, t, 0) for t in range(1000, 52000, 3000)],
                  "short_span": [(2, 7000, 800), (0, 3000, 900)],
                  "near_end": [(2, 22600, 0), (2, 22400, 0)]},
                 0),
}


def c_div(a, b):
    """C's integer division (truncates toward zero)"""
    q = abs(a) // b
    return q if a >= 0 else -q


def source_pcm(pieces):
    return np.concatenate([synth.synth_pcm(ch, n) for ch, n in pieces]).astype(np.float32)


def bounds(offset_ms, duration_ms, n_len):
    """whisper.cpp:2810-2811"""
    seek = c_div(offset_ms, 10)
    return seek, seek + (n_len if duration_ms == 0 else c_div(duration_ms, 10))


def span_window(o, prompt, seek, seek_end, max_tokens, single_segment):
    """o: a RefOracle encoded at seek.  Returns (tokens, result, kind, gaps); kind "no_window" for seek_end <= seek + 100."""
    eot, beg, n_max = o.special["eot"], o.special["beg"], o.n_text_ctx // 2 - 4
    if seek_end <= seek + 100:                                           # whisper.cpp:2816, 2871
        return [], dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0), "no_window", []
    o.decode(prompt, 0)
    toks, gaps = [o.sample(initial=True, force_timestamp=True)], []
    while True:
        r, kind, used = rule([t["id"] for t in toks], eot, beg, max_tokens, single_segment, n_max, seek, seek_end)
        if kind is not None:
            break
        lg, _ = o.decode([toks[-1]["id"]], len(prompt) + len(toks) - 1)
        gaps.append(top2_gap(lg[0]))
        toks.append(o.sample())
    assert used == len(toks)
    return toks, dict(n_sampled=len(toks), n_tokens=r["result_len"], seek_delta=r["seek_delta"], failed=r["failed"]), kind, gaps


def span_token_times(tokens, result, seek, eot, beg, bytes_of, energy, max_len, single_segment, hit):
    """what wsp_window_token_times returns for a row at `seek`: (segments after wrapping, times[n_tokens] as [t0, t1, vlen])"""
    segs = segments(tokens, result, seek, eot, beg, lambda i: bytes_of(i).decode(errors="replace"), single_segment=single_segment)
    n = 0 if result["failed"] else result["n_tokens"]
    times = [[-1, -1, 0.0] for _ in range(result["n_tokens"])]
    vlen = [mkt.voice_length(bytes_of(t["id"])) for t in tokens[:n]]
    state, out = [0, 0, 0], []
    for s in segs:
        sub = times[s["i0"]:s["i1"]]
        mkt.token_times(tokens[s["i0"]:s["i1"]], vlen[s["i0"]:s["i1"]], sub, s["t0"], s["t1"], beg, eot, energy, mkt.THOLD_PT,
                        mkt.THOLD_PTSUM, state, hit)
        if max_len > 0:
            out += mkt.wrap([t["id"] for t in tokens], times, bytes_of, s["i0"], s["i1"], s["t0"], s["t1"], eot, max_len)
        else:
            out.append(s)
    return out, times


def full_segments(o, pcm, language, max_tokens, single_segment, offset_ms, duration_ms, max_len):
    """the reference's whisper_full( offset_ms, duration_ms ) with token timestamps: [dict(t0, t1, text, ids, times)]"""
    import ctypes as C
    o.clear_prompt_past()
    L = o.L
    rc = L.ora_full_ex2(o.ctx, pcm.ctypes.data_as(C.POINTER(C.c_float)), pcm.size, o.threads, 2 | 0x100 | (4 if single_segment else 0),
                        language.encode(), max_tokens, offset_ms, duration_ms, max_len)
    assert rc == 0, rc
    out = []
    for i in range(L.ora_full_n_segments(o.ctx)):
        nt = L.ora_full_n_tokens(o.ctx, i)
        out.append(dict(t0=L.ora_full_segment_t0(o.ctx, i), t1=L.ora_full_segment_t1(o.ctx, i),
                        text=L.ora_full_segment_text(o.ctx, i).decode(errors="replace"),
                        ids=[L.ora_full_token_id(o.ctx, i, j) for j in range(nt)],
                        times=[[L.ora_full_token_t0(o.ctx, i, j), L.ora_full_token_t1(o.ctx, i, j), float(L.ora_full_token_vlen(o.ctx, i, j))]
                               for j in range(nt)]))
    return out


def check_against_full(o, pcm, language, max_tokens, single_segment, span, toks, segs, times, max_len):
    full = full_segments(o, pcm, language, max_tokens, single_segment, span[1], span[2], max_len)
    assert len(full) >= len(segs), (span, len(full), len(segs))
    for s, f in zip(segs, full):
        assert (s["t0"], s["t1"], s["text"]) == (f["t0"], f["t1"], f["text"]), (span, s, f)
        assert [t["id"] for t in toks[s["i0"]:s["i1"]]] == f["ids"], (span, s, f)
        for i, ft in zip(range(s["i0"], s["i1"]), f["times"]):
            assert times[i][0] == ft[0] and times[i][1] == ft[1] and np.float32(times[i][2]) == np.float32(ft[2]), (span, i, times[i], ft)


def lang_gap(probs):
    s = np.sort(probs)
    return float(s[-1] - s[-2])


def make_case(name):
    from oracle.ref import RefOracle
    from whisper_b200 import capi
    model, threads, sentinel, max_tokens, single, sources, needs, _shared = CASES[name]
    path = synth.model_path(model)
    vocab = capi.Model(path)
    oracles = {th: RefOracle(path, threads=th, log_level=0) for th in threads}
    o0 = oracles[threads[0]]
    eot, beg, sot = o0.special["eot"], o0.special["beg"], o0.special["sot"]
    bytes_of = lambda i: vocab.L.wsp_model_token_text(vocab.h, i) or b""
    text_of = lambda i: bytes_of(i).decode(errors="replace")
    pcms = [source_pcm(p) for p in sources]
    mels = [o0.pcm_to_mel(p) for p in pcms]
    energies = [mkt.signal_energy(p) for p in pcms]
    if sentinel:
        prompt_tpl = [sot, -1, o0.special["transcribe"]]
    else:
        prompt_tpl = [sot] + ([sot + 1, o0.special["transcribe"]] if o0.n_vocab == 51865 else [])
    cache = {}

    def run(span):
        """{th: row} for one span, its kinds and whether it clears every margin"""
        if span in cache:
            return cache[span]
        slot, off, dur = span
        n_len = mels[slot].shape[1]
        seek, seek_end = bounds(off, dur, n_len)
        rs, kinds, ok = {}, set(), True
        for th, o in oracles.items():
            o.set_mel(mels[slot])
            lid, lprobs = -1, None
            prompt = list(prompt_tpl)
            if sentinel:
                lid, lprobs = o.lang_auto_detect(off)
                assert lid >= 0, (span, lid)
                ok &= lid in LANG_CODE and lang_gap(lprobs) >= LANG_GAP_SAFE
                prompt[1] = sot + 1 + lid
            else:
                o.encode(seek)
            toks, res, kind, gaps = span_window(o, prompt, seek, seek_end, max_tokens, single)
            hit = set()
            tt = {ml: span_token_times(toks, res, seek, eot, beg, bytes_of, energies[slot], ml, bool(single), hit) for ml in MAX_LENS}
            segs = segments(toks, res, seek, eot, beg, text_of, single_segment=bool(single))
            ok &= (min(gaps) if gaps else np.inf) >= GAP_SAFE
            if TOKEN_TIMES[name]:
                ok &= mkt.p_clear(toks, res["n_tokens"]) and "read_past_end" not in hit
            rs[th] = dict(tokens=toks, result=res, kind=kind, gaps=gaps, segments=segs, times=tt, lang=lid)
            kinds.add(kind)
        r = rs[threads[0]]
        ran = r["kind"] != "no_window"
        if off == 0 and dur == 0:
            kinds.add("zero_span")
        if ran and off >= 30000 and pcms[slot].size > 480000:
            kinds.add("past_30s")
        if ran and off % 10:
            kinds.add("odd_offset")
        if dur <= 0:
            kinds.discard("audio_end")
        if 0 < dur < 1000 and not ran:
            kinds.add("short_span")
        if dur < 0 and not ran:
            kinds.add("neg_duration")
        clip_ms = pcms[slot].size // 16
        if ran and clip_ms - 1000 < off < clip_ms:
            kinds.add("near_end")
        if ran and seek >= n_len and dur == 0:
            kinds.add("past_end")
        if ran and off > 0 and not r["result"]["failed"] and r["result"]["n_tokens"] > 1 and r["tokens"][0]["id"] != beg:
            kinds.add("nonbeg_first")
        if "max_tokens" in kinds and r["result"]["failed"]:
            kinds.discard("max_tokens")
        print("  %s span %s: seek %d..%d, %s, n_sampled %d, lang %d, min gap %.3f %s" % (
            name, span, seek, seek_end, sorted(kinds), r["result"]["n_sampled"], r["lang"],
            min([min(x["gaps"]) for x in rs.values() if x["gaps"]] or [np.inf]), "ok" if ok else "margin"), flush=True)
        cache[span] = (rs, kinds, ok)
        return cache[span]

    kept = []
    for kind, cands in needs.items():
        if kind == "lang_diff":
            continue
        for span in cands:
            rs, kinds, ok = run(span)
            if ok and kind in kinds:
                if span not in kept:
                    kept.append(span)
                break
        else:
            if kind not in OPTIONAL:
                raise RuntimeError("%s: no candidate for %s" % (name, kind))
            print("  %s: no candidate for %s clears the margins" % (name, kind), flush=True)
    if "lang_diff" in needs:
        langs = {}
        for span in kept + needs["lang_diff"]:
            rs, _k, ok = run(span)
            if ok and span[0] == 0:
                langs.setdefault(rs[threads[0]]["lang"], span)
        if len(langs) < 2:
            raise RuntimeError("%s: no two rows of slot 0 detected differently" % name)
        for span in langs.values():
            if span not in kept:
                kept.append(span)
    # several rows on one slot, and a slot no row names
    named = {s[0] for s in kept}
    assert sum(1 for s in kept if s[0] == 0) >= 2 and 1 not in named, kept
    for span in kept:
        rs, _k, _ok = run(span)
        slot, off, dur = span
        for th, o in oracles.items():
            r = rs[th]
            if r["kind"] == "no_window" or r["result"]["failed"]:
                continue
            lang = LANG_CODE[r["lang"]] if sentinel else "en"
            for ml in MAX_LENS if TOKEN_TIMES[name] else (0,):
                segs, times = r["times"][ml]
                check_against_full(o, pcms[slot], lang, max_tokens, single, span, r["tokens"], segs, times, ml)
    B = len(kept)
    nm = o0.n_text_ctx // 2 - 4
    maxp = max(len(p) for p in sources)
    src = np.full((len(sources), maxp, 2), -1, np.int32)
    for i, p in enumerate(sources):
        src[i, :len(p)] = p
    out = {name + "_sources": src, name + "_spans": np.array(kept, np.int32), name + "_prompt": np.array(prompt_tpl, np.int32),
           name + "_threads": np.array(threads, np.int32), name + "_params": np.array([max_tokens, single], np.int32),
           name + "_kinds": np.array([",".join(sorted(run(s)[1])) for s in kept])}
    for th in threads:
        tok = np.full((B, nm, 2), -1, np.int32)
        prob = np.full((B, nm, 3), np.nan, np.float32)
        gaps = np.full((B, nm), np.nan, np.float32)
        res = np.zeros((B, 4), np.int32)
        segs = np.full((B, MAX_SEGS, 4), -1, np.int64)
        texts = np.full((B, MAX_SEGS), "", dtype=object)
        lang = np.full(B, -1, np.int32)
        for b, span in enumerate(kept):
            r = run(span)[0][th]
            for i, t in enumerate(r["tokens"]):
                tok[b, i] = (t["id"], t["tid"])
                prob[b, i] = (t["p"], t["pt"], t["ptsum"])
            gaps[b, :len(r["gaps"])] = r["gaps"]
            rr = r["result"]
            res[b] = (rr["n_sampled"], rr["n_tokens"], rr["seek_delta"], rr["failed"])
            for j, s in enumerate(r["segments"]):
                segs[b, j] = (s["t0"], s["t1"], s["i0"], s["i1"])
                texts[b, j] = s["text"]
            lang[b] = r["lang"]
        pre = "%s_t%d_" % (name, th)
        out[pre + "tokens"], out[pre + "probs"], out[pre + "gap"], out[pre + "result"] = tok, prob, gaps, res
        out[pre + "segments"], out[pre + "texts"], out[pre + "lang"] = segs, texts.astype(str), lang
        for ml in MAX_LENS if TOKEN_TIMES[name] else ():
            tsegs = np.full((B, MAX_SEGS, 4), -1, np.int64)
            ttexts = np.full((B, MAX_SEGS), "", dtype=object)
            times = np.full((B, nm, 2), -1, np.int64)
            vlen = np.zeros((B, nm), np.float32)
            for b, span in enumerate(kept):
                sg, tt = run(span)[0][th]["times"][ml]
                assert len(sg) <= MAX_SEGS
                for j, s in enumerate(sg):
                    tsegs[b, j] = (s["t0"], s["t1"], s["i0"], s["i1"])
                    ttexts[b, j] = s["text"]
                for i, t in enumerate(tt):
                    times[b, i] = (t[0], t[1])
                    vlen[b, i] = t[2]
            p = "%sml%d_" % (pre, ml)
            out[p + "segments"], out[p + "texts"], out[p + "times"], out[p + "vlen"] = tsegs, ttexts.astype(str), times, vlen
    return out


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)       # a subset of the cases is merged into the existing file
    new = {}
    for nm in names:
        new.update(make_case(nm))
    data = dict(np.load(OUT)) if os.path.exists(OUT) and len(names) < len(CASES) else {}
    data.update(new)
    np.savez_compressed(OUT, **data)
    print("chunks_spans %.0f KB" % (os.path.getsize(OUT) / 1024), flush=True)

#!/usr/bin/env python
"""Generate tests/golden/chunks_token_ts.npz from oracle/_ref — the reference's own CPU implementation — for wsp_window_token_times:
every chunk of a batch decoded as whisper_full's first window, cut into segments, given whisper_full's token-level timestamps
(token_timestamps, whisper.cpp:3374-3600) and wrapped at max_len characters (:2713-2763).

Per chunk, make_chunks_window_golden.window() decodes the first window over the reference's decode and samplers; then the reference's
own whisper_full (flag 0x100 = token_timestamps, with max_len) runs on the same clip, and its first segments — those whose tokens
together are window 1's segment tokens, in order — are stored: their t0, t1, text, token range, and every token's t0, t1 and vlen.
The restatement below (signal_energy, token_times, wrap, window_token_times) must give exactly the same, which ties it to
whisper_full itself; the CPU tests then hold the library's csrc/token_times.h to it.

A candidate (PCM chunk id, clip length) is kept only if, at every thread count of its case, every decoding margin is >= GAP_SAFE,
every result token's pt and ptsum lie more than P_TOL (the GPU's probability tolerance) from their thresholds, so that the
`pt > thold_pt && ptsum > thold_ptsum` decision cannot flip, and no segment ends in a text token whose energy at s1 exceeds the
token's threshold (the branch in which the reference reads past the segment's end).  Each case's batch must cover every branch of
the heuristics (BRANCHES), or the generator fails.  One branch is left out: a token end moved later.  Inside a segment a token's
end already equals the next token's start, which caps any later end, so a later end happens only at a segment's last text token —
the branch excluded above; tests/test_token_times.py reaches it on crafted segments.  The oracle's whisper_full has no speed-up
switch, so no speed-up case is pinned.

    python tests/golden/make_chunks_token_ts_golden.py [case ...]   # rewrites tests/golden/chunks_token_ts.npz
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden import make_chunks_window_golden as mkw  # noqa: E402
from tests.golden.make_golden import GAP_SAFE, prompt_of  # noqa: E402
from whisper_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "chunks_token_ts.npz")

THOLD_PT, THOLD_PTSUM = 0.01, 0.01      # whisper_full_default_params
P_TOL = 5e-3
MAX_LENS = (0, 12)
SHORT = 12000                           # a clip under 1 s: no window
LENGTHS = (480000, 160000, 440000, 240000, 420000, 320000, 400000, 200000, 360000, 120000, 280000, 460000)
CHUNK_TRIES = 24
CASES = {
    # name: (model, reference threads, batch)
    "micro_en": ("micro.en-sc", (1, 4), 6),
    "micro_ml": ("micro-sc", (1, 4), 6),
}
# what each batch must reach: the first token of a segment is beg; a gap split by voice length; a token start moved earlier / later
# by the energy; a token end moved earlier; at max_len 12 a segment that is split; a failed window; a clip under 1 s
BRANCHES = ("beg", "vlen_split", "t0_earlier", "t0_later", "t1_earlier", "wrap_split", "failed", "short")
MAX_SEGS = 48


# ---- restatement of the reference ---------------------------------------------------------------------------------------------
def signal_energy(pcm):
    """get_signal_energy (whisper.cpp:3356-3372) with hw = 32: the 65 shifted |x| arrays added in order in f32, then / 65"""
    x = np.abs(np.asarray(pcm, np.float32))
    n = x.size
    acc = np.zeros(n, np.float32)
    for j in range(-32, 33):
        sh = np.zeros(n, np.float32)
        lo, hi = max(0, -j), min(n, n - j)               # samples i with 0 <= i + j < n
        if hi > lo:
            sh[lo:hi] = x[lo + j:hi + j]
        acc += sh                                        # a +0.0 where the reference skips a term: the f32 sum is unchanged
    return acc / np.float32(65)


def voice_length(text: bytes):
    """voice_length (whisper.cpp:3330-3353) over the token's bytes, summed in f32"""
    res = np.float32(0)
    for ch in text:
        c = chr(ch)
        res = np.float32(res + np.float32(0.01 if c == " " else 2.0 if c == "," else 3.0 if c in ".!?" or "0" <= c <= "9" else 1.0))
    return float(res)


def _ts_to_sample(t, n):
    q = abs(t) * 16000 // 100                            # C's int64 division truncates toward zero
    return max(0, min(n - 1, q if t >= 0 else -q))


def _sample_to_ts(i):
    return (100 * i) // 16000


def token_times(tokens, vlen, times, t0, t1, beg, eot, energy, thold_pt, thold_ptsum, state, hit=None):
    """whisper_exp_compute_token_level_timestamps (whisper.cpp:3374-3600) for one segment: tokens = dicts (id, tid, pt, ptsum), vlen =
    floats, times = list of [t0, t1, vlen] changed in place, state = [t_beg, t_last, tid_last] changed in place.  hit (a set, may be
    None) collects the branches taken.  Returns False, changing nothing, without energy."""
    n_samples = len(energy)
    if n_samples == 0:
        return False
    n = len(tokens)
    if n == 0:
        return True
    if n == 1:
        times[0][0], times[0][1] = t0, t1
        return True
    hit = set() if hit is None else hit
    f32 = np.float32
    for j, tok in enumerate(tokens):
        if j == 0:
            if tok["id"] == beg:
                times[0][0] = times[0][1] = times[1][0] = t0
                state[0], state[1], state[2] = t0, t0, beg
                hit.add("beg")
            else:
                times[0][0] = state[1]
        tt = state[0] + 2 * (tok["tid"] - beg)
        times[j][2] = vlen[j]
        if f32(tok["pt"]) > f32(thold_pt) and f32(tok["ptsum"]) > f32(thold_ptsum) and tok["tid"] > state[2] and tt <= t1:
            if j > 0:
                times[j - 1][1] = tt
            times[j][0] = tt
            state[2] = tok["tid"]
    times[n - 2][1] = t1
    times[n - 1][0] = t1
    times[n - 1][1] = t1
    state[1] = t1
    p0 = p1 = 0
    while True:
        while p1 < n and times[p1][1] < 0:
            p1 += 1
        if p1 >= n:
            p1 -= 1
        if p1 > p0:
            hit.add("vlen_split")
            psum = 0.0
            for j in range(p0, p1 + 1):
                psum += float(times[j][2])
            dt = float(times[p1][1] - times[p0][0])
            for j in range(p0 + 1, p1 + 1):
                ct = times[j - 1][0] + dt * float(times[j - 1][2]) / psum
                times[j - 1][1] = int(ct)                # C's double -> int64 conversion truncates toward zero
                times[j][0] = int(ct)
        p1 += 1
        p0 = p1
        if p1 >= n:
            break
    for j in range(n - 1):
        if times[j][1] < 0:
            times[j + 1][0] = times[j][1]
        if j > 0 and times[j - 1][1] > times[j][0]:
            times[j][0] = times[j - 1][1]
            times[j][1] = max(times[j][0], times[j][1])
    hw = 16000 // 8
    for j in range(n):
        if tokens[j]["id"] >= eot:
            continue
        s0 = _ts_to_sample(times[j][0], n_samples)
        s1 = _ts_to_sample(times[j][1], n_samples)
        ss0, ss1 = max(s0 - hw, 0), min(s1 + hw, n_samples)
        ns = ss1 - ss0
        sm = np.add.accumulate(energy[ss0:ss1], dtype=np.float32)[-1] if ns > 0 else f32(0)   # sequential f32 sum
        thold = f32(0.5 * float(sm) / ns)
        old0, old1 = times[j][0], times[j][1]
        k = s0
        if energy[k] > thold and j > 0:
            while k > 0 and energy[k] > thold:
                k -= 1
            times[j][0] = _sample_to_ts(k)
            if times[j][0] < times[j - 1][1]:
                times[j][0] = times[j - 1][1]
            else:
                s0 = k
        else:
            while energy[k] < thold and k < s1:
                k += 1
            s0 = k
            times[j][0] = _sample_to_ts(k)
        k = s1
        if energy[k] > thold:
            if j == n - 1:
                hit.add("read_past_end")                 # the reference reads tokens[n] here (j < ns - 1)
            while k < n_samples - 1 and energy[k] > thold:
                k += 1
            times[j][1] = _sample_to_ts(k)
            if j < ns - 1 and j + 1 < n and times[j][1] > times[j + 1][0]:
                times[j][1] = times[j + 1][0]
            else:
                s1 = k
        else:
            while energy[k] < thold and k > s0:
                k -= 1
            s1 = k
            times[j][1] = _sample_to_ts(k)
        if times[j][0] < old0:
            hit.add("t0_earlier")
        if times[j][0] > old0:
            hit.add("t0_later")
        if times[j][1] > old1:
            hit.add("t1_later")
        if times[j][1] < old1:
            hit.add("t1_earlier")
    return True


def wrap(ids, times, bytes_of, i0, i1, t0, t1, eot, max_len):
    """whisper_wrap_segment (whisper.cpp:2713-2763) of tokens [i0, i1) over [t0, t1]: [dict(t0, t1, i0, i1, text)], the text that of
    the non-special tokens"""
    out, start, acc, begin, text = [], i0, 0, t0, b""
    k = i0
    while k < i1:
        if ids[k] >= eot:
            k += 1
            continue
        txt = bytes_of(ids[k])
        cur = len(txt)
        if acc + cur > max_len and k > start:
            out.append(dict(t0=begin, t1=times[k][0], i0=start, i1=k, text=text.decode(errors="replace")))
            begin, start, acc, text = times[k][0], k, 0, b""
            continue                                     # the new segment's loop restarts at this token
        acc += cur
        text += txt
        k += 1
    out.append(dict(t0=begin, t1=t1, i0=start, i1=i1, text=text.decode(errors="replace")))
    return out


def window_token_times(tokens, result, eot, beg, bytes_of, energy, max_len=0, thold_pt=THOLD_PT, thold_ptsum=THOLD_PTSUM,
                       speed_up=False, hit=None):
    """what wsp_window_token_times returns for one window: (segments after wrapping, times[n_tokens] as [t0, t1, vlen]); bytes_of(id) =
    the token's text as bytes"""
    segs = mkw.segments(tokens, result, 0, eot, beg, lambda i: bytes_of(i).decode(errors="replace"), speed_up=speed_up)
    n = 0 if result["failed"] else result["n_tokens"]
    times = [[-1, -1, 0.0] for _ in range(result["n_tokens"])]
    vlen = [voice_length(bytes_of(t["id"])) for t in tokens[:n]]
    state, out = [0, 0, 0], []
    for s in segs:
        sub = times[s["i0"]:s["i1"]]
        token_times(tokens[s["i0"]:s["i1"]], vlen[s["i0"]:s["i1"]], sub, s["t0"], s["t1"], beg, eot, energy, thold_pt, thold_ptsum,
                    state, hit)
        if max_len > 0:
            pieces = wrap([t["id"] for t in tokens], times, bytes_of, s["i0"], s["i1"], s["t0"], s["t1"], eot, max_len)
            if hit is not None and len(pieces) > 1:
                hit.add("wrap_split")
            out += pieces
        else:
            out.append(s)
    return out, times


# ---- the fixture ----------------------------------------------------------------------------------------------------------------
def full_segments(o, pcm, max_len):
    """the reference's whisper_full with token timestamps: [dict(t0, t1, text, ids, times)]"""
    import ctypes as C
    o.clear_prompt_past()
    L = o.L
    pcm = np.ascontiguousarray(pcm, np.float32)
    rc = L.ora_full_ex2(o.ctx, pcm.ctypes.data_as(C.POINTER(C.c_float)), pcm.size, o.threads, 2 | 0x100, b"en", 0, 0, 0, max_len)
    assert rc == 0
    out = []
    for i in range(L.ora_full_n_segments(o.ctx)):
        nt = L.ora_full_n_tokens(o.ctx, i)
        out.append(dict(t0=L.ora_full_segment_t0(o.ctx, i), t1=L.ora_full_segment_t1(o.ctx, i),
                        text=L.ora_full_segment_text(o.ctx, i).decode(errors="replace"),
                        ids=[L.ora_full_token_id(o.ctx, i, j) for j in range(nt)],
                        times=[[L.ora_full_token_t0(o.ctx, i, j), L.ora_full_token_t1(o.ctx, i, j), float(L.ora_full_token_vlen(o.ctx, i, j))]
                               for j in range(nt)]))
    return out


def check_against_full(o, pcm, toks, segs, times, max_len):
    """whisper_full's first segments must be the restatement's, token times included"""
    full = full_segments(o, pcm, max_len)
    assert len(full) >= len(segs), (len(full), len(segs))
    for s, f in zip(segs, full):
        assert (s["t0"], s["t1"], s["text"]) == (f["t0"], f["t1"], f["text"]), (s, f)
        assert [t["id"] for t in toks[s["i0"]:s["i1"]]] == f["ids"], (s, f)
        for i, ft in zip(range(s["i0"], s["i1"]), f["times"]):
            assert times[i][0] == ft[0] and times[i][1] == ft[1] and np.float32(times[i][2]) == np.float32(ft[2]), (i, times[i], ft)


def p_clear(toks, n):
    return all(abs(t["pt"] - THOLD_PT) > P_TOL and abs(t["ptsum"] - THOLD_PTSUM) > P_TOL for t in toks[:n])


def make_case(name):
    from oracle.ref import RefOracle
    from whisper_b200 import capi
    model, threads, batch = CASES[name]
    path = synth.model_path(model)
    vocab = capi.Model(path)
    oracles = {th: RefOracle(path, threads=th, log_level=0) for th in threads}
    o0 = oracles[threads[0]]
    eot, beg, prompt = o0.special["eot"], o0.special["beg"], prompt_of(o0)
    bytes_of = lambda i: vocab.L.wsp_model_token_text(vocab.h, i) or b""
    kept = []            # (chunk, n_samples, branches, {th: (tokens, result, gaps, {max_len: (segs, times)})})

    def run(ch, n):
        pcm = synth.synth_pcm(ch, n)
        energy = signal_energy(pcm)
        mel = o0.pcm_to_mel(pcm)
        rs, hit, ok = {}, set(), True
        for th, o in oracles.items():
            o.set_mel(mel)
            o.encode(0)
            toks, res, kind, gaps = mkw.window(o, prompt, n, 0, 0)
            if kind == "short":
                hit.add("short")
            if res["failed"]:
                hit.add("failed")
            per = {}
            for ml in MAX_LENS:
                h = set()
                per[ml] = window_token_times(toks, res, eot, beg, bytes_of, energy, ml, hit=h)
                hit |= h
            ok &= (min(gaps) if gaps else np.inf) >= GAP_SAFE and p_clear(toks, res["n_tokens"])
            rs[th] = (toks, res, gaps, per)
        ok &= "read_past_end" not in hit
        return pcm, rs, hit, ok

    def covered():
        return set().union(*[k[2] for k in kept]) & set(BRANCHES) if kept else set()

    pcm, rs, hit, ok = run(0, SHORT)
    assert ok and "short" in hit
    kept.append((0, SHORT, hit, rs))
    for ch in range(CHUNK_TRIES):
        for n in LENGTHS:
            if covered() == set(BRANCHES) and len(kept) >= batch:
                break
            pcm, rs, hit, ok = run(ch, n)
            new = hit & set(BRANCHES) - covered()
            fill = covered() >= set(BRANCHES) - {"failed"} and ch not in [k[0] for k in kept] and rs[threads[0]][1]["n_tokens"] > 1
            take = ok and (bool(new) or (fill and len(kept) < batch - (0 if "failed" in covered() else 1)))
            print("  %s chunk %d, %d samples: %s, n_tokens %d %s" % (name, ch, n, sorted(hit), rs[threads[0]][1]["n_tokens"],
                                                                  "keep" if take else "skip"), flush=True)
            if take:
                for th, o in oracles.items():
                    toks, res, _g, per = rs[th]
                    if not res["failed"]:
                        for ml in MAX_LENS:
                            check_against_full(o, pcm, toks, per[ml][0], per[ml][1], ml)
                kept.append((ch, n, hit, rs))
        if covered() == set(BRANCHES) and len(kept) >= batch:
            break
    if covered() != set(BRANCHES) or len(kept) < batch:
        raise RuntimeError("%s: batch lacks %s (%d chunks)" % (name, sorted(set(BRANCHES) - covered()), len(kept)))
    kept = kept[:batch]
    if set().union(*[k[2] for k in kept]) & set(BRANCHES) != set(BRANCHES):
        raise RuntimeError("%s: the first %d chunks lack a branch" % (name, batch))
    out = {name + "_chunks": np.array([k[0] for k in kept], np.int32),
           name + "_n_samples": np.array([k[1] for k in kept], np.int32),
           name + "_prompt": np.array(prompt, np.int32), name + "_threads": np.array(threads, np.int32),
           name + "_branches": np.array([",".join(sorted(k[2] & set(BRANCHES))) for k in kept])}
    nm = mkw.n_max_of(o0)
    for th in threads:
        tok = np.full((batch, nm, 2), -1, np.int32)             # id, tid
        prob = np.full((batch, nm, 3), np.nan, np.float32)      # p, pt, ptsum
        gaps = np.full((batch, nm), np.nan, np.float32)
        res = np.zeros((batch, 4), np.int32)                    # n_sampled, n_tokens, seek_delta, failed
        for b, (_ch, _n, _h, rs) in enumerate(kept):
            toks, r, g, _per = rs[th]
            for i, t in enumerate(toks):
                tok[b, i] = (t["id"], t["tid"])
                prob[b, i] = (t["p"], t["pt"], t["ptsum"])
            gaps[b, :len(g)] = g
            res[b] = (r["n_sampled"], r["n_tokens"], r["seek_delta"], r["failed"])
        pre = "%s_t%d_" % (name, th)
        out[pre + "tokens"], out[pre + "probs"], out[pre + "gap"], out[pre + "result"] = tok, prob, gaps, res
        for ml in MAX_LENS:
            segs = np.full((batch, MAX_SEGS, 4), -1, np.int64)  # t0, t1, i0, i1
            texts = np.full((batch, MAX_SEGS), "", dtype=object)
            times = np.full((batch, nm, 2), -1, np.int64)       # token t0, t1
            vlen = np.zeros((batch, nm), np.float32)
            for b, (_ch, _n, _h, rs) in enumerate(kept):
                sg, tt = rs[th][3][ml]
                assert len(sg) <= MAX_SEGS
                for j, s in enumerate(sg):
                    segs[b, j] = (s["t0"], s["t1"], s["i0"], s["i1"])
                    texts[b, j] = s["text"]
                for i, t in enumerate(tt):
                    times[b, i] = (t[0], t[1])
                    vlen[b, i] = t[2]
            p = "%sml%d_" % (pre, ml)
            out[p + "segments"], out[p + "texts"], out[p + "times"], out[p + "vlen"] = segs, texts.astype(str), times, vlen
    return out


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)       # a subset of the cases is merged into the existing file
    new = {}
    for nm in names:
        new.update(make_case(nm))
    data = dict(np.load(OUT)) if os.path.exists(OUT) and len(names) < len(CASES) else {}
    data.update(new)
    np.savez_compressed(OUT, **data)
    print("chunks_token_ts %.0f KB" % (os.path.getsize(OUT) / 1024), flush=True)

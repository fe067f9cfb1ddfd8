"""The span fixtures (tests/golden/chunks_spans.npz, made by tests/golden/make_chunks_spans_golden.py from oracle/_ref): each case
covers every kind its generator requires, with several rows on one slot and a slot no row names; every margin clears its bound;
every stored result is the window rule restated at the row's seek and seek_end over its stored ids; every stored segment list is what
wsp_window_segments and the restated segmentation make of the stored tokens at that seek; and the stored token times are what the
library's token-time code (csrc/token_times.h, through wsp_test_token_times) gives over the source's signal energy.  CPU only."""
import os

import numpy as np
import pytest

from tests.golden import make_chunks_spans_golden as mks
from tests.golden import make_chunks_token_ts_golden as mkt
from tests.golden import make_chunks_window_golden as mkw
from tests.golden.make_golden import GAP_SAFE
from whisper_b200 import capi, synth

PATH = os.path.join(os.path.dirname(__file__), "golden", "chunks_spans.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(PATH)


def sources(g, name):
    return [mks.source_pcm([tuple(int(x) for x in p) for p in s if p[0] >= 0]) for s in g[name + "_sources"]]


def rows(g, name, th, ml=None):
    """per row: (tokens as dicts, result dict, segments as dicts, gaps)"""
    p = "%s_t%d_" % (name, th)
    q = p if ml is None else "%sml%d_" % (p, ml)
    out = []
    for b in range(g[p + "result"].shape[0]):
        n_s, n_t, sd, f = [int(x) for x in g[p + "result"][b]]
        toks = [dict(id=int(i), tid=int(t), p=float(pp), pt=float(pt), ptsum=float(ps))
                for (i, t), (pp, pt, ps) in zip(g[p + "tokens"][b, :n_s], g[p + "probs"][b, :n_s])]
        segs = g[q + "segments"][b]
        k = int((segs[:, 0] >= 0).sum())
        sg = [dict(t0=int(s[0]), t1=int(s[1]), i0=int(s[2]), i1=int(s[3]), text=str(t)) for s, t in zip(segs[:k], g[q + "texts"][b, :k])]
        out.append((toks, dict(n_sampled=n_s, n_tokens=n_t, seek_delta=sd, failed=f), sg, g[p + "gap"][b]))
    return out


def test_fixture_is_small(g):
    assert os.path.getsize(PATH) < 300_000
    assert all(name + "_spans" in g.files for name in mks.CASES)


@pytest.mark.parametrize("name", list(mks.CASES))
def test_coverage(g, name):
    _model, threads, sentinel, mt, single, srcs, needs, _shared = mks.CASES[name]
    assert g[name + "_threads"].tolist() == list(threads) and g[name + "_params"].tolist() == [mt, single]
    kinds = set(",".join(g[name + "_kinds"].tolist()).split(","))
    assert set(needs) - {"lang_diff"} - set(mks.OPTIONAL) <= kinds
    spans = g[name + "_spans"]
    slots = spans[:, 0].tolist()
    assert max(slots.count(s) for s in set(slots)) >= 2, "several rows on one slot"
    assert set(range(len(srcs))) - set(slots), "a slot no row names"
    pcms = sources(g, name)
    assert any(p.size > 480000 for p in pcms)
    p = "%s_t%d_" % (name, threads[0])
    if sentinel:
        assert (g[name + "_prompt"] == capi.TOKEN_LANGUAGE_AUTO).sum() == 1
        langs = g[p + "lang"]
        assert any(len({int(langs[b]) for b in range(len(slots)) if slots[b] == s}) >= 2 for s in set(slots)), "two languages on a slot"
    if mt:
        assert "max_tokens" in kinds and single


@pytest.mark.parametrize("name", list(mks.CASES))
def test_results_segments_and_margins(g, name):
    model, threads, sentinel, mt, single, _srcs, _needs, _shared = mks.CASES[name]
    m = capi.Model(synth.model_path(model))
    eot, beg, n_max = m.special["eot"], m.special["beg"], m.n_text_ctx // 2 - 4
    text = lambda i: m.token_text(i) or ""
    pcms = sources(g, name)
    spans = [tuple(int(x) for x in s) for s in g[name + "_spans"]]
    for th in threads:
        for b, ((toks, res, segs, gaps), (slot, off, dur)) in enumerate(zip(rows(g, name, th), spans)):
            seek, seek_end = mks.bounds(off, dur, pcms[slot].size // 160)
            if seek_end <= seek + 100:
                assert res == dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0) and segs == [], b
                continue
            assert np.nanmin(gaps, initial=np.inf) >= GAP_SAFE, b
            ids = [t["id"] for t in toks]
            want, kind, used = mkw.rule(ids, eot, beg, mt, single, n_max, seek, seek_end)
            assert kind is not None and used == len(ids), b
            assert (res["n_tokens"], res["seek_delta"], res["failed"]) == (want["result_len"], want["seek_delta"], want["failed"]), b
            assert segs == mkw.segments(toks, res, seek, eot, beg, text, single_segment=bool(single)), b
            assert segs == m.window_segments(toks, res, seek, capi.SEGMENT_SINGLE if single else 0), b
            assert mkt.p_clear(toks, res["n_tokens"]), b
        if not sentinel:
            assert (g["%s_t%d_lang" % (name, th)] == -1).all()


@pytest.mark.parametrize("ml", mks.MAX_LENS)
@pytest.mark.parametrize("name", [n for n in mks.CASES if mks.TOKEN_TIMES[n]])
def test_token_times_are_the_library_s(g, name, ml):
    """the stored token times, restated over the source's whole energy from t_beg = t_last = 0, and csrc/token_times.h agree"""
    model, threads, _sentinel, _mt, single, _srcs, _needs, _shared = mks.CASES[name]
    m = capi.Model(synth.model_path(model))
    eot, beg = m.special["eot"], m.special["beg"]
    bytes_of = lambda i: m.token_bytes(i)
    pcms = sources(g, name)
    energies = [mkt.signal_energy(p) for p in pcms]
    spans = [tuple(int(x) for x in s) for s in g[name + "_spans"]]
    for th in threads:
        q = "%s_t%d_ml%d_" % (name, th, ml)
        for b, ((toks, res, segs, _gaps), (slot, off, _dur)) in enumerate(zip(rows(g, name, th, ml), spans)):
            seek = off // 10
            got_segs, times = mks.span_token_times(toks, res, seek, eot, beg, bytes_of, energies[slot], ml, bool(single), set())
            assert [(s["t0"], s["t1"], s["i0"], s["i1"]) for s in got_segs] == [(s["t0"], s["t1"], s["i0"], s["i1"]) for s in segs], b
            n = res["n_tokens"]
            assert [(int(a), int(z)) for a, z, _v in times] == [tuple(x) for x in g[q + "times"][b, :n].tolist()], b
            # the library's code over the same segments (plain cut, before wrapping), in order from a new call's state
            cut = mkw.segments(toks, res, seek, eot, beg, lambda i: bytes_of(i).decode(errors="replace"), single_segment=bool(single))
            state = (0, 0, 0)
            for s in cut:
                sub = toks[s["i0"]:s["i1"]]
                vlen = [mkt.voice_length(bytes_of(t["id"])) for t in sub]
                lib, state, _ok = capi.test_token_times(sub, vlen, s["t0"], s["t1"], beg, eot, energies[slot], state=state)
                want = times[s["i0"]:s["i1"]]
                assert [(a, z) for a, z, _v in lib] == [(a, z) for a, z, _v in want], (b, s)

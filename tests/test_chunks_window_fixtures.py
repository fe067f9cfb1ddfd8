"""The window batch fixtures (tests/golden/chunks_window.npz, made by tests/golden/make_chunks_window_golden.py from oracle/_ref): the
batches together cover every kind of window end the generator requires, every margin is >= GAP_SAFE, every stored result is the window
rule restated over its stored ids, and every stored segment list is what wsp_window_segments and the restated segmentation make of
the stored tokens.  Where the oracle is built, one chunk is re-run and must reproduce the stored window.  CPU only."""
import os

import numpy as np
import pytest

from tests.golden import make_chunks_window_golden as mk
from tests.golden.make_golden import GAP_SAFE, prompt_of
from whisper_b200 import capi, synth

PATH = os.path.join(os.path.dirname(__file__), "golden", "chunks_window.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(PATH)


def windows(g, name, th):
    """per chunk: (tokens as dicts, result dict, segments as dicts, gaps)"""
    p = "%s_t%d_" % (name, th)
    out = []
    for b in range(g[p + "result"].shape[0]):
        n_s, n_t, sd, f = [int(x) for x in g[p + "result"][b]]
        toks = [dict(id=int(i), tid=int(t), p=float(pp), pt=float(pt), ptsum=float(ps))
                for (i, t), (pp, pt, ps) in zip(g[p + "tokens"][b, :n_s], g[p + "probs"][b, :n_s])]
        segs = g[p + "segments"][b]
        k = int((segs[:, 0] >= 0).sum())
        sg = [dict(t0=int(s[0]), t1=int(s[1]), i0=int(s[2]), i1=int(s[3]), text=str(t)) for s, t in zip(segs[:k], g[p + "texts"][b, :k])]
        out.append((toks, dict(n_sampled=n_s, n_tokens=n_t, seek_delta=sd, failed=f), sg, g[p + "gap"][b]))
    return out


def test_fixture_is_small(g):
    assert os.path.getsize(PATH) < 300_000
    assert all(name + "_chunks" in g.files for name in mk.CASES)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_coverage(g, name):
    _model, threads, batch, mt, single, need = mk.CASES[name]
    assert g[name + "_threads"].tolist() == list(threads) and g[name + "_params"].tolist() == [mt, single]
    assert g[name + "_chunks"].shape == (batch,)
    kinds = set(",".join(g[name + "_kinds"].tolist()).split(","))
    assert set(need) <= kinds
    assert (g[name + "_n_samples"] < 16000).any(), "a clip under 1 s"
    for th in threads:
        rs = [w[1] for w in windows(g, name, th)]
        assert any(r["failed"] for r in rs) == ("n_max" in need)
        assert any(r["n_sampled"] == 0 for r in rs)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_results_segments_and_margins(g, name):
    model, threads, _batch, mt, single, need = mk.CASES[name]
    m = capi.Model(synth.model_path(model))
    eot, beg, n_max = m.special["eot"], m.special["beg"], m.n_text_ctx // 2 - 4
    text = lambda i: m.token_text(i) or ""
    for th in threads:
        kinds = {"single_segment"} if single else set()
        for b, (toks, res, segs, gaps) in enumerate(windows(g, name, th)):
            seek_end = int(g[name + "_n_samples"][b]) // 160
            if seek_end <= 100:
                assert res == dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0) and segs == []
                kinds.add("short")
                continue
            r, kind, used = mk.rule([t["id"] for t in toks], eot, beg, mt, single, n_max, 0, seek_end)
            assert kind is not None and used == res["n_sampled"]
            kinds.add(kind)
            assert (r["result_len"], r["seek_delta"], r["failed"]) == (res["n_tokens"], res["seek_delta"], res["failed"])
            assert segs == mk.segments(toks, res, 0, eot, beg, text, single_segment=bool(single))
            flags = capi.SEGMENT_SINGLE if single else 0
            assert segs == m.window_segments(toks, res, 0, flags)
            n = res["n_sampled"]
            assert (gaps[:n - 1] >= GAP_SAFE).all() and np.isnan(gaps[n - 1:]).all()
        # the kinds of end, derived again from the stored ids
        assert set(need) <= kinds, (th, kinds)


def test_reference_rerun(g, ref_available):
    if not ref_available:
        pytest.skip("oracle/_ref not built")
    from oracle.ref import RefOracle
    name = "micro_en"
    model, threads, _batch, mt, single, _need = mk.CASES[name]
    th = threads[-1]
    o = RefOracle(synth.model_path(model), threads=th)
    b = int(np.argmax(g["%s_t%d_result" % (name, th)][:, 0]))
    o.pcm_to_mel(synth.synth_pcm(int(g[name + "_chunks"][b]), int(g[name + "_n_samples"][b])))
    o.encode(0)
    assert prompt_of(o) == g[name + "_prompt"].tolist()
    toks, res, _kind, _gaps = mk.window(o, prompt_of(o), int(g[name + "_n_samples"][b]), mt, single)
    want = windows(g, name, th)[b]
    assert res == want[1]
    assert [(t["id"], t["tid"]) for t in toks] == [(t["id"], t["tid"]) for t in want[0]]

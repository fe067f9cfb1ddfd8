"""The token-timestamp batch fixtures (tests/golden/chunks_token_ts.npz, made by tests/golden/make_chunks_token_ts_golden.py from
oracle/_ref): every stored segment list and token time is what the Python restatement makes of the stored tokens over the clip's
signal energy, each batch reaches every branch the generator requires, every margin is >= GAP_SAFE, every result token's pt and ptsum
lie more than the GPU's probability tolerance from their thresholds, and no segment ends in the branch where the reference reads past
the segment.  Where the oracle is built, one chunk is re-run through the reference's whisper_full.  CPU only."""
import os

import numpy as np
import pytest

from oracle import ref
from tests.golden import make_chunks_token_ts_golden as mk
from tests.golden.make_golden import GAP_SAFE
from whisper_b200 import capi, synth

PATH = os.path.join(os.path.dirname(__file__), "golden", "chunks_token_ts.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(PATH)


def windows(g, name, th):
    """per chunk: (tokens as dicts, result dict, gaps)"""
    p = "%s_t%d_" % (name, th)
    out = []
    for b in range(g[p + "result"].shape[0]):
        n_s, n_t, sd, f = [int(x) for x in g[p + "result"][b]]
        toks = [dict(id=int(i), tid=int(t), p=float(pp), pt=float(pt), ptsum=float(ps))
                for (i, t), (pp, pt, ps) in zip(g[p + "tokens"][b, :n_s], g[p + "probs"][b, :n_s])]
        out.append((toks, dict(n_sampled=n_s, n_tokens=n_t, seek_delta=sd, failed=f), g[p + "gap"][b]))
    return out


def stored(g, name, th, ml, b, n):
    q = "%s_t%d_ml%d_" % (name, th, ml)
    segs = g[q + "segments"][b]
    k = int((segs[:, 0] >= 0).sum())
    s = [(int(x[0]), int(x[1]), int(x[2]), int(x[3]), str(t)) for x, t in zip(segs[:k], g[q + "texts"][b, :k])]
    t = [(int(a), int(z), float(v)) for (a, z), v in zip(g[q + "times"][b, :n].tolist(), g[q + "vlen"][b, :n].tolist())]
    return s, t


def test_fixture_is_small(g):
    assert os.path.getsize(PATH) < 300_000
    assert all(name + "_chunks" in g.files for name in mk.CASES)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_restatement_coverage_margins(g, name):
    model, threads, batch = mk.CASES[name]
    assert g[name + "_threads"].tolist() == list(threads) and g[name + "_chunks"].size == batch
    m = capi.Model(synth.model_path(model))
    eot, beg = m.special["eot"], m.special["beg"]
    hit = set()
    for th in threads:
        for b, (toks, res, gaps) in enumerate(windows(g, name, th)):
            pcm = synth.synth_pcm(int(g[name + "_chunks"][b]), int(g[name + "_n_samples"][b]))
            energy = mk.signal_energy(pcm)
            if pcm.size // 160 <= 100:
                hit.add("short")
                assert res == dict(n_sampled=0, n_tokens=0, seek_delta=0, failed=0)
            if res["failed"]:
                hit.add("failed")
            assert np.all(gaps[~np.isnan(gaps)] >= GAP_SAFE), (name, th, b)
            assert mk.p_clear(toks, res["n_tokens"]), (name, th, b)
            for ml in mk.MAX_LENS:
                h = set()
                segs, times = mk.window_token_times(toks, res, eot, beg, m.token_bytes, energy, ml, hit=h)
                got = ([(s["t0"], s["t1"], s["i0"], s["i1"], s["text"]) for s in segs], [(t[0], t[1], float(np.float32(t[2]))) for t in times])
                assert got == stored(g, name, th, ml, b, res["n_tokens"]), (name, th, ml, b)
                assert "read_past_end" not in h, (name, th, ml, b)
                if res["failed"] or pcm.size // 160 <= 100:
                    assert segs == []
                hit |= h
            assert set(str(g[name + "_branches"][b]).split(",")) - {""} <= hit
    assert set(mk.BRANCHES) <= hit, sorted(set(mk.BRANCHES) - hit)


@pytest.mark.skipif(not ref.available(), reason="oracle/_ref not built")
def test_one_chunk_against_whisper_full(g):
    name = "micro_en"
    model, threads, _batch = mk.CASES[name]
    th = threads[-1]
    wins = windows(g, name, th)
    b = max(range(len(wins)), key=lambda i: wins[i][1]["n_tokens"] * (1 - wins[i][1]["failed"]))
    toks, res, _gaps = wins[b]
    pcm = synth.synth_pcm(int(g[name + "_chunks"][b]), int(g[name + "_n_samples"][b]))
    o = ref.RefOracle(synth.model_path(model), threads=th, log_level=0)
    m = capi.Model(synth.model_path(model))
    for ml in mk.MAX_LENS:
        segs, times = mk.window_token_times(toks, res, m.special["eot"], m.special["beg"], m.token_bytes, mk.signal_energy(pcm), ml)
        mk.check_against_full(o, pcm, toks, segs, times, ml)

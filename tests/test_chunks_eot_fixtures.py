"""The end-of-text batch fixtures (tests/golden/chunks_eot.npz, made by tests/golden/make_chunks_eot_golden.py from oracle/_ref): every
case holds a batch with at least two distinct EOT steps and at least one chunk that reaches the cap, each chunk's tokens end at its
first EOT, and the reference's top-2 margin is >= GAP_SAFE at every step of every output.  Where the oracle is built, one chunk of
the micro.en case is re-run and must reproduce the stored tokens exactly.  CPU only."""
import os

import numpy as np
import pytest

from tests.golden import make_chunks_eot_golden as mk
from tests.golden.make_golden import GAP_SAFE, prompt_of
from whisper_b200 import synth

PATH = os.path.join(os.path.dirname(__file__), "golden", "chunks_eot.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(PATH)


def test_fixture_is_small(g):
    assert os.path.getsize(PATH) < 200_000
    assert all(name + "_chunks" in g.files for name in mk.CASES)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_case_shape(g, name):
    model, threads, batch = mk.CASES[name]
    assert g[name + "_threads"].tolist() == list(threads)
    assert g[name + "_chunks"].shape == (batch,) and g[name + "_n_samples"].shape == (batch,)
    assert int(g[name + "_cap"]) == mk.CAP
    assert int(g[name + "_eot"]) == (50256 if ".en" in model else 50257)   # multilingual files shift the specials by one
    assert (g[name + "_n_samples"] <= 480000).all()


@pytest.mark.parametrize("name", list(mk.CASES))
def test_case_properties(g, name):
    _model, threads, batch = mk.CASES[name]
    eot, cap = int(g[name + "_eot"]), mk.CAP
    for th in threads:
        p = "%s_t%d_" % (name, th)
        toks, gaps, n_out, ends = g[p + "tokens"], g[p + "gap"], g[p + "n_out"], g[p + "eot_step"]
        assert toks.shape == (batch, cap) and gaps.shape == (batch, cap - 1)
        assert len(set(ends[ends > 0].tolist())) >= 2, "two distinct EOT steps"
        assert (ends == 0).any(), "one chunk at the cap"
        for b in range(batch):
            n, row = int(n_out[b]), toks[b]
            assert 1 <= n <= cap and (row[n:] == -1).all() and (row[:n] >= 0).all()
            hits = np.flatnonzero(row[:n] == eot)
            if ends[b]:
                assert n == ends[b] and hits.tolist() == [n - 1], "the output ends at its first EOT"
            else:
                assert n == cap and hits.size == 0
            assert (gaps[b, :n - 1] >= GAP_SAFE).all() and np.isnan(gaps[b, n - 1:]).all()
        # zero-padded clips are what moves a chunk off its script: the batch holds some
        assert (g[name + "_n_samples"] < 480000).any()


def test_reference_rerun(g, ref_available):
    if not ref_available:
        pytest.skip("oracle/_ref not built")
    from oracle.ref import RefOracle
    model, threads, _batch = mk.CASES["micro_en"]
    o = RefOracle(synth.model_path(model), threads=threads[-1])
    p = "micro_en_t%d_" % threads[-1]
    b = int(np.argmax(g[p + "eot_step"]))
    o.pcm_to_mel(synth.synth_pcm(int(g["micro_en_chunks"][b]), int(g["micro_en_n_samples"][b])))
    o.encode(0)
    assert prompt_of(o) == g["micro_en_prompt"].tolist()
    toks, _gaps = mk.until_eot(o, prompt_of(o), mk.CAP)
    assert toks.tolist() == g[p + "tokens"][b, :int(g[p + "n_out"][b])].tolist()

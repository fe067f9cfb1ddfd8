"""The language-detection batch fixtures (tests/golden/chunks_lang.npz, made by tests/golden/make_chunks_lang_golden.py from oracle/_ref):
every case's batch holds both active languages, each chunk's top-2 language-probability gap is at least
10x the GPU's 2e-4 tolerance, every decoding margin is >= GAP_SAFE, the tokens end at their first EOT or the cap, and some chunk
decodes differently under the other language's prompt.  Where the oracle is built, one chunk of the base case is re-run and must
reproduce the stored language, probabilities and tokens exactly.  CPU only."""
import os

import numpy as np
import pytest

from tests.golden import make_chunks_lang_golden as mk
from tests.golden.make_golden import GAP_SAFE
from whisper_b200 import synth

PATH = os.path.join(os.path.dirname(__file__), "golden", "chunks_lang.npz")
EOT, SOT, TRANSCRIBE = 50257, 50258, 50359          # micro-sc is multilingual: the specials are shifted by one


@pytest.fixture(scope="module")
def g():
    return np.load(PATH)


def test_fixture_is_small(g):
    assert os.path.getsize(PATH) < 200_000
    assert all(name + "_chunks" in g.files for name in mk.CASES)


@pytest.mark.parametrize("name", list(mk.CASES))
def test_case_shape(g, name):
    threads, batch, audio_ctx, first, lengths = mk.CASES[name]
    assert g[name + "_threads"].tolist() == list(threads)
    assert g[name + "_chunks"].shape == (batch,) and set(g[name + "_n_samples"].tolist()) <= set(lengths)
    assert (g[name + "_chunks"] >= first).all() and (g[name + "_chunks"] < first + mk.CHUNK_TRIES).all()
    assert int(g[name + "_audio_ctx"]) == audio_ctx
    assert int(g[name + "_cap"]) == mk.CAP
    assert g[name + "_prompt"].tolist() == [SOT, -1, TRANSCRIBE]


@pytest.mark.parametrize("name", list(mk.CASES))
def test_case_properties(g, name):
    threads, batch = mk.CASES[name][:2]
    cap = mk.CAP
    for th in threads:
        p = "%s_t%d_" % (name, th)
        ids, probs = g[p + "lang_id"], g[p + "lang_probs"]
        assert probs.shape == (batch, 99) and np.allclose(probs.sum(axis=1), 1.0, atol=1e-5)
        assert (ids == probs.argmax(axis=1)).all() and set(ids.tolist()) <= set(mk.ACTIVE)
        assert set(ids.tolist()) == set(mk.ACTIVE), "both languages"
        s = np.sort(probs, axis=1)
        assert (s[:, -1] - s[:, -2] >= mk.LANG_GAP_SAFE).all(), "no top tie within 10x the tolerance"
        assert (ids == g[name + "_t%d_lang_id" % threads[0]]).all()
        differs = 0
        for b in range(batch):
            for key, n_key in (("tokens", "n_out"), ("other_tokens", "other_n_out")):
                n, row = int(g[p + n_key][b]), g[p + key][b]
                assert 1 <= n <= cap and (row[n:] == -1).all() and (row[:n] >= 0).all()
                hits = np.flatnonzero(row[:n] == EOT)
                assert hits.tolist() in ([n - 1], []) and (hits.size or n == cap), "the output ends at its first EOT or the cap"
            n = int(g[p + "n_out"][b])
            gaps = g[p + "gap"][b]
            assert (gaps[:n - 1] >= GAP_SAFE).all() and np.isnan(gaps[n - 1:]).all()
            differs += g[p + "tokens"][b].tolist() != g[p + "other_tokens"][b].tolist()
        assert differs >= 1, "a wrong language in the prompt must show in the tokens"


def test_reference_rerun(g, ref_available):
    if not ref_available:
        pytest.skip("oracle/_ref not built")
    from oracle.ref import RefOracle
    threads = mk.CASES["base"][0]
    p = "base_t%d_" % threads[-1]
    o = RefOracle(synth.model_path(mk.MODEL), threads=threads[-1])
    b = int(np.flatnonzero(g[p + "lang_id"] == mk.ACTIVE[0])[0])
    lid, probs, toks, _gaps, otoks = mk.run_chunk(o, synth.synth_pcm(int(g["base_chunks"][b]), int(g["base_n_samples"][b])))
    assert lid == int(g[p + "lang_id"][b])
    assert np.array_equal(probs, g[p + "lang_probs"][b])
    assert toks.tolist() == g[p + "tokens"][b, :int(g[p + "n_out"][b])].tolist()
    assert otoks.tolist() == g[p + "other_tokens"][b, :int(g[p + "other_n_out"][b])].tolist()

"""The audio_ctx fixtures (tests/golden/audio_ctx.npz, made by tests/golden/make_audio_ctx_golden.py from oracle/_ref): shapes,
decision margins and token variety — the checks tests/test_oracle.py::test_fixtures_discriminate makes on the other fixtures — and,
where the oracle is built, a re-run of one case that must reproduce the stored data exactly.  CPU only."""
import os

import numpy as np
import pytest

from tests.golden.make_audio_ctx_golden import AUDIO_CTX, COL_STEP, FULL_RUNS, LOGIT_THIN, MODELS, N_STEPS, THREADS, rows_of
from tests.golden.make_golden import GAP_SAFE, LOGIT_STEP, MIN_DISTINCT

VOCAB = {"en": 51864, "ml": 51865}
D_MODEL, N_LAYERS = 128, 4       # the "micro" shape (whisper_b200/synth.py)


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(os.path.dirname(__file__), "golden", "audio_ctx.npz"))


def test_fixture_is_small(g):
    assert os.path.getsize(os.path.join(os.path.dirname(__file__), "golden", "audio_ctx.npz")) < 1_000_000
    assert g["audio_ctx"].tolist() == list(AUDIO_CTX) and g["threads"].tolist() == list(THREADS)
    assert int(g["n_steps"]) == N_STEPS and int(g["logit_step"]) == LOGIT_STEP * LOGIT_THIN and int(g["col_step"]) == COL_STEP


@pytest.mark.parametrize("key", list(MODELS))
@pytest.mark.parametrize("n", AUDIO_CTX)
def test_case_shapes_and_margins(g, key, n):
    p = "%s_n%d_" % (key, n)
    r1, r2 = rows_of(n), rows_of(2 * n)
    dc = len(range(0, D_MODEL, COL_STEP))
    assert g[p + "enc_input"].shape == (r2.size, len(range(0, 80, COL_STEP)))
    assert g[p + "enc_temp1"].shape == (r2.size, dc)
    assert g[p + "enc_layer0_in"].shape == (r1.size, dc)
    assert g[p + "encode_out"].shape == (r1.size, dc)
    assert g[p + "cross_k"].shape == g[p + "cross_v"].shape == (N_LAYERS, r1.size, dc)
    n_sub = len(range(0, VOCAB[key], LOGIT_STEP * LOGIT_THIN))
    prompt = g[key + "_prompt"]
    for th in THREADS:
        q = p + "t%d_" % th
        assert g[q + "prompt_logits"].shape == (prompt.size, n_sub)
        assert g[q + "step_logits"].shape == (N_STEPS - 1, n_sub)
        assert g[q + "tokens"].shape == (N_STEPS,)
        assert np.isfinite(g[q + "step_logits"]).all()
        if g[p + "tokens_pinned"]:
            # pinned greedy sequences: every decision clear of a near-tie, and not a degenerate repetition
            assert g[q + "gap"].min() >= GAP_SAFE
            assert len(set(g[q + "tokens"].tolist())) >= MIN_DISTINCT
    # a shorter window really is shorter: frames past 2n never reach the encoder, and its last row is the clip's frame 2n - 1
    assert np.abs(g[p + "enc_input"]).max() > 0


@pytest.mark.parametrize("key", list(MODELS))
def test_most_cases_pin_tokens_and_the_override_matters(g, key):
    pinned = [n for n in AUDIO_CTX if g["%s_n%d_tokens_pinned" % (key, n)]]
    assert 1499 in pinned and 750 in pinned and len(pinned) >= 4
    # on the same clip, a different audio_ctx gives the decoder different cross-attention memories, and different logits
    pairs = [(a, b) for a in AUDIO_CTX for b in AUDIO_CTX if a > b and g["%s_n%d_chunk" % (key, a)] == g["%s_n%d_chunk" % (key, b)]]
    assert pairs
    for a, b in pairs:
        assert np.abs(g["%s_n%d_t4_step_logits" % (key, a)] - g["%s_n%d_t4_step_logits" % (key, b)]).max() > 0.1, (a, b)


@pytest.mark.parametrize("name", list(FULL_RUNS))
def test_whisper_full_runs_discriminate(g, name):
    toks = g[name + "_tokens"]
    assert float(g[name + "_min_gap"]) >= GAP_SAFE
    assert g[name + "_t"].shape[0] >= 3 and g[name + "_ntok"].sum() == toks.size
    assert len(set(toks.tolist())) >= MIN_DISTINCT


def test_regenerated_case_is_identical(g):
    """Where oracle/_ref is built: the reference re-run on one stored case (micro.en-sc, n = 129, reference threads 1 and 4) gives
    exactly the stored tensors, logits and tokens."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref is not built")
    from tests.golden import make_audio_ctx_golden as mk
    from tests.golden.make_golden import logits_sample
    from whisper_b200 import synth
    key, n = "en", 129
    p = "%s_n%d_" % (key, n)
    model = MODELS[key][0]
    o1 = ref.RefOracle(synth.model_path(model), threads=1)
    mel = o1.pcm_to_mel(synth.synth_pcm(int(g[p + "chunk"]), 480000))
    for th in (1, 4):
        o, r = mk.run_case(model, mel, n, th)
        assert np.array_equal(r["tokens"], g[p + "t%d_tokens" % th])
        assert np.array_equal(r["step_logits"][..., ::LOGIT_THIN], g[p + "t%d_step_logits" % th])
        assert np.array_equal(logits_sample(r["prompt_logits"])[..., ::LOGIT_THIN], g[p + "t%d_prompt_logits" % th])
        assert np.array_equal(r["gap"], g[p + "t%d_gap" % th])
        if th == 1:
            k, v = mk.cross_kv(o, n)
            assert np.array_equal(k[:, rows_of(n), ::COL_STEP].astype(np.float16), g[p + "cross_k"])
            assert np.array_equal(v[:, rows_of(n), ::COL_STEP].astype(np.float16), g[p + "cross_v"])

"""The speed-up fixtures (tests/golden/speed_up.npz, made by tests/golden/make_speed_up_golden.py from oracle/_ref): shapes, frame counts,
decision margins and token variety; the numpy restatement of the phase-vocoder log-mel against every stored mel; the two misreadings of
the fold's edge that the high-frequency signal must expose; and, where the oracle is built, a re-run of one case that must reproduce
the stored data exactly.  CPU only."""
import os

import numpy as np
import pytest

from oracle.whisper_np import NpModel
from tests.golden import make_speed_up_golden as mk
from tests.golden.make_golden import GAP_SAFE, LOGIT_STEP, MIN_DISTINCT
from whisper_b200 import synth

PATH = os.path.join(os.path.dirname(__file__), "golden", "speed_up.npz")
VOCAB = {"en": 51864, "ml": 51865}
D_MODEL, N_LAYERS = 128, 4       # the "micro" shape (whisper_b200/synth.py)
CASES = [(key, name, "%s_%s_" % (key, name)) for key in mk.MODELS for name in mk.CLIPS] + \
        [(mk.AUDIO_CTX_CASE[0], mk.AUDIO_CTX_CASE[1], "%s_%s_n%d_" % mk.AUDIO_CTX_CASE)]


def tol_mel(g):
    """Twice the largest difference between the reference's mel and the f64-DFT restatement the generator measured over every
    fixture mel (the reference's own f32 FFT round-off): the GPU's DFT is exact to f32 rounding as well."""
    return 2.0 * float(g["mel_spread"])


@pytest.fixture(scope="module")
def g():
    return np.load(PATH)


@pytest.fixture(scope="module")
def filters():
    return NpModel(synth.model_path("micro.en-sc")).filters


def test_fixture_is_small_and_consistent(g):
    assert os.path.getsize(PATH) < 1_500_000
    assert g["threads"].tolist() == list(mk.THREADS) and int(g["n_steps"]) == mk.N_STEPS
    assert int(g["logit_step"]) == LOGIT_STEP * mk.LOGIT_THIN and int(g["col_step"]) == mk.COL_STEP
    assert int(g["row_step"]) == mk.ROW_STEP and int(g["mel_keep"]) == mk.MEL_KEEP
    # the spread is f32 round-off of log10 values of order 1, and far below the fold-edge effects below
    assert 0 < float(g["mel_spread"]) < 1e-3


@pytest.mark.parametrize("n", mk.MEL_LENGTHS)
def test_mel_only_frames_and_restatement(g, filters, n):
    mel = g["mel_len%d" % n]
    assert mel.shape == (80, n // 320)           # n_len = n_samples / fft_step with fft_step 320 (whisper.cpp:2080, 2303)
    assert np.abs(mk.log_mel(mk.mel_pcm(n), filters) - mel).max(initial=0.0) < tol_mel(g)


def test_high_frequency_signal_pins_the_fold_edge(g, filters):
    """On two tones just under 8 kHz the restatement matches the reference; folding bin 401 as well, or doubling bin 400, would not."""
    hf = g["mel_hf"]
    assert hf.shape == (80, mk.HF_SAMPLES // 320)
    tol = tol_mel(g)
    assert np.abs(mk.log_mel(mk.hf_pcm(), filters) - hf).max() < tol
    for misread in ({"fold_401": True}, {"double_400": True}):
        assert np.abs(mk.log_mel(mk.hf_pcm(), filters, **misread) - hf).max() > tol, misread
    # the top band weighs averaged bin 200 = 0.5 (P[400] + P[401]), which is where the tones' energy is
    assert filters[79, 200] > 0


@pytest.mark.parametrize("key,name,p", CASES)
def test_case_mel_restatement(g, filters, key, name, p):
    pcm = mk.case_pcm(int(g[p + "chunk"]), name)
    assert tuple(g[p + "mel_shape"]) == (80, pcm.size // 320)
    mel = mk.log_mel(pcm, filters)[:, ::mk.MEL_KEEP]
    assert np.abs(mel - g[p + "mel"]).max() < tol_mel(g)


@pytest.mark.parametrize("key,name,p", CASES)
def test_case_shapes_and_margins(g, key, name, p):
    n = mk.AUDIO_CTX_CASE[2] if p.endswith("_n%d_" % mk.AUDIO_CTX_CASE[2]) else 1500
    rows = len(range(0, n, mk.ROW_STEP))
    dc = len(range(0, D_MODEL, mk.COL_STEP))
    assert g[p + "encode_out"].shape == (rows, dc)
    assert g[p + "cross_k"].shape == g[p + "cross_v"].shape == (N_LAYERS, rows, dc)
    n_sub = len(range(0, VOCAB[key], LOGIT_STEP * mk.LOGIT_THIN))
    prompt = g[key + "_prompt"]
    for th in mk.THREADS:
        q = p + "t%d_" % th
        assert g[q + "prompt_logits"].shape == (prompt.size, n_sub)
        assert g[q + "step_logits"].shape == (mk.N_STEPS - 1, n_sub)
        assert g[q + "tokens"].shape == (mk.N_STEPS,)
        assert np.isfinite(g[q + "step_logits"]).all()
    if g[p + "tokens_pinned"]:
        # pinned greedy sequences: every decision clear of a near-tie, and not a degenerate repetition
        for th in mk.THREADS:
            q = p + "t%d_" % th
            assert g[q + "gap"].min() >= GAP_SAFE
            assert len(set(g[q + "tokens"].tolist())) >= MIN_DISTINCT


def test_every_full_window_pins_tokens(g):
    """Only the 45.7 s clips may leave their tokens unpinned: their window is zero-padded past frame 2285, and a random encoder's
    response to silence throws the scripted decoder off its script (as for make_golden's padded case)."""
    for key, name, p in CASES:
        assert g[p + "tokens_pinned"] or name == "s45", p


def test_language_detection_fixture(g):
    assert g["lang_chunks"].tolist() == list(mk.LANG_CHUNKS)
    assert g["lang_probs"].shape[0] == len(mk.LANG_CHUNKS)
    assert np.allclose(g["lang_probs"].sum(1), 1.0, atol=1e-4)
    assert (g["lang_probs"].argmax(1) == g["lang_id"]).all()


def test_regenerated_case_is_identical(g):
    """Where oracle/_ref is built: the reference re-run on the high-frequency signal and on one stored case (micro.en-sc, 75 s,
    reference threads 1 and 4) gives exactly the stored mel, tensors, logits and tokens."""
    from oracle import ref
    if not ref.available():
        pytest.skip("oracle/_ref is not built")
    from tests.golden.make_golden import logits_sample
    o1 = ref.RefOracle(synth.model_path("micro.en-sc"), threads=4)
    assert np.array_equal(mk.vocoder_mel(o1, mk.hf_pcm()), g["mel_hf"])
    key, name = "en", "s75"
    p = "%s_%s_" % (key, name)
    mel = mk.vocoder_mel(o1, mk.case_pcm(int(g[p + "chunk"]), name))
    assert np.array_equal(mel[:, ::mk.MEL_KEEP], g[p + "mel"])
    for th in (1, 4):
        o, r = mk.run_case(mk.MODELS[key][0], mel, mk.CLIPS[name][1], th)
        assert np.array_equal(r["tokens"], g[p + "t%d_tokens" % th])
        assert np.array_equal(r["step_logits"][..., ::mk.LOGIT_THIN], g[p + "t%d_step_logits" % th])
        assert np.array_equal(logits_sample(r["prompt_logits"])[..., ::mk.LOGIT_THIN], g[p + "t%d_prompt_logits" % th])
        if th == 1:
            k, v = o.cross_kv()
            assert np.array_equal(k[:, ::mk.ROW_STEP, ::mk.COL_STEP].astype(np.float16), g[p + "cross_k"])
            assert np.array_equal(v[:, ::mk.ROW_STEP, ::mk.COL_STEP].astype(np.float16), g[p + "cross_v"])

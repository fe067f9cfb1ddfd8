"""The per-op decoder attention kernel (attn_decode_kernel, step mode 0) at long self-attention contexts, on an H100.

A prompt pass takes self attention to at most a few dozen keys, and single-token steps past that run the step kernels.  Here the
per-op kernel sees up to the model's 448 text positions: 440 tokens are fed in two calls of at most 256, then 8 tokens at
n_past = 440 return their logits, so the last query attends over all 448 keys (the kernel's second register batch of K starts at
key 384).  The oracle is oracle/whisper_np.NpDecoder on the GPU's own cross-K/V, fed the same three calls: the reference cuts its
threads' key ranges from each call's n_past + N, so the cache rows of later positions depend on how the calls were cut.
"""
import numpy as np
import pytest

from oracle import whisper_np as wn
from tests.test_gpu_audio_ctx import TOL_LOGIT, open_model
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

MODEL = "micro.en-sc"
CALLS = ((0, 256), (256, 440), (440, 448))   # [n_past, end) of each decode call; the last one returns all logits


def feed(c, tokens):
    """The three decode calls; returns the logits of the last one ([8][n_vocab])."""
    for n_past, end in CALLS[:-1]:
        c.decode([tokens[n_past:end]], n_past, 1, capi.DECODE_NO_SAMPLE)
    n_past, end = CALLS[-1]
    c.decode([tokens[n_past:end]], n_past, 1, capi.DECODE_ALL_LOGITS)
    return c.logits(end - n_past)


@pytest.mark.parametrize("threads", [1, 4, 16])
def test_per_op_attention_over_448_keys(threads):
    m, e, c = open_model(MODEL)
    assert m.n_text_ctx == CALLS[-1][1]
    rng = np.random.default_rng(448)
    tokens = [m.special["sot"]] + rng.integers(0, m.special["eot"], CALLS[-1][1] - 1).tolist()
    c.set_reference_threads(threads)
    c.set_step_mode(0)
    try:
        c.pcm_to_mel(0, synth.synth_pcm(7))
        c.encode(1, [0])
        L, H, d = m.n_text_layer, m.n_text_head, m.n_text_state
        ck, cv = (c.get_tensor(nm).reshape(L, H, -1, 64).transpose(0, 2, 1, 3).reshape(L, -1, d) for nm in ("cross_k", "cross_v"))
        got = feed(c, tokens)
    finally:
        c.set_step_mode(2)
        c.set_reference_threads(4)
    dec = wn.NpDecoder(wn.NpModel(synth.model_path(MODEL)), ck, cv, pv_threads=threads)
    for n_past, end in CALLS:
        want, _ = dec.decode(tokens[n_past:end], n_past)
    tol = TOL_LOGIT * max(1.0, float(want.std()) / 3.0)
    err = np.abs(got - want).max(axis=1)
    assert err.max() < tol, "max |logit error| per query row %s, tolerance %.3g" % (np.round(err, 4).tolist(), tol)


def test_reference_threads_outside_1_to_16_are_rejected():
    m, e, c = open_model(MODEL)
    for n in (0, -1, 17):
        with pytest.raises(capi.WspError) as ex:
            c.set_reference_threads(n)
        assert ex.value.status == -1, n     # WSP_E_INVALIDARG
    c.set_reference_threads(4)

"""Speed-up — the reference's 2x phase-vocoder log-mel (whisper_pcm_to_mel_phase_vocoder) — on an H100, through the C ABI.

Oracle: tests/golden/speed_up.npz (outputs of oracle/_ref, the reference's unmodified CPU code, made by
tests/golden/make_speed_up_golden.py).  The mel tolerance is derived from the reference's own f32 FFT round-off
(tests/test_speed_up_fixtures.py::tol_mel); encoder, cross-K/V and logit tolerances are those of tests/test_gpu_parity.py.  Greedy
tokens must be identical.  The batch, switching and default-identity checks compare the GPU with itself, bit for bit.
"""
import os

import numpy as np
import pytest

from tests.golden import make_speed_up_golden as mk
from tests.test_speed_up_fixtures import CASES, tol_mel
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

TOL_ENC, TOL_KV, TOL_LOGIT = 8e-3, 4e-3, 3e-2

_cache = {}


def golden():
    if "g" not in _cache:
        _cache["g"] = np.load(os.path.join(os.path.dirname(__file__), "golden", "speed_up.npz"))
    return _cache["g"]


def open_model(name, batch=1):
    key = (name, batch)
    if key not in _cache:
        m = capi.Model(synth.model_path(name))
        e = _cache.get(("engine", name)) or capi.Engine(m, 0)
        _cache[("engine", name)] = e
        _cache[key] = (m, e, capi.Context(e, batch))
    return _cache[key]


def case_setup(c, key, name, p):
    """speed-up on, the case's mel in slot 0 and its audio_ctx set; returns the mel offset of its window"""
    g = golden()
    c.set_speed_up(1)
    c.set_audio_ctx(mk.AUDIO_CTX_CASE[2] if p.endswith("_n%d_" % mk.AUDIO_CTX_CASE[2]) else 0)
    c.pcm_to_mel(0, mk.case_pcm(int(g[p + "chunk"]), name))
    return mk.CLIPS[name][1]


def reset(c):
    c.set_speed_up(0)
    c.set_audio_ctx(0)
    c.set_step_mode(2)
    c.set_reference_threads(4)


@pytest.mark.parametrize("n", mk.MEL_LENGTHS + ("hf",))
def test_mel(n):
    g = golden()
    m, e, c = open_model("micro.en-sc")
    c.set_speed_up(1)
    try:
        pcm, want = (mk.hf_pcm(), g["mel_hf"]) if n == "hf" else (mk.mel_pcm(n), g["mel_len%d" % n])
        c.pcm_to_mel(0, pcm)
        assert c.L.wsp_mel_len(c.h, 0) == pcm.size // 320
        mel = c.get_mel(0)
        assert mel.shape == want.shape
        if mel.size:
            assert np.array_equal(c.get_tensor("mel"), mel.ravel())
        assert np.abs(mel - want).max(initial=0.0) < tol_mel(g)
    finally:
        reset(c)


@pytest.mark.parametrize("key,name,p", CASES)
def test_encoder_and_cross_kv(key, name, p):
    g = golden()
    m, e, c = open_model(mk.MODELS[key][0])
    d, L, H = m.n_audio_state, m.n_text_layer, m.n_audio_head
    try:
        off = case_setup(c, key, name, p)
        mel = c.get_mel(0)
        assert mel.shape == tuple(g[p + "mel_shape"])
        assert np.abs(mel[:, ::mk.MEL_KEEP] - g[p + "mel"]).max() < tol_mel(g)
        c.encode(1, [off])
        n = c.get_tensor("encode-out").size // d
        gain = synth.SC_ENC_GAIN_CALIBRATED
        assert np.abs(c.get_tensor("encode-out").reshape(n, d)[::mk.ROW_STEP, ::mk.COL_STEP] - g[p + "encode_out"]).max() < TOL_ENC * gain
        for nm in ("cross_k", "cross_v"):
            got = c.get_tensor(nm).reshape(L, H, n, 64).transpose(0, 2, 1, 3).reshape(L, n, d)
            assert np.abs(got[:, ::mk.ROW_STEP, ::mk.COL_STEP] - g[p + nm].astype(np.float32)).max() < TOL_KV * gain
    finally:
        reset(c)


@pytest.mark.parametrize("key,name,p", CASES)
@pytest.mark.parametrize("threads", mk.THREADS)
@pytest.mark.parametrize("mode", [2, 1, 0])
def test_decoder_teacher_forced(key, name, p, threads, mode):
    """Prompt (all-logits path) and every single-token step fed with the reference's own tokens, in each step mode, at reference
    threads 1, 4 and 16: logits within tolerance and every greedy choice identical where the fixture pins the tokens."""
    g = golden()
    q = p + "t%d_" % threads
    pinned = bool(g[p + "tokens_pinned"])
    m, e, c = open_model(mk.MODELS[key][0])
    try:
        off = case_setup(c, key, name, p)
        c.set_reference_threads(threads)
        c.set_step_mode(mode)
        c.encode(1, [off])
        prompt = g[key + "_prompt"].tolist()
        idx = np.arange(0, m.n_vocab, int(g["logit_step"]))
        tol = TOL_LOGIT * max(1.0, float(np.concatenate([g[q + "prompt_logits"].ravel(), g[q + "step_logits"].ravel()]).std()) / 3.0)
        c.decode([prompt], 0, 1, capi.DECODE_ALL_LOGITS)
        assert np.abs(c.logits(len(prompt))[:, idx] - g[q + "prompt_logits"]).max() < tol
        toks = g[q + "tokens"]
        s = c.decode([prompt], 0, 1, capi.DECODE_FORCE_TIMESTAMP | capi.DECODE_INITIAL)[0]
        assert s["id"] == toks[0] or not pinned
        n_past = len(prompt)
        for i in range(1, mk.N_STEPS):
            s = c.decode([[int(toks[i - 1])]], n_past, 1, 0)[0]
            n_past += 1
            assert np.abs(c.logits(1)[0, idx] - g[q + "step_logits"][i - 1]).max() < tol, "step %d" % i
            assert s["id"] == toks[i] or not pinned, "step %d" % i
    finally:
        reset(c)


@pytest.mark.parametrize("key,name,p", CASES)
@pytest.mark.parametrize("threads", mk.THREADS)
@pytest.mark.parametrize("mode", [2, 1, 0])
def test_greedy_free_running(key, name, p, threads, mode):
    """The decoder fed its own choices reproduces the reference's greedy sequence: wsp_run_chunks (tokens fed back on the device, the
    step replayed as a CUDA graph) for clips encoded from frame 0, the host loop for the window at mel offset 1000."""
    g = golden()
    if not g[p + "tokens_pinned"]:
        pytest.skip("no PCM chunk keeps the reference's decisions clear of near-ties on this zero-padded window (see the generator)")
    m, e, c = open_model(mk.MODELS[key][0])
    want = g[p + "t%d_tokens" % threads].tolist()
    prompt = g[key + "_prompt"].tolist()
    try:
        off = case_setup(c, key, name, p)
        c.set_reference_threads(threads)
        c.set_step_mode(mode)
        if off == 0:
            toks, _ = c.run_chunks([mk.case_pcm(int(g[p + "chunk"]), name)], prompt, mk.N_STEPS)
            assert toks[0].tolist() == want
        else:
            c.encode(1, [off])
            got = [c.decode([prompt], 0, 1, capi.DECODE_FORCE_TIMESTAMP | capi.DECODE_INITIAL)[0]["id"]]
            for i in range(1, mk.N_STEPS):
                got.append(c.decode([[got[-1]]], len(prompt) + i - 1, 1, 0)[0]["id"])
            assert got == want
    finally:
        reset(c)


def mixed_clips():
    """8 clips of mixed lengths for micro.en-sc: the three fixture clips encoded from frame 0 and five others (under 1 s to 90 s)"""
    g = golden()
    named = [mk.case_pcm(int(g["en_%s_chunk" % nm]), nm) for nm in ("s60", "s45", "s75")]
    others = [synth.synth_pcm(70 + i, n) for i, n in enumerate((960000, 12000, 1440000, 500000, 640000))]
    return [named[0], others[0], named[1], others[1], named[2], others[2], others[3], others[4]], {0: "s60", 2: "s45", 4: "s75"}


def run_batch(c, pcms, prompt, resident):
    if resident:
        for b, x in enumerate(pcms):
            c.upload_pcm(b, x)
        toks, _ = c.run_chunks_resident(len(pcms), prompt, mk.N_STEPS)
    else:
        toks, _ = c.run_chunks(pcms, prompt, mk.N_STEPS)
    return toks, [c.get_tensor("cross_k", b) for b in range(len(pcms))], [c.get_mel(b) for b in range(len(pcms))]


@pytest.mark.parametrize("resident", [False, True])
def test_batch_of_mixed_clips(resident):
    """wsp_run_chunks / wsp_run_chunks_resident with speed-up on, 8 clips in one batch: the fixture clips give the fixture's tokens, and
    every slot's mel, cross-K memory and tokens are bit-identical to the same clip run alone."""
    g = golden()
    m, e, _ = open_model("micro.en-sc")
    prompt = g["en_prompt"].tolist()
    pcms, named = mixed_clips()
    c = capi.Context(e, 8)
    solo = capi.Context(e, 1)
    try:
        c.set_speed_up(1)
        solo.set_speed_up(1)
        toks, cross, mels = run_batch(c, pcms, prompt, resident)
        for b, nm in named.items():
            if g["en_%s_tokens_pinned" % nm]:
                assert toks[b].tolist() == g["en_%s_t4_tokens" % nm].tolist(), nm
        for b, x in enumerate(pcms):
            t1, k1, m1 = run_batch(solo, [x], prompt, resident)
            assert mels[b].shape == (80, x.size // 320)
            assert np.array_equal(mels[b], m1[0]), b
            assert np.array_equal(cross[b], k1[0]), b
            assert np.array_equal(toks[b], t1[0]), b
    finally:
        c.close()
        solo.close()


def outputs(c, pcms, prompt):
    toks, _ = c.run_chunks(pcms, prompt, 16)
    c.pcm_to_mel(0, pcms[0])
    return toks, c.logits(len(pcms)), c.get_tensor("cross_k", len(pcms) - 1), c.get_mel(0)


def test_switching_back_and_default_are_identity():
    """A context switched on, used, and switched off computes bit for bit what a fresh context computes; wsp_set_speed_up(c, 0) is the
    same as never calling it; and a context switched on equals a fresh one switched on."""
    m, e, _ = open_model("micro.en-sc")
    prompt = m.prompt_init()
    pcms = [synth.synth_pcm(50 + i, 480000 + 160000 * i) for i in range(3)]
    fresh, zero, used, on = (capi.Context(e, 4) for _ in range(4))
    try:
        want = outputs(fresh, pcms, prompt)
        zero.set_speed_up(0)
        got_zero = outputs(zero, pcms, prompt)
        used.set_speed_up(1)
        got_on = outputs(used, pcms, prompt)
        used.set_speed_up(0)
        got_off = outputs(used, pcms, prompt)
        on.set_speed_up(True)
        want_on = outputs(on, pcms, prompt)
        for a, b, x, y, z in zip(want, got_zero, got_off, got_on, want_on):
            assert np.array_equal(a, b) and np.array_equal(a, x)
            assert np.array_equal(y, z)
        assert got_on[3].shape[1] == pcms[0].size // 320 and want[3].shape[1] == pcms[0].size // 160
    finally:
        for c in (fresh, zero, used, on):
            c.close()


def test_invalid_values_and_streamed_window():
    m, e, _ = open_model("micro.en-sc")
    c = capi.Context(e, 1)
    ref = capi.Context(e, 1)
    try:
        for bad in (2, -1, 320):
            with pytest.raises(capi.WspError) as ex:
                c.set_speed_up(bad)
            assert ex.value.status == -1
        pcm = synth.synth_pcm(4, 160000 + 240)
        c.set_speed_up(1)
        with pytest.raises(capi.WspError) as ex:
            c.pcm_to_mel_window(0, pcm, 1000)
        assert ex.value.status == -8        # WSP_E_NOTIMPL
        c.set_mel(0, np.zeros((80, 100), np.float32))   # unaffected by the setting
        assert c.get_mel(0).shape == (80, 100)
        c.set_speed_up(0)
        mx = c.pcm_to_mel_window(0, pcm, 1000)
        assert mx == ref.pcm_to_mel_window(0, pcm, 1000)
        assert np.array_equal(c.get_mel(0), ref.get_mel(0))
    finally:
        c.close()
        ref.close()


def test_language_detection():
    """whisper_lang_auto_detect on the phase-vocoder mel of three 60 s clips (micro-sc): the language id and probabilities."""
    g = golden()
    m, e, c = open_model("micro-sc")
    c.set_speed_up(1)
    try:
        for i, ch in enumerate(g["lang_chunks"].tolist()):
            c.pcm_to_mel(0, synth.synth_pcm(ch, 960000))
            lid, probs = c.detect_language(0, g["lang_probs"].shape[1])
            assert lid == int(g["lang_id"][i])
            assert np.abs(probs - g["lang_probs"][i]).max() < 2e-4
    finally:
        reset(c)

"""sFullParams::audio_ctx — the shortened encoder context — on an H100, through the C ABI and the COM-style surface.

Oracle: tests/golden/audio_ctx.npz (outputs of oracle/_ref, the reference's unmodified CPU code, made by
tests/golden/make_audio_ctx_golden.py).  Tolerances are those of DESIGN.md §2 (tests/test_gpu_parity.py); greedy tokens must be
identical wherever the fixture pins them.  The stale-state and default-identity checks compare the GPU with itself, bit for bit.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests.golden.make_audio_ctx_golden import AUDIO_CTX, COL_STEP, FULL_RUNS, MODELS, N_STEPS, THREADS, rows_of
from tests.golden.make_golden import full_pcm
from tests.test_gpu_com import _lib, capture_signal
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

TOL_ENC, TOL_KV, TOL_LOGIT = 8e-3, 4e-3, 3e-2
TOL_INPUT = 1e-3      # the encoder's input window is the f16-rounded log-mel (values in [-1.5, 1.5]) + the mel tolerance 5e-4
E_INVALIDARG = 0x80070057

_cache = {}


def golden():
    if "g" not in _cache:
        _cache["g"] = np.load(os.path.join(os.path.dirname(__file__), "golden", "audio_ctx.npz"))
    return _cache["g"]


def open_model(name, batch=1):
    key = (name, batch)
    if key not in _cache:
        m = capi.Model(synth.model_path(name))
        e = _cache.get(("engine", name)) or capi.Engine(m, 0)
        _cache[("engine", name)] = e
        _cache[key] = (m, e, capi.Context(e, batch))
    return _cache[key]


CASES = [(key, n) for key in MODELS for n in AUDIO_CTX]


def case_pcm(key, n):
    return synth.synth_pcm(int(golden()["%s_n%d_chunk" % (key, n)]), 480000)


@pytest.mark.parametrize("key,n", CASES)
def test_encoder_and_cross_kv(key, n):
    """The 2n-frame input window, conv1, the input of layer 0, ln_post and the cross-K/V memories (n rows per layer) against the
    reference's trace points at that audio_ctx; the tensor shapes follow the last encode."""
    g = golden()
    p = "%s_n%d_" % (key, n)
    m, e, c = open_model(MODELS[key][0])
    d, L, H = m.n_audio_state, m.n_text_layer, m.n_audio_head
    r1, r2 = rows_of(n), rows_of(2 * n)
    c.pcm_to_mel(0, case_pcm(key, n))
    c.set_audio_ctx(n)
    try:
        c.set_encoder_layers(0)
        c.encode(1, [0])
        assert c.get_tensor("enc.input").size == 2 * n * 80
        assert np.abs(c.get_tensor("enc.input").reshape(2 * n, 80)[r2, ::COL_STEP] - g[p + "enc_input"]).max() < TOL_INPUT
        assert np.abs(c.get_tensor("enc.conv1").reshape(2 * n, d)[r2, ::COL_STEP] - g[p + "enc_temp1"]).max() < TOL_ENC
        assert np.abs(c.get_tensor("enc.x").reshape(n, d)[r1, ::COL_STEP] - g[p + "enc_layer0_in"]).max() < TOL_ENC
        c.set_encoder_layers(-1)
        c.encode(1, [0])
        gain = synth.SC_ENC_GAIN_CALIBRATED
        assert np.abs(c.get_tensor("encode-out").reshape(n, d)[r1, ::COL_STEP] - g[p + "encode_out"]).max() < TOL_ENC * gain
        for nm in ("cross_k", "cross_v"):
            got = c.get_tensor(nm).reshape(L, H, n, 64).transpose(0, 2, 1, 3).reshape(L, n, d)
            assert np.abs(got[:, r1, ::COL_STEP] - g[p + nm].astype(np.float32)).max() < TOL_KV * gain
    finally:
        c.set_encoder_layers(-1)
        c.set_audio_ctx(0)


@pytest.mark.parametrize("key,n", CASES)
@pytest.mark.parametrize("threads", THREADS)
@pytest.mark.parametrize("mode", [2, 1, 0])
def test_decoder_teacher_forced(key, n, threads, mode):
    """Prompt (all-logits path) and every single-token step fed with the reference's own tokens, in each step mode (2 = dataflow kernel,
    1 = barrier kernel, 0 = one kernel per op), at reference threads 1, 4 and 16 — at n = 100 the last of 16 threads owns no key."""
    g = golden()
    p = "%s_n%d_t%d_" % (key, n, threads)
    pinned = bool(g["%s_n%d_tokens_pinned" % (key, n)])
    m, e, c = open_model(MODELS[key][0])
    c.set_reference_threads(threads)
    c.set_step_mode(mode)
    try:
        c.pcm_to_mel(0, case_pcm(key, n))
        c.set_audio_ctx(n)
        c.encode(1, [0])
        prompt = g[key + "_prompt"].tolist()
        idx = np.arange(0, m.n_vocab, int(g["logit_step"]))
        c.decode([prompt], 0, 1, capi.DECODE_ALL_LOGITS)
        want = g[p + "prompt_logits"]
        # logits of rms ~3 on the script; at n = 16 the .en model's run at rms ~19 (the reference's own differ from thread count to
        # thread count by the f16 rounding of activations that large): the tolerance scales with the rms, as for make_golden's padded case
        tol = TOL_LOGIT * max(1.0, float(np.concatenate([want.ravel(), g[p + "step_logits"].ravel()]).std()) / 3.0)
        assert np.abs(c.logits(len(prompt))[:, idx] - want).max() < tol
        toks = g[p + "tokens"]
        s = c.decode([prompt], 0, 1, capi.DECODE_FORCE_TIMESTAMP | capi.DECODE_INITIAL)[0]
        if pinned:
            assert s["id"] == toks[0]
        n_past = len(prompt)
        for i in range(1, N_STEPS):
            s = c.decode([[int(toks[i - 1])]], n_past, 1, 0)[0]
            n_past += 1
            assert np.abs(c.logits(1)[0, idx] - g[p + "step_logits"][i - 1]).max() < tol, "step %d" % i
            if pinned:
                assert s["id"] == toks[i], "step %d" % i
    finally:
        c.set_step_mode(2)
        c.set_reference_threads(4)
        c.set_audio_ctx(0)


@pytest.mark.parametrize("key,n", CASES)
@pytest.mark.parametrize("threads", THREADS)
@pytest.mark.parametrize("mode", [2, 1, 0])
def test_greedy_free_running(key, n, threads, mode):
    """wsp_run_chunks (tokens fed back on the device, the step replayed as a CUDA graph) reproduces the reference's greedy sequence."""
    g = golden()
    if not g["%s_n%d_tokens_pinned" % (key, n)]:
        pytest.skip("no PCM chunk keeps the reference's decisions clear of near-ties at this audio_ctx (see the generator)")
    m, e, c = open_model(MODELS[key][0])
    c.set_reference_threads(threads)
    c.set_step_mode(mode)
    c.set_audio_ctx(n)
    try:
        toks, _ = c.run_chunks([case_pcm(key, n)], g[key + "_prompt"].tolist(), N_STEPS)
        assert toks[0].tolist() == g["%s_n%d_t%d_tokens" % (key, n, threads)].tolist()
    finally:
        c.set_step_mode(2)
        c.set_reference_threads(4)
        c.set_audio_ctx(0)


# ---- the COM-style surface: runFull, runStreamed, runCapture -------------------------------------------------------------------
SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "audio_ctx_shim", "_build", "libwsac_test.so")


def shim():
    capi.lib()                       # the product library (the shim links against it)
    if not os.path.exists(SHIM):
        pytest.fail("tests/audio_ctx_shim/_build/libwsac_test.so is missing: run __graft_entry__.build()")
    L = C.CDLL(SHIM)
    vp, i32, fp = C.c_void_p, C.c_int32, C.POINTER(C.c_float)
    L.wsac_open.restype = i32; L.wsac_open.argtypes = [C.c_char_p, i32, C.POINTER(vp)]
    L.wsac_close.argtypes = [vp]
    L.wsac_run.restype = i32
    L.wsac_run.argtypes = [vp, i32, fp, i32, C.c_uint32, C.c_char_p, i32, i32, i32, i32, i32, i32]
    L.wsac_run_capture.restype = i32
    L.wsac_run_capture.argtypes = [vp, fp, i32, C.c_uint32, C.c_char_p, i32, C.c_float, C.c_float, i32, C.POINTER(i32)]
    L.wsac_n_segments.restype = i32; L.wsac_n_segments.argtypes = [vp]
    for f in ("wsac_segment_t0", "wsac_segment_t1"):
        getattr(L, f).restype = C.c_int64; getattr(L, f).argtypes = [vp, i32]
    L.wsac_segment_n_tokens.restype = i32; L.wsac_segment_n_tokens.argtypes = [vp, i32]
    L.wsac_token.restype = i32; L.wsac_token.argtypes = [vp, i32, i32]
    return L


def segments(L, h):
    """[(t0, t1) in 100 ns ticks, tokens] of the session's last run"""
    return [dict(t0=L.wsac_segment_t0(h, i), t1=L.wsac_segment_t1(h, i), tokens=[L.wsac_token(h, i, j) for j in range(L.wsac_segment_n_tokens(h, i))])
            for i in range(L.wsac_n_segments(h))]


@pytest.fixture
def fresh():
    """A session of its own per test: audio_ctx is context state that outlives a call, so no other test's context is touched."""
    L = shim()
    opened = []

    def open_(model):
        h = C.c_void_p()
        hr = L.wsac_open(synth.model_path(model).encode(), 0, C.byref(h))
        assert hr == 0, hex(hr & 0xFFFFFFFF)
        opened.append(h)
        return h

    yield L, open_
    for h in opened:
        L.wsac_close(h)


def full_call(L, h, pcm, flags, lang, max_tokens, off, dur, audio_ctx, streamed=False, max_block=4096):
    hr = L.wsac_run(h, int(streamed), pcm.ctypes.data_as(C.POINTER(C.c_float)), pcm.size, flags, lang, max_tokens, 4, off, dur, audio_ctx, max_block)
    return hr, (segments(L, h) if hr >= 0 else [])


@pytest.mark.parametrize("name", list(FULL_RUNS))
@pytest.mark.parametrize("streamed", [False, True])
def test_whisper_full_runs(fresh, name, streamed):
    """whisper_full at audio_ctx 750 / 384 (with offset and max_tokens), and on the multilingual model "de" at 750 followed by "auto"
    at 0 on the same context: the second call detects the language with the FIRST call's audio_ctx, as whisper_full does
    (whisper.cpp:2789-2801 before :2836).  runStreamed reads the clip in ragged blocks (DESIGN.md §7 on its per-window mel)."""
    g = golden()
    L, open_ = fresh
    model, flags, max_tokens, off, dur, calls = FULL_RUNS[name]
    h = open_(model)
    pcm = np.ascontiguousarray(full_pcm(int(g[name + "_pcm_base"])), np.float32)
    for lang, actx in calls:
        hr, segs = full_call(L, h, pcm, flags, lang.encode(), max_tokens, off, dur, actx, streamed, max_block=977)
        assert hr == 0
    assert [[s["t0"] // 100000, s["t1"] // 100000] for s in segs] == g[name + "_t"].tolist()     # fixture times: 10 ms units
    assert [len(s["tokens"]) for s in segs] == g[name + "_ntok"].tolist()
    assert [t for s in segs for t in s["tokens"]] == g[name + "_tokens"].tolist()


def test_run_capture_with_audio_ctx(fresh):
    """runCapture hands audio_ctx to the runFull of every utterance: the segments equal runFull's on the same cuts."""
    L, open_ = fresh
    cuts = _lib()                     # where the capture loop cuts (host code, the existing boundary-test helpers)
    h = open_("micro.en-sc1")
    x = np.ascontiguousarray(capture_signal(), np.float32)
    xp = x.ctypes.data_as(C.POINTER(C.c_float))
    starts, sizes = (C.c_int64 * 16)(), (C.c_int32 * 16)()
    n_cuts = cuts.wspc_capture_cuts(xp, x.size, 20.0, 29.5, starts, sizes, 16)
    assert n_cuts == 2
    info = (C.c_int32 * 2)()
    assert L.wsac_run_capture(h, xp, x.size, 2, b"en", 4, 20.0, 29.5, 750, info) == 0
    assert info[1] == x.size
    got = [(s["t0"], s["t1"], s["tokens"]) for s in segments(L, h)]
    want = []
    for k in range(n_cuts):
        seg = np.ascontiguousarray(x[starts[k]:starts[k] + sizes[k]])
        hr, segs = full_call(L, h, seg, 2, b"en", 0, 0, 0, 750)
        assert hr == 0
        offset = starts[k] * 10000000 // 16000
        want += [(s["t0"] + offset, s["t1"] + offset, s["tokens"]) for s in segs]
    assert len(want) >= 4
    assert got == want


def test_audio_ctx_above_the_model_is_rejected(fresh):
    L, open_ = fresh
    h = open_("micro.en-sc1")
    pcm = np.ascontiguousarray(full_pcm(10)[:16000 * 20], np.float32)
    for streamed in (False, True):
        hr, _ = full_call(L, h, pcm, 2, b"en", 0, 0, 0, 1501, streamed)
        assert (hr & 0xFFFFFFFF) == E_INVALIDARG
    hr, segs = full_call(L, h, pcm, 2, b"en", 0, 0, 0, -5)        # <= 0: the model's default, as in the reference
    assert hr == 0 and segs
    m, e, c = open_model("micro.en-sc")
    with pytest.raises(capi.WspError) as ex:
        c.set_audio_ctx(1501)
    assert ex.value.status == -1


def run_setting(c, pcms, n, prompt, steps=16):
    c.set_audio_ctx(n)
    toks, _ = c.run_chunks(pcms, prompt, steps)
    return toks, c.logits(len(pcms)), c.get_tensor("encode-out", len(pcms) - 1)


def test_no_stale_state_between_settings():
    """One context runs n = 100, 1500, 129 at batch 8 and then 129 at batch 3, with CUDA graphs on; every result is bit-identical to a
    fresh context's.  Halo rows of the packed encoder input, V^T pad columns and the captured step graph all depend on n."""
    m, e, _ = open_model("micro.en-sc")
    prompt = m.prompt_init()
    pcms = [synth.synth_pcm(40 + i, 480000 - 8000 * i) for i in range(8)]
    used = capi.Context(e, 8)
    try:
        for n, b in ((100, 8), (1500, 8), (129, 8), (129, 3)):
            got = run_setting(used, pcms[:b], n, prompt)
            ref = capi.Context(e, 8)
            try:
                want = run_setting(ref, pcms[:b], n, prompt)
            finally:
                ref.close()
            for a, w in zip(got, want):
                assert np.array_equal(a, w), "n = %d, batch %d" % (n, b)
    finally:
        used.close()


def test_default_setting_is_identity():
    """wsp_set_audio_ctx(c, 0) and (c, 1500) compute exactly what a context that never called it computes."""
    m, e, _ = open_model("micro.en-sc")
    prompt = m.prompt_init()
    pcms = [synth.synth_pcm(50 + i) for i in range(3)]
    outs = []
    for n in (None, 0, 1500):
        c = capi.Context(e, 4)
        try:
            if n is not None:
                c.set_audio_ctx(n)
            toks, _ = c.run_chunks(pcms, prompt, 16)
            outs.append((toks, c.logits(3), c.get_tensor("cross_k", 2)))
        finally:
            c.close()
    for o in outs[1:]:
        for a, w in zip(o, outs[0]):
            assert np.array_equal(a, w)

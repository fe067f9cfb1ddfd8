"""The COM-style drop-in surface (include/whisper_b200_com.h) on an H100: loadModel -> createContext -> fullDefaultParams -> runFull ->
getResults, exactly the call sequence of the reference's CLI (Examples/main/main.cpp:210-318), driven through the flat wspc_*
helpers (ctypes cannot call C++ vtables).  The transcription driver is compared with the reference's whisper_full()
(Whisper/source/whisper.cpp:2765-3125) via fixtures generated from oracle/_ref (tests/golden/full_runs.npz, scripted models)."""
import ctypes as C
import os

import numpy as np
import pytest

from tests.golden.make_golden import FULL_MAX_LEN, FULL_MODEL, FULL_RUNS, full_pcm
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu


SHIM = os.path.join(os.path.dirname(os.path.abspath(__file__)), "boundary", "_build", "libwspc_test.so")


def _lib():
    capi.lib()                       # the product library (the shim links against it)
    if not os.path.exists(SHIM):
        pytest.fail("tests/boundary/_build/libwspc_test.so is missing: run __graft_entry__.build()")
    L = C.CDLL(SHIM)
    vp, i32 = C.c_void_p, C.c_int32
    L.wspc_open.restype = i32; L.wspc_open.argtypes = [C.c_char_p, i32, C.POINTER(vp)]
    L.wspc_close.argtypes = [vp]
    L.wspc_run_full.restype = i32
    L.wspc_run_full.argtypes = [vp, C.POINTER(C.c_float), i32, C.c_uint32, C.c_char_p, i32, i32, i32, i32, C.POINTER(i32), i32]
    for f in ("wspc_n_segments", "wspc_n_segment_callbacks", "wspc_is_multilingual", "wspc_query_interfaces"):
        getattr(L, f).restype = i32; getattr(L, f).argtypes = [vp]
    for f in ("wspc_segment_t0", "wspc_segment_t1"):
        getattr(L, f).restype = C.c_int64; getattr(L, f).argtypes = [vp, i32]
    L.wspc_segment_text.restype = C.c_char_p; L.wspc_segment_text.argtypes = [vp, i32]
    L.wspc_segment_n_tokens.restype = i32; L.wspc_segment_n_tokens.argtypes = [vp, i32]
    L.wspc_token_id.restype = i32; L.wspc_token_id.argtypes = [vp, i32, i32]
    L.wspc_token_p.restype = C.c_float; L.wspc_token_p.argtypes = [vp, i32, i32]
    L.wspc_token_flags.restype = i32; L.wspc_token_flags.argtypes = [vp, i32, i32]
    L.wspc_tokenize.restype = i32; L.wspc_tokenize.argtypes = [vp, C.c_char_p, C.POINTER(i32), i32]
    L.wspc_string_from_token.restype = C.c_char_p; L.wspc_string_from_token.argtypes = [vp, i32]
    L.wspc_special_tokens.restype = i32; L.wspc_special_tokens.argtypes = [vp, C.POINTER(i32)]
    L.wspc_run_streamed.restype = i32
    L.wspc_run_streamed.argtypes = [vp, C.POINTER(C.c_float), i32, C.c_uint32, C.c_char_p, i32, i32, i32, i32, i32, C.POINTER(i32)]
    L.wspc_run_capture.restype = i32
    L.wspc_run_capture.argtypes = [vp, C.POINTER(C.c_float), i32, C.c_uint32, C.c_char_p, i32, C.c_float, C.c_float, C.POINTER(i32)]
    L.wspc_capture_cuts.restype = i32
    L.wspc_capture_cuts.argtypes = [C.POINTER(C.c_float), i32, C.c_float, C.c_float, C.POINTER(C.c_int64), C.POINTER(i32), i32]
    for f in ("wspc_captured_t0", "wspc_captured_t1"):
        getattr(L, f).restype = C.c_int64; getattr(L, f).argtypes = [vp, i32]
    L.wspc_captured_text.restype = C.c_char_p; L.wspc_captured_text.argtypes = [vp, i32]
    L.wspc_captured_n_tokens.restype = i32; L.wspc_captured_n_tokens.argtypes = [vp, i32]
    L.wspc_captured_token.restype = i32; L.wspc_captured_token.argtypes = [vp, i32, i32]
    L.wspc_run_full_stereo.restype = i32
    L.wspc_run_full_stereo.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float), i32, C.c_uint32, i32, C.POINTER(i32), i32, C.POINTER(i32)]
    L.wspc_set_max_len.argtypes = [vp, i32]
    for f in ("wspc_token_t0", "wspc_token_t1"):
        getattr(L, f).restype = C.c_int64; getattr(L, f).argtypes = [vp, i32, i32]
    L.wspc_segment_callback_total.restype = i32; L.wspc_segment_callback_total.argtypes = [vp]
    L.wspc_find_language_key.restype = C.c_uint32; L.wspc_find_language_key.argtypes = [C.c_char_p]
    L.wspc_language_count.restype = i32
    return L


_sessions = {}


def open_session(model):
    L = _lib()
    if model not in _sessions:
        h = C.c_void_p()
        hr = L.wspc_open(synth.model_path(model).encode(), 0, C.byref(h))
        assert hr == 0, hex(hr & 0xFFFFFFFF)
        _sessions[model] = h
    return L, _sessions[model]


@pytest.fixture(scope="module")
def session():
    yield open_session(FULL_MODEL)
    L = _lib()
    for h in _sessions.values():
        L.wspc_close(h)
    _sessions.clear()


def run_full(L, h, pcm, flags=0, language=b"en", max_tokens=0, threads=4, off=0, dur=0, prompt=None, max_len=0):
    pcm = np.ascontiguousarray(pcm, np.float32)
    pt = None if prompt is None else np.ascontiguousarray(prompt, np.int32)
    L.wspc_set_max_len(h, max_len)
    hr = L.wspc_run_full(h, pcm.ctypes.data_as(C.POINTER(C.c_float)), pcm.size, flags, language, max_tokens, threads, off, dur,
                         None if pt is None else pt.ctypes.data_as(C.POINTER(C.c_int32)), 0 if pt is None else pt.size)
    segs = []
    for i in range(L.wspc_n_segments(h)):
        n = L.wspc_segment_n_tokens(h, i)
        segs.append(dict(t0=L.wspc_segment_t0(h, i), t1=L.wspc_segment_t1(h, i), text=L.wspc_segment_text(h, i).decode(errors="replace"),
                         tokens=[L.wspc_token_id(h, i, j) for j in range(n)], flags=[L.wspc_token_flags(h, i, j) for j in range(n)],
                         token_t=[[L.wspc_token_t0(h, i, j), L.wspc_token_t1(h, i, j)] for j in range(n)]))
    return hr, segs


def _segments(L, h):
    segs = []
    for i in range(L.wspc_n_segments(h)):
        n = L.wspc_segment_n_tokens(h, i)
        segs.append(dict(t0=L.wspc_segment_t0(h, i), t1=L.wspc_segment_t1(h, i), text=L.wspc_segment_text(h, i).decode(errors="replace"),
                         tokens=[L.wspc_token_id(h, i, j) for j in range(n)]))
    return segs


def run_streamed(L, h, pcm, flags=0, language=b"en", max_tokens=0, threads=4, off=0, dur=0, max_block=4096):
    pcm = np.ascontiguousarray(pcm, np.float32)
    info = (C.c_int32 * 3)()
    hr = L.wspc_run_streamed(h, pcm.ctypes.data_as(C.POINTER(C.c_float)), pcm.size, flags, language, max_tokens, threads, off, dur, max_block, info)
    return hr, (_segments(L, h) if hr >= 0 else []), list(info)


# iContext::runStreamed (ContextImpl.misc.cpp:391-419) runs the loop of runFull over a spectrogram that is produced window by window from a
# pull source and normalised per window (MelStreamer.cpp:128-170).  The reference has no CPU implementation of it to generate fixtures
# from; but on these clips a window's own maximum and the clip's differ by < 0.003 and only the ~10 of 240 000 values per window that sit
# more than 8 below the maximum see the difference (checked on the CPU: test_oracle-side numbers in DESIGN.md §7), four orders of magnitude
# below the fixtures' decision margins — so the streamed transcript must be the whisper_full fixture's.
@pytest.mark.parametrize("name", ["plain", "special_offset_duration", "ml_german", "special_nocontext_max40"])
def test_run_streamed_matches_reference_driver(name):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "full_runs.npz"))
    model, flags, max_tokens, off, dur, lang, calls = FULL_RUNS[name]
    assert calls == 1
    L, h = open_session(model)
    pcm = full_pcm(int(g[name + "_pcm_base"]))
    hr, segs, info = run_streamed(L, h, pcm, flags=flags | 2, language=lang.encode(), max_tokens=max_tokens, off=off, dur=dur,
                                  max_block={"plain": 4096, "special_offset_duration": 977, "ml_german": 16000, "special_nocontext_max40": 50000}[name])
    assert hr == 0
    assert [[s["t0"], s["t1"]] for s in segs] == g[name + "_t"].tolist()
    assert [t for s in segs for t in s["tokens"]] == g[name + "_tokens"].tolist()
    assert [s["text"] for s in segs] == g[name + "_text"].tolist()
    assert L.wspc_segment_callback_total(h) == len(segs)
    # progress sink: called at the top of every window and once with 1.0 at the end (ContextImpl.cpp:533-540, 788-792), never decreasing
    assert info[0] >= 3 and info[1] == 1
    # the source was read sequentially to (about) where the last window ended, not slurped: every read returned <= max_block samples
    assert info[2] > 10


def test_run_streamed_without_reader_thread_and_rules(session):
    """cpuThreads = 1 selects the on-demand reader (MelStreamerSimple) — and the 1-thread reference arithmetic — so the comparison is
    runStreamed against runFull on this GPU; TokenTimestamps is refused in streaming mode, a clip under one second is a no-op."""
    L, h = session
    pcm = full_pcm(10)[:16000 * 47]
    hr, want = run_full(L, h, pcm, flags=2, threads=1)
    assert hr == 0 and len(want) > 5
    hr, segs, info = run_streamed(L, h, pcm, flags=2, threads=1, max_block=12345)
    assert hr == 0 and info[1] == 1
    assert [(s["t0"], s["t1"], s["text"], s["tokens"]) for s in segs] == [(s["t0"], s["t1"], s["text"], s["tokens"]) for s in want]
    hr, _, _ = run_streamed(L, h, pcm, flags=2 | 0x100)
    assert (hr & 0xFFFFFFFF) == 0x80004001                     # E_NOTIMPL (ContextImpl.misc.cpp:393-397)
    hr, segs, _ = run_streamed(L, h, pcm[:8000], flags=2)
    assert hr == 0 and segs == []
    # language = auto on the multilingual model: the first window is made for the detection pass, then again for the loop
    from tests.golden.make_golden import FULL_MODEL_ML
    Lm, hm = open_session(FULL_MODEL_ML)
    hr, want = run_full(Lm, hm, pcm, flags=2, language=b"auto")
    assert hr == 0 and len(want) > 5
    hr, segs, _ = run_streamed(Lm, hm, pcm, flags=2, language=b"auto", max_block=3333)
    assert hr == 0
    assert [(s["t0"], s["t1"], s["text"], s["tokens"]) for s in segs] == [(s["t0"], s["t1"], s["text"], s["tokens"]) for s in want]


def test_detect_speaker_from_the_segment_callback(session):
    """iContext::detectSpeaker (ContextImpl.diarize.cpp:75-112): per-channel sum of |sample| over a segment's interval of the stereo
    samples that came with the clip, a channel wins when it exceeds 1.1 x the other; only answers while a run is in progress."""
    L, h = session
    mono = full_pcm(10)[:16000 * 40]
    t = np.arange(mono.size) / 16000.0
    # left loud for 2 s, right loud for 2 s, balanced for 2 s, ...; (left + right) / 2 stays the mono mix
    phase = (t // 2).astype(np.int64) % 3
    g_left = np.choose(phase, [1.6, 0.4, 1.0]).astype(np.float32)
    stereo = np.empty(2 * mono.size, np.float32)
    stereo[0::2] = mono * g_left
    stereo[1::2] = mono * (2.0 - g_left)
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    speakers, after = (C.c_int32 * 64)(), C.c_int32(0)
    n = L.wspc_run_full_stereo(h, fp(mono), fp(stereo), mono.size, 2, 32000, speakers, 64, C.byref(after))
    assert n >= 8
    segs = _segments(L, h)
    assert len(segs) == n
    want = []
    for s in segs:
        a, b = s["t0"] * 160, s["t1"] * 160
        left, right = np.abs(stereo[2 * a:2 * b:2]).sum(dtype=np.float64), np.abs(stereo[2 * a + 1:2 * b:2]).sum(dtype=np.float64)
        want.append((1 if left > 1.1 * right else 0) | (2 if right > 1.1 * left else 0))
    assert list(speakers)[:n] == want and {1, 2} <= set(want)          # Left = 1, Right = 2, Unsure = 0 (TranscribeStructs.h)
    assert (after.value & 0xFFFFFFFF) == 0x80040007                    # OLE_E_BLANK outside the callbacks
    # a mono-only buffer: NoStereoData
    n2 = L.wspc_run_full_stereo(h, fp(mono), None, mono.size, 2, 32000, speakers, 64, None)
    assert n2 == n and set(list(speakers)[:n2]) == {0xFF}


def capture_signal():
    """64 s "live" signal: two stretches of audio from the family the scripted test models are calibrated on (29 s and 28 s — they only
    emit timestamped text when most of a 30 s window holds such audio), separated by a faint 60 Hz hum.  The hum matters: the voice
    detector compares each frame's dominant frequency with the floor it learned while nobody spoke, and white noise has no stable one."""
    rng = np.random.default_rng(3)

    def hum(seconds):
        n = int(16000 * seconds)
        t = np.arange(n) / 16000.0
        return (0.002 * np.sin(2 * np.pi * 60 * t) + 0.0002 * rng.uniform(-1, 1, n)).astype(np.float32)

    return np.concatenate([hum(1.0), synth.synth_pcm(10)[:16000 * 29], hum(3.0), synth.synth_pcm(11)[:16000 * 28], hum(3.0)])


def test_run_capture_transcribes_the_detected_utterances(session):
    """iContext::runCapture (ContextImpl.capture.cpp:392-429) on a live source played from an array: the listening loop cuts utterances
    with the voice detector (both pinned on the CPU: tests/test_vad.py, tests/boundary/capture_test.cpp) and transcribes each on its
    background thread; the segments delivered through new_segment_callback must be those of runFull on exactly those slices, shifted by
    the utterance's position in the stream (iAudioBuffer::getTime -> mediaTimeOffset, ContextImpl.misc.cpp:264-286)."""
    L, h = session
    x = capture_signal()
    xp = x.ctypes.data_as(C.POINTER(C.c_float))
    starts, sizes = (C.c_int64 * 16)(), (C.c_int32 * 16)()
    n_cuts = L.wspc_capture_cuts(xp, x.size, 20.0, 29.5, starts, sizes, 16)
    assert n_cuts == 2 and all(sizes[k] > 16000 * 28 for k in range(2))
    info = (C.c_int32 * 4)()
    hr = L.wspc_run_capture(h, xp, x.size, 2, b"en", 4, 20.0, 29.5, info)          # NoContext: every utterance starts from a clean prompt
    assert hr == 0
    assert info[1] == n_cuts and info[2] == 0 and info[3] == x.size
    got = [(L.wspc_captured_t0(h, i), L.wspc_captured_t1(h, i), L.wspc_captured_text(h, i).decode(errors="replace"),
            [L.wspc_captured_token(h, i, j) for j in range(L.wspc_captured_n_tokens(h, i))]) for i in range(info[0])]
    want = []
    for k in range(n_cuts):
        hr, segs = run_full(L, h, x[starts[k]:starts[k] + sizes[k]], flags=2)
        assert hr == 0
        offset = starts[k] * 10000000 // 16000
        want += [(s["t0"] * 100000 + offset, s["t1"] * 100000 + offset, s["text"], s["tokens"]) for s in segs]
    assert len(want) >= 8 and want[-1][0] > starts[1] * 625          # both utterances produced timestamped text
    assert got == want
    # parameter validation (ContextImpl.capture.cpp:397-411) and a NULL capture object
    assert (L.wspc_run_capture(h, xp, x.size, 2, b"en", 4, 0.05, 3.0, info) & 0xFFFFFFFF) == 0x80070057
    assert (L.wspc_run_capture(h, xp, x.size, 2, b"en", 4, 2.0, 31.0, info) & 0xFFFFFFFF) == 0x80070057


@pytest.mark.parametrize("name", list(FULL_RUNS))
def test_run_full_matches_reference_driver(session, name):
    """whisper_full on 78 s of audio per case: window seeking from timestamp tokens, prompt carry-over between windows (and, for
    `context_second_call`, between two runFull calls on one context), segment splitting, eFullParamsFlags, language / task tokens of the
    multilingual model, token-level timestamps and max_len wrapping — segments, tokens, texts and token times equal to the reference's."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "full_runs.npz"))
    model, flags, max_tokens, off, dur, lang, calls = FULL_RUNS[name]
    L, h = open_session(model)
    pcm = full_pcm(int(g[name + "_pcm_base"]))
    kw = dict(language=lang.encode(), max_tokens=max_tokens, off=off, dur=dur, max_len=FULL_MAX_LEN.get(name, 0))
    # the fixture ran on a fresh context: NoContext on the first call clears what earlier cases left in this session's context
    hr, segs = run_full(L, h, pcm, flags=flags | 2, **kw)
    if calls == 2:
        assert hr == 0
        hr, segs = run_full(L, h, pcm, flags=flags, **kw)      # second call WITHOUT NoContext: starts from the first call's text (whisper.cpp:2850-2861)
    assert hr == 0
    ref_t = g[name + "_t"]
    assert len(segs) == len(ref_t)
    assert [[s["t0"], s["t1"]] for s in segs] == ref_t.tolist()
    assert [len(s["tokens"]) for s in segs] == g[name + "_ntok"].tolist()
    assert [t for s in segs for t in s["tokens"]] == g[name + "_tokens"].tolist()
    assert [s["text"] for s in segs] == g[name + "_text"].tolist()
    assert L.wspc_segment_callback_total(h) == len(segs)  # new_segment_callback reports every segment (n_new > 1 after a wrap)
    eot = 50257 if model.startswith("micro-") else 50256
    for s in segs:                                        # eTokenFlags::Special <=> id >= eot (convertThings.cpp:200-203)
        assert s["flags"] == [1 if t >= eot else 0 for t in s["tokens"]]
    if flags & 0x100:
        assert [t for s in segs for t in s["token_t"]] == g[name + "_token_t"].tolist()
    else:
        assert all(t == [-1, -1] for s in segs for t in s["token_t"])       # not computed: whisper_token_data's initial -1 (whisper.cpp:1880)


def test_language_auto_detect_matches_reference():
    """whisper_lang_auto_detect (whisper.cpp:2428-2495): encode, decode [sot], the reference's softmax over the language tokens'
    PROBABILITIES (quirk kept), arg-max.  Through the C ABI: wsp_detect_language."""
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "lang_detect.npz"))
    m = capi.Model(synth.model_path("micro-sc"))
    e = capi.Engine(m, 0)
    c = capi.Context(e, 1)
    try:
        for i, ch in enumerate(g["chunks"].tolist()):
            c.pcm_to_mel(0, synth.synth_pcm(ch, 480000))
            lid, probs = c.detect_language(0, g["lang_probs"].shape[1])
            assert lid == int(g["lang_id"][i])
            assert np.abs(probs - g["lang_probs"][i]).max() < 2e-4
    finally:
        c.close(); e.close(); m.close()


def test_short_audio_is_a_noop(session):
    L, h = session
    hr, segs = run_full(L, h, synth.synth_pcm(0, 8000))      # < 1 s: whisper_full returns without doing anything (whisper.cpp:2813-2818)
    assert hr == 0 and segs == []
    hr, segs = run_full(L, h, np.zeros(0, np.float32))
    assert hr == 0 and segs == []


def test_unknown_language_and_unsupported_flags(session):
    L, h = session
    hr, _ = run_full(L, h, synth.synth_pcm(0, 32000), language=b"zz")
    assert (hr & 0xFFFFFFFF) == 0x80070057                     # E_INVALIDARG
    hr, _ = run_full(L, h, synth.synth_pcm(0, 32000), flags=0x200)   # SpeedupAudio
    assert (hr & 0xFFFFFFFF) == 0x80004001                     # E_NOTIMPL


def test_imodel_surface(session):
    L, h = session
    assert L.wspc_query_interfaces(h) == 0
    assert L.wspc_is_multilingual(h) == 0
    st = (C.c_int32 * 8)()
    assert L.wspc_special_tokens(h, st) == 0
    assert list(st) == [50256, 50257, 50360, 50361, 50362, 50363, 50358, 50359]
    assert L.wspc_string_from_token(h, 42) == b" t42"
    assert L.wspc_string_from_token(h, 50363) == b"[_BEG_]"
    # the synthetic vocabulary is " t<i>": the GPT-2 pre-split separates letters from digits, so nothing matches (as in the reference)
    out = (C.c_int32 * 16)()
    assert L.wspc_tokenize(h, b" t12 t345", out, 16) == 0
    assert L.wspc_language_count() == 99
    assert L.wspc_find_language_key(b"en") == ord("e") | (ord("n") << 8)
    assert L.wspc_find_language_key(b"haw") == ord("h") | (ord("a") << 8) | (ord("w") << 16)
    assert L.wspc_find_language_key(b"english") == ord("e") | (ord("n") << 8)
    assert L.wspc_find_language_key(b"klingon") == 0xFFFFFFFF


# iModel::tokenize against the reference's whisper_tokenize (whisper.cpp:2192-2245, 2378-2391) on the "-words" vocabulary
# (synth.tokenizer_test_words).  Expected ids were produced by oracle/_ref (RefOracle.tokenize) with tests/golden/make_golden.py
# --tokenizer; they include the reference's quirk of emitting one single-character token right after every non-final match.
TOKENIZER_GOLDEN = {
    b" hello hellox 12345!": [100, 100, 23, 103, 29, 30, 31],
    b" hello world's , worlds 345 12": [100, 109, 107, 108, 109, 18, 36, 29, 30, 31, 103],
    b" t12 t345": [36, 19, 27, 28, 36, 19, 104],
    b"": [],
}


def test_tokenize_matches_reference():
    L = _lib()
    h = C.c_void_p()
    assert L.wspc_open(synth.model_path("micro.en-words").encode(), 0, C.byref(h)) == 0
    try:
        out = (C.c_int32 * 64)()
        for text, want in TOKENIZER_GOLDEN.items():
            n = L.wspc_tokenize(h, text, out, 64)
            assert n == len(want) and list(out)[:n] == want, (text, list(out)[:max(n, 0)])
    finally:
        L.wspc_close(h)

"""Stereo chunks and per-segment speakers on the batch path, on an H100: wsp_upload_pcm_stereo (downmix_stereo_kernel) and
wsp_chunk_speakers (speaker_kernel), iContext::detectSpeaker for a whole batch.

Oracles: numpy for the downmix ((l + r) * 0.5 in f32, bit for bit); the COM path's runFull + detectSpeaker for each clip alone (through
the wspc_run_full_stereo shim); the host rule of csrc/speaker.h (wsp_test_speakers) and the lane-order numpy restatement of
tests/test_speakers.py on crafted cases, including the ones one ulp either side of 1.1 that a pairwise sum would decide differently.
"""
import ctypes as C
import os

import numpy as np
import pytest

from tests import test_gpu_com as com
from tests import test_speakers as ref
from tests.golden import make_chunks_window_golden as mkw
from whisper_b200 import capi, synth

pytestmark = pytest.mark.gpu

F32 = np.float32
E_INVALIDARG, E_POINTER, E_BOUNDS = -1, -2, -7
_cache = {}


def engine(model):
    if model not in _cache:
        m = capi.Model(synth.model_path(model))
        _cache[model] = (m, capi.Engine(m, 0))
    return _cache[model]


def launches(f):
    L = capi.lib()
    before = L.wsp_launch_count()
    r = f()
    return r, int(L.wsp_launch_count() - before)


def downmix(lr):
    return ((lr[:, 0] + lr[:, 1]) * F32(0.5)).astype(F32)


def gains_stereo(mono, rotate=0):
    """the channel-gain pattern of test_gpu_com.py's detectSpeaker test: left loud for 2 s, right loud for 2 s, balanced for 2 s, ...
    (started `rotate` phases later)"""
    t = np.arange(mono.size) / 16000.0
    phase = ((t // 2).astype(np.int64) + rotate) % 3
    g = np.choose(phase, [1.6, 0.4, 1.0]).astype(F32)
    return np.stack([mono * g, mono * (F32(2.0) - g)], axis=1).astype(F32)


def window_clip(i):
    """clips of the window fixtures' family: the fixture's PCM chunk ids over its candidate lengths"""
    return synth.synth_pcm(i % 4, mkw.LENGTHS[i % len(mkw.LENGTHS)])


# ---- the downmix ------------------------------------------------------------------------------------------------------------------
DOWNMIX_LENGTHS = (0, 1, 2, 3, 159, 161, 160 * 37 - 1, 160 * 37 + 1, 480000)


def test_downmix_bit_identical():
    m, e = engine("micro.en-sc")
    c = capi.Context(e, 2)
    rng = np.random.default_rng(1)
    try:
        for n in DOWNMIX_LENGTHS:
            lr = (rng.standard_normal((n, 2)) * [0.3, 0.7]).astype(F32)
            _, k = launches(lambda: c.upload_pcm_stereo(1, lr))
            assert k == 1, n
            assert c.get_tensor("pcm", 1).tobytes() == downmix(lr).tobytes(), n
            assert c.get_tensor("pcm_stereo", 1).tobytes() == lr.tobytes(), n
        # wsp_upload_pcm drops the stereo
        c.upload_pcm(1, synth.synth_pcm(0, 1000))
        assert c.get_tensor("pcm_stereo", 1).size == 0 and c.get_tensor("pcm", 1).tobytes() == synth.synth_pcm(0, 1000).tobytes()
    finally:
        c.close()


@pytest.mark.parametrize("model,batch", [("micro.en-sc", 5), ("medium-sc", 8)])
def test_stereo_upload_runs_as_its_mono(model, batch):
    """run_chunks_window from the stereo upload equals the same call after upload_pcm of the downmix: tokens, results, segments,
    energy and token times"""
    m, e = engine(model)
    if batch == 5:
        g = np.load(os.path.join(os.path.dirname(__file__), "golden", "chunks_window.npz"))
        monos = [synth.synth_pcm(int(ch), int(n)) for ch, n in zip(g["micro_en_chunks"], g["micro_en_n_samples"])]
    else:
        monos = [synth.synth_pcm(b, (480000, 440000, 160000, 400000, 240000, 12000)[b % 6]) for b in range(batch)]
    lrs = [gains_stereo(p, b) for b, p in enumerate(monos)]
    c = capi.Context(e, batch)
    try:
        c.set_token_timestamps(1)
        runs = []
        for stereo in (True, False):
            for b, lr in enumerate(lrs):
                c.upload_pcm_stereo(b, lr) if stereo else c.upload_pcm(b, downmix(lr))
            out, _ = c.run_chunks_window(None, m.prompt_init(), batch=batch, token_times=dict(max_len=0))
            runs.append((out, [c.get_tensor("energy", b).tobytes() for b in range(batch)]))
        assert runs[0][0] == runs[1][0]
        assert runs[0][1] == runs[1][1]
        assert any(o["segments"] for o in runs[0][0])
    finally:
        c.close()


# ---- speakers against the COM path ------------------------------------------------------------------------------------------------
def com_session(model):
    L = com._lib()
    h = C.c_void_p()
    assert L.wspc_open(synth.model_path(model).encode(), 0, C.byref(h)) == 0
    return L, h


def com_speakers(L, h, mono, lr):
    """runFull of the clip alone, detectSpeaker asked about every segment from the segment callback -> [(t0, t1, speaker)]"""
    fp = lambda a: a.ctypes.data_as(C.POINTER(C.c_float))
    sp = (C.c_int32 * 256)()
    inter = np.ascontiguousarray(lr).reshape(-1)
    n = L.wspc_run_full_stereo(h, fp(mono), fp(inter), mono.size, 2, 0, sp, 256, None)
    assert n >= 0, hex(n & 0xFFFFFFFF)
    return [(L.wspc_segment_t0(h, i), L.wspc_segment_t1(h, i), int(sp[i])) for i in range(n)]


def test_speakers_match_detect_speaker():
    """each chunk's speakers equal runFull + detectSpeaker on that clip alone, for every clip whose runFull is one window (its
    segments are the batch window's); with max_len 12 the wrapped token-time segments equal runFull's and their speakers the rule's"""
    m, e = engine("micro.en-sc")
    B = 16
    lrs = [gains_stereo(window_clip(i), i) for i in range(B)]
    monos = [downmix(lr) for lr in lrs]
    c = capi.Context(e, B)
    L, h = com_session("micro.en-sc")
    try:
        c.set_token_timestamps(1)
        out, _ = c.run_chunks_window(lrs, m.prompt_init(), speakers=True)
        wrapped, _ = c.run_chunks_window(lrs, m.prompt_init(), speakers=True, token_times=dict(max_len=12))
        matched, answers, n_wrapped = 0, set(), 0
        for b in range(B):
            want = com_speakers(L, h, monos[b], lrs[b])
            got = [(s["t0"], s["t1"], s["speaker"]) for s in out[b]["segments"]]
            if [w[:2] for w in want] != [g[:2] for g in got] or not got:
                continue                                    # runFull went past the first window
            matched += 1
            assert got == want, b
            answers |= {g[2] for g in got}
            # max_len 12: runFull's wrapped segments are the batch's, each answered by the host rule over the clip's stereo
            hr, segs = com.run_full(L, h, monos[b], flags=2 | 0x100, max_len=12)
            assert hr == 0
            gw = [(s["t0"], s["t1"]) for s in wrapped[b]["segments"]]
            assert [(s["t0"], s["t1"]) for s in segs] == gw, b
            assert [s["speaker"] for s in wrapped[b]["segments"]] == capi.test_speakers(lrs[b], gw), b
            n_wrapped += len(gw)
        assert matched >= 4 and n_wrapped > matched
        assert {capi.SPEAKER_LEFT, capi.SPEAKER_RIGHT, capi.SPEAKER_UNSURE} <= answers, answers
    finally:
        L.wspc_close(h)
        c.close()


# ---- the kernel against the host rule ---------------------------------------------------------------------------------------------
def device_speakers(c, lrs, segs):
    """upload each chunk (None: mono only) and answer its segments in one wsp_chunk_speakers call"""
    for b, lr in enumerate(lrs):
        if lr is None:
            c.upload_pcm(b, synth.synth_pcm(b, 4000))
        else:
            c.upload_pcm_stereo(b, lr)
    return c.chunk_speakers([[dict(t0=a, t1=z) for a, z in s] for s in segs])


def test_crafted_and_random_cases_on_the_device():
    m, e = engine("micro.en-sc")
    c = capi.Context(e, 16)
    try:
        cases = [(name, lr, segs, want) for name, lr, segs, want, _ in ref.crafted_cases()]
        cases += [(name, lr, segs, [ref.speaker_ref(lr, a, z) for a, z in segs]) for name, lr, segs in ref.random_cases()]
        for i in range(0, len(cases), 16):
            part = cases[i:i + 16]
            got = device_speakers(c, [lr for _, lr, _, _ in part], [segs for _, _, segs, _ in part])
            for (name, lr, segs, want), g in zip(part, got):
                assert g == want, name
                assert g == capi.test_speakers(lr, segs), name
        # the near-1.1 cases include ones a pairwise sum decides differently
        assert any(n.startswith("order_") for n, _, _, _ in cases)
    finally:
        c.close()


def test_full_batches_and_long_lists():
    m, e = engine("micro.en-sc")
    c = capi.Context(e, 16)
    rng = np.random.default_rng(5)
    try:
        # B = 16 chunks of 30 s, one segment 0..3000 each
        lrs = [gains_stereo(synth.synth_pcm(b % 4, 480000), b) * rng.uniform(0.8, 1.2, 2).astype(F32) for b in range(16)]
        segs = [[(0, 3000)] for _ in lrs]
        (got, k) = launches(lambda: device_speakers(c, lrs, segs))
        assert got == [capi.test_speakers(lr, s) for lr, s in zip(lrs, segs)]
        # more than 200 segments in one chunk, an empty list, a slot that was last given mono
        long_segs = [(int(a), int(a + rng.integers(0, 60))) for a in rng.integers(-2, 3005, 256)]
        long_segs += [(-1, 5), (3000, 3010), (2999, 3100), (3004, 3004)]
        lrs2 = [lrs[0], lrs[1], None, lrs[3]]
        segs2 = [long_segs, [], [(0, 10), (5, 5), (100, 3000)], [(10, 20)]]
        got = device_speakers(c, lrs2, segs2)
        assert got[0] == capi.test_speakers(lrs[0], long_segs) and len(got[0]) == 260
        assert got[1] == [] and got[3] == capi.test_speakers(lrs[3], [(10, 20)])
        assert got[2] == [capi.SPEAKER_NO_STEREO, capi.SPEAKER_UNSURE, capi.SPEAKER_NO_STEREO]
        assert {capi.SPEAKER_OUT_OF_RANGE, capi.SPEAKER_LEFT, capi.SPEAKER_RIGHT} <= set(got[0])
        # a batch without segments launches nothing
        (got, k) = launches(lambda: c.chunk_speakers([[], []]))
        assert got == [[], []] and k == 0
    finally:
        c.close()


def test_speed_up_segments():
    """under speed-up the window's segment times are doubled: real time over the original samples"""
    m, e = engine("micro.en-sc")
    lrs = [gains_stereo(synth.synth_pcm(b, n), b) for b, n in enumerate((960000, 960000, 640000, 320000))]
    c = capi.Context(e, len(lrs))
    try:
        c.set_speed_up(1)
        out, _ = c.run_chunks_window(lrs, m.prompt_init(), speakers=True)
        assert any(o["segments"] for o in out)
        for o, lr in zip(out, lrs):
            segs = [(s["t0"], s["t1"]) for s in o["segments"]]
            assert [s["speaker"] for s in o["segments"]] == capi.test_speakers(lr, segs)
    finally:
        c.close()


# ---- nothing else changes ---------------------------------------------------------------------------------------------------------
def test_other_calls_unchanged():
    """after stereo uploads and speaker calls, run_chunks, run_chunks_until_eot and run_chunks_window from host PCM are bit-identical
    with unchanged launches; the stereo upload costs one launch and wsp_chunk_speakers one"""
    m, e = engine("micro.en-sc")
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "chunks_window.npz"))
    pcms = [synth.synth_pcm(int(ch), int(n)) for ch, n in zip(g["micro_en_chunks"], g["micro_en_n_samples"])]
    prompt = m.prompt_init()
    batch = len(pcms)

    def calls(c):
        (w, _), nw = launches(lambda: c.run_chunks_window(pcms, prompt))
        (a, _), na = launches(lambda: c.run_chunks(pcms, prompt, 60))
        la = c.logits(batch)
        (u, _), nu = launches(lambda: c.run_chunks_until_eot(pcms, prompt, 100))
        return w, a.tolist(), la.tobytes(), [t.tolist() for t in u], (nw, na, nu)

    fresh = capi.Context(e, batch)
    try:
        want = calls(fresh)
    finally:
        fresh.close()
    c = capi.Context(e, batch)
    try:
        for b, p in enumerate(pcms):
            _, k = launches(lambda: c.upload_pcm_stereo(b, gains_stereo(p, b)))
            assert k == 1
        _, k = launches(lambda: c.chunk_speakers([[dict(t0=0, t1=100)]] * batch))
        assert k == 1
        c.run_chunks_window(None, prompt, batch=batch, speakers=True)
        assert calls(c) == want
    finally:
        c.close()


def test_errors_launch_nothing():
    m, e = engine("micro.en-sc")
    c = capi.Context(e, 2)
    L = capi.lib()
    segs = (capi.Segment * 4)(*[capi.Segment(0, 10, 0, 0)] * 4)
    out = np.zeros(4, np.int32)
    i = capi._i

    def call(ctx, batch, start, sg=segs, o=None, n_launches=0):
        before = L.wsp_launch_count()
        st = np.ascontiguousarray(start, np.int32) if start is not None else None
        rc = L.wsp_chunk_speakers(ctx, batch, None if st is None else i(st), sg, i(out) if o is None else o)
        assert L.wsp_launch_count() == before + n_launches
        return rc

    try:
        lr = gains_stereo(synth.synth_pcm(0, 16000))
        c.upload_pcm_stereo(0, lr)
        c.upload_pcm_stereo(1, lr)
        assert call(None, 2, [0, 2, 4]) == E_POINTER
        assert call(c.h, 2, None) == E_POINTER
        assert call(c.h, 2, [0, 2, 4], sg=None) == E_POINTER
        assert call(c.h, 2, [0, 2, 4], o=C.cast(None, C.POINTER(C.c_int32))) == E_POINTER
        assert call(c.h, 2, [1, 2, 4]) == E_INVALIDARG
        assert call(c.h, 2, [0, 3, 2]) == E_INVALIDARG
        assert call(c.h, 3, [0, 1, 2, 3]) == E_BOUNDS
        assert call(c.h, 0, [0]) == E_BOUNDS
        assert call(c.h, 2, [0, 2, 4], n_launches=1) == 0 and out.tolist() == [capi.test_speakers(lr, [(0, 10)])[0]] * 4
        before = L.wsp_launch_count()
        fp = capi._f(lr)
        assert L.wsp_upload_pcm_stereo(c.h, 2, fp, 100) == E_BOUNDS
        assert L.wsp_upload_pcm_stereo(c.h, 0, fp, -1) == E_INVALIDARG
        assert L.wsp_upload_pcm_stereo(c.h, 0, None, 100) == E_INVALIDARG
        assert L.wsp_upload_pcm_stereo(None, 0, fp, 100) == E_POINTER
        assert L.wsp_launch_count() == before
    finally:
        c.close()

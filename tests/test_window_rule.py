"""whisper_full's window rule and segmentation on the host, no GPU: csrc/window_rule.h (through the wsp_test_window_rule hook; runFull
and the sampler epilogue run the same code) and wsp_window_segments against the Python restatements of whisper.cpp:2926-3003 and
3026-3119 in tests/golden/make_chunks_window_golden.py, on crafted token sequences that reach every branch."""
import numpy as np
import pytest

from tests.golden import make_chunks_window_golden as mk
from whisper_b200 import capi, synth

EOT, BEG = 50256, 50363          # micro.en's specials
TEXT = (5, 6, 7, 220)


def hook(ids, max_tokens=0, single=False, n_max=220, seek=0, seek_end=3000):
    return capi.test_window_rule(ids, EOT, BEG, max_tokens, single, n_max, seek, seek_end)


def restated(ids, max_tokens=0, single=False, n_max=220, seek=0, seek_end=3000):
    r, kind, used = mk.rule(list(ids), EOT, BEG, max_tokens, single, n_max, seek, seek_end)
    return dict(r, ended=int(kind is not None)), kind, used


# (ids, max_tokens, single_segment, n_max, seek, seek_end, kind, failed, result_len, seek_delta)
CRAFTED = [
    ([BEG, 5, 6, BEG + 100, 7, EOT], 0, 0, 220, 0, 3000, "eot", 0, 4, 200),
    ([5, 6, EOT], 0, 0, 220, 0, 4000, "eot", 1, 0, 3000),                       # EOT with no timestamp: failed
    ([5, 6, EOT], 0, 0, 220, 0, 3100, "eot", 0, 3, 3000),                       # ... unless the window reaches the end of the audio
    ([BEG, 5, BEG + 100, 6, 7, BEG + 60, 5], 0, 0, 220, 0, 3000, "back_in_time", 0, 3, 200),
    ([BEG, 5, BEG + 100, BEG + 60, 5, EOT], 0, 0, 220, 0, 3000, "eot", 0, 4, 120),   # consecutive: not back in time
    ([BEG + 1, 5, 6, 7, 5, 6], 3, 0, 220, 0, 3000, "max_tokens", 0, 1, 2),
    ([5, 6, 7, 5], 2, 0, 220, 0, 4000, "max_tokens", 1, 0, 3000),
    ([BEG, 5, BEG + 450, 6], 0, 0, 220, 0, 1000, "audio_end", 0, 3, 900),
    ([BEG, 5, BEG + 200, 6], 0, 0, 220, 500, 1000, "audio_end", 0, 3, 400),     # seek + seek_delta + 100 >= seek_end
    ([BEG, 5, BEG + 100, 6, EOT], 0, 1, 220, 0, 3000, "eot", 0, 5, 3000),       # single segment
    ([5, 6] * 10, 0, 0, 10, 0, 3000, "n_max", 1, 0, 3000),
    ([BEG, 5, BEG + 800, 6] + [7] * 10, 0, 0, 10, 0, 3000, "n_max", 0, 3, 1600),
    ([BEG, 5, BEG + 700, 6] + [7] * 10, 0, 0, 10, 0, 3000, "n_max", 1, 3, 1400),
    ([BEG, 5, 6], 0, 0, 220, 0, 3000, None, 0, 0, 3000),                        # not ended yet; BEG itself is no timestamp
]


@pytest.mark.parametrize("case", CRAFTED, ids=[str(i) for i in range(len(CRAFTED))])
def test_crafted_sequences(case):
    ids, mt, single, n_max, seek, seek_end, kind, failed, result_len, seek_delta = case
    got, used = hook(ids, mt, single, n_max, seek, seek_end)
    want, wkind, wused = restated(ids, mt, single, n_max, seek, seek_end)
    assert wkind == kind
    assert (got, used) == (want, wused)
    assert (got["failed"], got["result_len"], got["seek_delta"]) == (failed, result_len, seek_delta)


def test_random_sequences_reach_every_branch():
    rng = np.random.default_rng(7)
    kinds = set()
    for _ in range(3000):
        n = int(rng.integers(1, 40))
        alphabet = list(TEXT) + [EOT] + [BEG + int(k) for k in rng.integers(0, 1500, 4)]
        p = np.array([0.55, 0.1, 0.05, 0.05, 0.03, 0.06, 0.06, 0.05, 0.05])
        ids = [int(x) for x in rng.choice(alphabet, n, p=p / p.sum())]
        args = (int(rng.choice([0, 0, 3, 8])), bool(rng.integers(0, 2)), int(rng.choice([220, 12, 25])), int(rng.choice([0, 0, 700])),
                int(rng.choice([4000, 3000, 1500, 400, 150])))
        got, used = hook(ids, *args)
        want, kind, wused = restated(ids, *args)
        assert (got, used) == (want, wused), (ids, args)
        kinds.add((kind, want["failed"]))
    for k in [("eot", 0), ("eot", 1), ("back_in_time", 0), ("max_tokens", 0), ("max_tokens", 1), ("audio_end", 0), ("n_max", 0), ("n_max", 1), (None, 0)]:
        assert k in kinds, k


@pytest.fixture(scope="module")
def model():
    return capi.Model(synth.model_path("micro.en-sc"))


def tokens_of(ids, rng):
    # tid: the most probable timestamp; for a timestamp token it is the token itself, as the reference's sampler gives
    return [dict(id=i, tid=i if i > BEG else BEG + int(rng.integers(0, 1500)), p=0.5, pt=0.25, ptsum=0.125) for i in ids]


@pytest.mark.parametrize("flags", [0, capi.SEGMENT_SINGLE, capi.SEGMENT_PRINT_SPECIAL, capi.SEGMENT_SPEED_UP,
                                   capi.SEGMENT_PRINT_SPECIAL | capi.SEGMENT_SPEED_UP])
def test_segments_match_restatement(model, flags):
    assert (model.special["eot"], model.special["beg"]) == (EOT, BEG)
    rng = np.random.default_rng(flags)
    text = lambda i: model.token_text(i) or ""
    seen = set()
    for _ in range(400):
        n = int(rng.integers(1, 30))
        alphabet = list(TEXT) + [EOT, model.special["sot"]] + [BEG + int(k) for k in rng.integers(0, 1500, 3)]
        ids = [int(x) for x in rng.choice(alphabet, n)]
        toks = tokens_of(ids, rng)
        res = dict(n_sampled=n, n_tokens=int(rng.integers(0, n + 1)), seek_delta=int(rng.integers(1, 3001)), failed=int(rng.random() < 0.1))
        seek = int(rng.choice([0, 0, 1234]))
        got = model.window_segments(toks, res, seek, flags)
        want = mk.segments(toks, res, seek, EOT, BEG, text, single_segment=bool(flags & capi.SEGMENT_SINGLE),
                           print_special=bool(flags & capi.SEGMENT_PRINT_SPECIAL), speed_up=bool(flags & capi.SEGMENT_SPEED_UP))
        assert got == want, (ids, res, seek)
        seen.add(len(got))
    assert {0, 1} <= seen and max(seen) >= (1 if flags & capi.SEGMENT_SINGLE else 3)


def test_speed_up_doubles_times(model):
    rng = np.random.default_rng(3)
    toks = tokens_of([BEG, 5, 6, BEG + 200, BEG + 210, 7, 220, BEG + 400, 5], rng)
    res = dict(n_sampled=9, n_tokens=9, seek_delta=3000, failed=0)
    a = model.window_segments(toks, res, 100, 0)
    b = model.window_segments(toks, res, 100, capi.SEGMENT_SPEED_UP)
    assert len(a) == 3 and [(s["t0"] * 2, s["t1"] * 2, s["i0"], s["i1"], s["text"]) for s in a] == \
        [(s["t0"], s["t1"], s["i0"], s["i1"], s["text"]) for s in b]
    # consecutive timestamps are skipped: the second segment starts after both, at the time of the first
    assert (a[0]["i1"], a[1]["i0"], a[1]["t0"]) == (4, 5, 100 + 2 * 200)


def test_segments_errors(model):
    rng = np.random.default_rng(0)
    toks = tokens_of([BEG, 5, BEG + 10, 6, BEG + 20, 7, BEG + 30], rng)
    res = dict(n_sampled=7, n_tokens=7, seek_delta=60, failed=0)
    L = capi.lib()
    td = (capi.TokenData * 7)(*[capi.TokenData(t["id"], t["tid"], t["p"], t["pt"], t["ptsum"]) for t in toks])
    r = capi.WindowResult(7, 7, 60, 0)
    n = np.zeros(1, np.int32)
    segs = (capi.Segment * 8)()
    assert L.wsp_window_segments(model.h, td, r, 0, 0, None, 0, capi._i(n)) == -7 and n[0] == 3   # count only: more than cap 0
    assert L.wsp_window_segments(model.h, td, r, 0, 0, segs, 2, capi._i(n)) == -7 and n[0] == 3
    assert L.wsp_window_segments(model.h, td, r, 0, 0, segs, 3, capi._i(n)) == 0 and n[0] == 3
    assert L.wsp_window_segments(model.h, None, r, 0, 0, segs, 3, capi._i(n)) == -2
    bad = capi.WindowResult(3, 7, 60, 0)
    assert L.wsp_window_segments(model.h, td, bad, 0, 0, segs, 3, capi._i(n)) == -1
    assert len(model.window_segments(toks, res)) == 3

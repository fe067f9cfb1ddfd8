"""whisper_full's token-level timestamps on the host, no GPU: csrc/token_times.h (through the wsp_test_token_times hook; runFull and
wsp_window_token_times run the same code) against the Python restatement of whisper.cpp:3374-3600 in
tests/golden/make_chunks_token_ts_golden.py, on crafted segments that reach every branch and on random ones."""
import numpy as np
import pytest

from tests.golden import make_chunks_token_ts_golden as mk
from whisper_b200 import capi

EOT, BEG = 50256, 50363          # micro.en's specials
SR = 16000


def tok(id_, tid=BEG, pt=0.5, ptsum=0.5):
    return dict(id=id_, tid=tid, p=0.9, pt=pt, ptsum=ptsum)


def both(tokens, vlen, t0, t1, energy, state=(0, 0, 0), times=None, thold_pt=0.01, thold_ptsum=0.01):
    """(hook result, restated result, branches the restatement took); each result = (times, state, had energy)"""
    times = times or [[-1, -1, 0.0] for _ in tokens]
    got = capi.test_token_times(tokens, vlen, t0, t1, BEG, EOT, energy, thold_pt, thold_ptsum, state, [list(t) for t in times])
    want_t, want_s, hit = [list(t) for t in times], list(state), set()
    ok = mk.token_times(tokens, vlen, want_t, t0, t1, BEG, EOT, np.asarray(energy, np.float32), thold_pt, thold_ptsum, want_s, hit)
    want_t = [[a, b, float(np.float32(v))] for a, b, v in want_t]
    return got, (want_t, want_s, ok), hit


def energy_of(n, bursts, floor=0.01, level=0.5):
    """a clip of n samples that is quiet except for [s, e) bursts"""
    x = np.full(n, floor, np.float32)
    for s, e in bursts:
        x[s:e] = level
    return mk.signal_energy(x)


def test_signal_energy_restatement_is_the_reference_loop():
    rng = np.random.default_rng(1)
    for n in (0, 1, 5, 64, 65, 66, 300):
        x = rng.standard_normal(n).astype(np.float32)
        want = np.zeros(n, np.float32)
        for i in range(n):
            s = np.float32(0)
            for j in range(-32, 33):
                if 0 <= i + j < n:
                    s = np.float32(s + np.float32(abs(x[i + j])))
            want[i] = s / np.float32(65)
        assert mk.signal_energy(x).tobytes() == want.tobytes()


def test_no_energy_changes_nothing():
    toks = [tok(BEG), tok(5), tok(BEG + 10)]
    (t, s, ok), (wt, ws, wok), _ = both(toks, [1.0, 1.0, 1.0], 0, 20, np.zeros(0, np.float32), state=(3, 4, 5))
    assert not ok and not wok and s == [3, 4, 5] and t == [[-1, -1, 0.0]] * 3


@pytest.mark.parametrize("n", [0, 1])
def test_short_segments(n):
    toks = [tok(5)][:n]
    got, want, _ = both(toks, [1.0] * n, 7, 90, energy_of(SR, [(0, 8000)]), state=(1, 2, 3))
    assert got == want
    if n == 1:
        assert got[0] == [[7, 90, 0.0]] and got[1] == [1, 2, 3]      # times only; vlen and the state are left alone


# crafted segments: (tokens, vlen, t0, t1, bursts of the 2 s clip, state, times on entry, branches the segment must take)
CRAFTED = [
    # a leading beg and a confident timestamp on every token (no gap to split): starts move later, ends earlier with the energy
    ([tok(BEG, BEG), tok(5, BEG + 10), tok(6, BEG + 40), tok(7, BEG + 60), tok(BEG + 80, BEG + 80)], [0.0, 2.0, 1.0, 3.0, 0.0], 0, 160,
     [(2000, 9000), (14000, 26000)], (0, 0, 0), None, {"beg", "t0_later", "t1_earlier"}),
    # no leading beg: the first start is t_last of the state; one burst over the whole clip
    ([tok(5, BEG + 20), tok(220, BEG + 30), tok(6, BEG + 50), tok(EOT, BEG + 70)], [1.0, 0.01, 2.0, 0.0], 40, 120,
     [(0, 32000)], (40, 30, 0), None, {"vlen_split"}),
    # unconfident timestamps (pt, ptsum at or below the thresholds) and a tid not above tid_last: only the voice lengths place tokens
    ([tok(BEG, BEG), tok(5, BEG + 10, pt=0.01), tok(6, BEG + 20, ptsum=0.005), tok(7, BEG + 2, pt=0.9)], [0.0, 1.0, 3.0, 1.0], 10, 100,
     [(1000, 3000), (20000, 30000)], (0, 0, 0), None, {"beg", "vlen_split", "t0_earlier", "t1_earlier", "t1_later"}),
    # a timestamp past the segment's end (tt > t1) is not taken; a quiet clip
    ([tok(BEG, BEG), tok(5, BEG + 90), tok(6, BEG + 95)], [0.0, 1.0, 1.0], 0, 100, [], (0, 0, 0), None, {"beg", "t1_later"}),
    # the fix-up: times handed in that overlap, and a negative segment end that leaves negative ends behind
    ([tok(5), tok(6), tok(7), tok(8)], [1.0, 1.0, 1.0, 1.0], 50, 150, [(8000, 30000)], (50, 50, 0),
     [[-1, 120, 0.0], [-1, 90, 0.0], [-1, 80, 0.0], [-1, -1, 0.0]], {"t1_later"}),
    ([tok(5), tok(6), tok(7)], [1.0, 1.0, 1.0], 30, -4, [(0, 4000)], (30, 30, 0), None, {"vlen_split"}),
    # every token of the segment inside loud audio that starts before the segment
    ([tok(5, BEG), tok(6, BEG + 30), tok(7, BEG + 60), tok(8, BEG + 90)], [1.0, 1.0, 1.0, 1.0], 20, 110, [(0, 30000), (31000, 32000)],
     (0, 20, 0), None, {"vlen_split"}),
]


@pytest.mark.parametrize("case", range(len(CRAFTED)))
def test_crafted(case):
    toks, vlen, t0, t1, bursts, state, times, need = CRAFTED[case]
    got, want, hit = both(toks, vlen, t0, t1, energy_of(2 * SR, bursts), state=state, times=times)
    assert got == want
    assert need <= hit, (need, hit)


def test_crafted_reach_every_comparison():
    """across the crafted segments, each side of every energy comparison and every kind of move"""
    hit = set()
    for toks, vlen, t0, t1, bursts, state, times, _need in CRAFTED:
        h = set()
        tt = [list(t) for t in (times or [[-1, -1, 0.0]] * len(toks))]
        mk.token_times(toks, vlen, tt, t0, t1, BEG, EOT, energy_of(2 * SR, bursts), 0.01, 0.01, list(state), h)
        hit |= h
    assert {"beg", "vlen_split", "t0_earlier", "t0_later", "t1_earlier", "t1_later"} <= hit, hit


def test_random_segments():
    rng = np.random.default_rng(7)
    hit = set()
    for trial in range(150):
        n = int(rng.integers(2, 14))
        ids = rng.choice([5, 6, 7, 220, 11, 13, EOT, BEG, BEG + 1, BEG + 300], size=n, p=[.2, .15, .15, .1, .1, .1, .05, .05, .05, .05]).tolist()
        if rng.random() < 0.5:
            ids[0] = BEG
        t0 = int(rng.integers(0, 300))
        t1 = t0 + int(rng.integers(0, 900))
        toks = [tok(int(i), BEG + int(rng.integers(0, 700)), pt=float(rng.choice([0.005, 0.01, 0.02, 0.4])),
                    ptsum=float(rng.choice([0.005, 0.01, 0.03, 0.8]))) for i in ids]
        vlen = [float(np.float32(v)) for v in rng.choice([0.01, 1.0, 2.0, 3.0, 4.01], size=n)]
        n_samples = int(rng.integers(1, 14 * SR))
        bursts = [(int(s), int(s) + int(rng.integers(100, 3 * SR))) for s in rng.integers(0, n_samples, size=int(rng.integers(0, 6)))]
        x = (rng.standard_normal(n_samples) * 0.02).astype(np.float32)
        for s, e in bursts:
            x[s:e] *= float(rng.uniform(5, 50))
        state = (int(rng.integers(0, 200)), int(rng.integers(0, 200)), int(rng.choice([0, BEG, BEG + 100])))
        got, want, h = both(toks, vlen, t0, t1, mk.signal_energy(x), state=state)
        assert got == want, trial
        hit |= h
    assert {"beg", "vlen_split", "t0_earlier", "t0_later", "t1_earlier", "t1_later"} <= hit, hit

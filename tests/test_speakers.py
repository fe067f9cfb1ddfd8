"""iContext::detectSpeaker's rule (csrc/speaker.h) on the host through wsp_test_speakers, against a numpy restatement of the
reference (Whisper/Whisper/ContextImpl.diarize.cpp:17-108, Spectrogram.cpp:142-168).

The reference sums |L| and |R| in four f32 SSE lanes { L even, R even, L odd, R odd }, each a chain in frame order, and a channel wins
when it exceeds 1.1 times the other.  The restatement keeps those chains (np.add.accumulate adds in order) and decides in f32.  The
crafted cases put each channel's sum exactly on a known f32 value one ulp either side of the 1.1 boundary, and some of them are built
so that a pairwise sum lands elsewhere: the mutation check shows that a pairwise restatement answers differently, so these tests
tell the two orders apart.  tests/test_gpu_chunks_speakers.py runs the same cases through the kernel of wsp_chunk_speakers.
No GPU needed.
"""
import numpy as np

from whisper_b200 import capi

F32 = np.float32
K = F32(1.1)
UNSURE, LEFT, RIGHT, NO_STEREO, OUT_OF_RANGE = 0, 1, 2, 255, -1


def span(n_frames, t0, t1):
    """the frames a segment covers: an answer, or (first, count)"""
    if t1 <= t0:
        return UNSURE
    if n_frames == 0:
        return NO_STEREO
    if t0 < 0 or t0 * 160 >= n_frames:
        return OUT_OF_RANGE
    return t0 * 160, min((t1 - t0) * 160, n_frames - t0 * 160)


def chain(v):
    """an f32 sum in order"""
    return F32(0) if v.size == 0 else F32(np.add.accumulate(np.asarray(v, F32), dtype=F32)[-1])


def lane_sums(lr, t0, t1):
    """(left, right) in the reference's lane order, or the answer when no sums are needed"""
    s = span(lr.shape[0], t0, t1)
    if not isinstance(s, tuple):
        return s
    first, count = s
    x = np.abs(lr[first:first + count].astype(F32))
    return F32(chain(x[0::2, 0]) + chain(x[1::2, 0])), F32(chain(x[0::2, 1]) + chain(x[1::2, 1]))


def pairwise(v):
    v = np.asarray(v, F32)
    if v.size == 0:
        return F32(0)
    if v.size == 1:
        return v[0]
    h = v.size // 2
    return F32(pairwise(v[:h]) + pairwise(v[h:]))


def pairwise_sums(lr, t0, t1):
    """the same sums as one pairwise tree per channel: the order the kernel must NOT use"""
    s = span(lr.shape[0], t0, t1)
    if not isinstance(s, tuple):
        return s
    first, count = s
    x = np.abs(lr[first:first + count].astype(F32))
    return pairwise(x[:, 0]), pairwise(x[:, 1])


def decide(sums):
    if not isinstance(sums, tuple):
        return sums
    left, right = sums
    return (LEFT if left > F32(right * K) else 0) | (RIGHT if right > F32(left * K) else 0)


def speaker_ref(lr, t0, t1):
    return decide(lane_sums(lr, t0, t1))


def boundary(a):
    """the least f32 r with fl(r * 1.1f) >= a: r against a is not a win for a, the f32 just below r is"""
    a = F32(a)
    r = F32(a / K)
    while F32(r * K) >= a:
        r = np.nextafter(r, F32(0))
    while F32(r * K) < a:
        r = np.nextafter(r, F32(np.inf))
    return r


def stereo(left, right, n):
    lr = np.zeros((n, 2), F32)
    lr[:len(left), 0] = left
    lr[:len(right), 1] = right
    return lr


def crafted_cases():
    """[(name, lr, [(t0, t1)], expected answers, (left, right) lane sums of the near-1.1 segment or None)]"""
    rng = np.random.default_rng(7)
    cases = []
    # near 1.1, every channel's lane sum an exact f32 value: left 0.75 = 0.5 (even lane) + 0.25 (odd lane), the right channel a
    # single sample (its lanes add exact zeros); and the mirror image
    for n in (320, 321):                                     # even and odd frame counts
        a = F32(0.75)
        r = boundary(a)
        below = np.nextafter(r, F32(0))
        for name, want, rv in (("left_wins", LEFT, below), ("left_unsure", UNSURE, r)):
            cases.append(("%s_%d" % (name, n), stereo([0.5, -0.25], [0.0, rv], n), [(0, 2)], [want], (a, F32(rv))))
            cases.append(("%s_%d_mirror" % (name, n), stereo([0.0, -rv], [-0.5, 0.25], n), [(0, 2)],
                          [{LEFT: RIGHT, UNSURE: UNSURE}[want]], (F32(rv), a)))
    # the tail frame: an odd count whose last frame (an even lane, alone in its pair) carries the deciding sample
    n = 161
    lr = stereo([0.0] * 160 + [0.75], [0.0] * 160 + [float(boundary(F32(0.75)))], n)
    cases.append(("tail_frame_unsure", lr, [(0, 2)], [UNSURE], (F32(0.75), boundary(F32(0.75)))))
    lr = stereo([0.0] * 160 + [0.75], [0.0] * 160 + [float(np.nextafter(boundary(F32(0.75)), F32(0)))], n)
    cases.append(("tail_frame_left", lr, [(0, 2)], [LEFT], None))
    # order-sensitive: left = [2^24, 2^24, 1 x 318].  Each lane chain stays at 2^24 (2^24 + 1 rounds to even), so the lane-order left is
    # exactly 2^25; a pairwise tree adds the ones first and lands near 2^25 + 318.  The right channel sits on the 1.1 boundary of 2^25.
    big = F32(2.0 ** 24)
    left = [big, big] + [1.0] * 318
    r = boundary(F32(2.0 ** 25))
    for name, want, rv in (("order_unsure", UNSURE, r), ("order_left", LEFT, np.nextafter(r, F32(0)))):
        cases.append((name, stereo(left, [rv], 320), [(0, 2)], [want], (F32(2.0 ** 25), F32(rv))))
        cases.append((name + "_mirror", stereo([rv], [-x for x in left], 320), [(0, 2)], [{LEFT: RIGHT, UNSURE: UNSURE}[want]],
                      (F32(rv), F32(2.0 ** 25))))
    # the rule's other branches over one loud-left clip of 1001 frames (6.25 units of 160)
    n = 1001
    x = rng.standard_normal((n, 2)).astype(F32)
    x[:, 0] *= 3.0
    segs = [(0, 3), (2, 2), (3, 2), (4, 50), (6, 7), (7, 9), (-1, 3), (-5, -1), (50, 60)]
    want = [LEFT, UNSURE, UNSURE, LEFT, LEFT, OUT_OF_RANGE, OUT_OF_RANGE, OUT_OF_RANGE, OUT_OF_RANGE]
    cases.append(("branches", x, segs, want, None))
    # an even-length clip whose last unit is partial: t1 past the end is cut there
    cases.append(("t1_past_even", x[:1000], [(6, 100), (0, 1000)], [LEFT, LEFT], None))
    # no stereo: an empty interval is still Unsure, anything else NoStereoData
    cases.append(("no_stereo", np.zeros((0, 2), F32), [(0, 3), (3, 3), (-2, 1), (5, 4)], [NO_STEREO, UNSURE, NO_STEREO, UNSURE], None))
    return cases


def random_cases(seed=11, n_cases=12):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n_cases):
        n = int(rng.integers(1, 20000))
        lr = rng.standard_normal((n, 2)).astype(F32) * rng.uniform(0.2, 2.0, 2).astype(F32)
        units = n // 160 + 3
        segs = [(int(a), int(a + rng.integers(-3, 40))) for a in rng.integers(-3, units + 3, 25)]
        out.append(("random_%d" % k, lr, segs))
    return out


def test_crafted_cases_match_the_restatement():
    for name, lr, segs, want, sums in crafted_cases():
        assert [speaker_ref(lr, a, b) for a, b in segs] == want, name
        if sums is not None:
            assert lane_sums(lr, *segs[0]) == sums, name            # each channel's sum is the exact value the case was built on
        assert capi.test_speakers(lr, segs) == want, name


def test_near_boundary_cases_are_one_ulp_apart():
    """the wins and unsure cases differ by one ulp of one channel's sum, on either side of the 1.1 boundary"""
    by_name = {name: (lr, segs, sums) for name, lr, segs, want, sums in crafted_cases()}
    for n in (320, 321):
        _, _, (a, r_win) = by_name["left_wins_%d" % n]
        _, _, (_, r_unsure) = by_name["left_unsure_%d" % n]
        assert np.nextafter(r_win, F32(1)) == r_unsure
        assert F32(r_win * K) < a <= F32(r_unsure * K)


def test_random_segment_lists():
    for name, lr, segs in random_cases():
        want = [speaker_ref(lr, a, b) for a, b in segs]
        assert capi.test_speakers(lr, segs) == want, name
        assert capi.test_speakers(None, segs) == [UNSURE if b <= a else NO_STEREO for a, b in segs]
    # every answer occurs
    got = {x for _, lr, segs in random_cases() for x in capi.test_speakers(lr, segs)}
    assert {UNSURE, LEFT, RIGHT, OUT_OF_RANGE} <= got


def test_pairwise_order_flips_a_crafted_case():
    """mutation check: a pairwise restatement answers at least one near-1.1 case differently, so the cases above pin the lane order"""
    flipped = []
    for name, lr, segs, want, sums in crafted_cases():
        got = [decide(pairwise_sums(lr, a, b)) for a, b in segs]
        if got != want:
            flipped.append(name)
    assert flipped and all(n.startswith("order_") for n in flipped), flipped


def test_argument_errors():
    L = capi.lib()
    segs = (capi.Segment * 1)(capi.Segment(0, 1, 0, 0))
    out = np.zeros(1, np.int32)
    assert L.wsp_test_speakers(None, 10, segs, 1, capi._i(out)) == -2            # WSP_E_POINTER
    lr = np.zeros((10, 2), F32)
    assert L.wsp_test_speakers(capi._f(lr), 10, None, 1, capi._i(out)) == -2
    assert L.wsp_test_speakers(capi._f(lr), -1, segs, 1, capi._i(out)) == -1     # WSP_E_INVALIDARG
    assert L.wsp_test_speakers(capi._f(lr), 10, None, 0, None) == 0

"""The GPU sampler (kernels_decode.cu: sample_cluster_kernel, a cluster of 4 CTAs per vocabulary row) on vocabularies far below the
real 51864 tokens, against the numpy restatement of whisper_sample_best (oracle/whisper_np.sample_best) on the probabilities the
kernel returns.  tests/test_gpu_sampler.py covers the real vocabulary, exact ties included, against the reference's own sampler."""
from types import SimpleNamespace

import numpy as np
import pytest

from oracle import whisper_np
from whisper_b200 import capi

pytestmark = pytest.mark.gpu


def small_vocab_rows(n_vocab, seed):
    """16 rows for a vocabulary of n_vocab tokens whose last 150 are timestamps: a clear text leader (rows 0-3), plain random
    rows (4-7), banned tokens as the top 1..3 (8-13) and the best timestamp beyond beg+100 (14-15).  Returns (logits, model)."""
    rng = np.random.default_rng(seed)
    beg = n_vocab - 150
    m = SimpleNamespace(token_beg=beg, token_sot=beg - 6, token_solm=beg - 2, token_not=beg - 1)
    lg = (rng.standard_normal((16, n_vocab)) * 2.0).astype(np.float32)
    for r in range(4):
        lg[r, 11 + 37 * r] = 9.0 + 0.5 * r
    for r in range(8, 14):
        order = [m.token_sot, m.token_solm, m.token_not]
        rng.shuffle(order)
        for i, t in enumerate(order[:1 + r % 3]):
            lg[r, t] = 11.0 - i
        lg[r, 3 + 5 * r] = 8.5
    for r in range(14, 16):
        lg[r, beg + 101 + (17 * r) % 40] = 14.0
        lg[r, beg + (9 * r) % 101] = 12.0
    return lg, m


def test_gpu_sampler_small_vocabulary():
    """Vocabularies far below the real 51864 tokens.  Every cluster CTA holds a slice of the row: 250 or 1024 tokens with the
    timestamps and banned tokens in the last slice, and for 9 tokens slices of 3, 3, 3 and 0 with the timestamp range clipped at the
    end of the row.  Checked in all three sampling modes against the numpy restatement of whisper_sample_best on the returned
    probabilities; the token each row picks has a probability no other token shares, so the reference's std::partial_sort and numpy's
    stable sort agree (the seeds are chosen so; the first assertion checks it)."""
    cases = [small_vocab_rows(1000, 3), small_vocab_rows(4095, 2)]
    rng = np.random.default_rng(1)
    cases.append(((rng.standard_normal((16, 9)) * 2.0).astype(np.float32), SimpleNamespace(token_beg=5, token_sot=1, token_solm=2, token_not=3)))
    for lg, m in cases:
        n_vocab = lg.shape[1]
        special = [m.token_beg, m.token_sot, m.token_solm, m.token_not]
        ids = set()
        for force_ts, initial in ((False, False), (True, False), (True, True)):
            probs, got = capi.test_sample(lg, special, force_ts, initial)
            assert np.allclose(probs.sum(-1), 1.0, atol=2e-5)
            for r in range(lg.shape[0]):
                want = whisper_np.sample_best(m, probs[r], force_ts, initial)
                assert np.count_nonzero(probs[r] == np.float32(want["p"])) == 1, (n_vocab, r, want)
                g = got[r]
                label = (n_vocab, force_ts, initial, r, g, want)
                assert g["id"] == want["id"], label
                assert g["tid"] == want["tid"], label
                assert abs(g["p"] - want["p"]) <= 1e-6, label
                assert abs(g["ptsum"] - want["ptsum"]) <= 1e-6, label
                assert abs(g["pt"] - want["pt"]) <= 2e-6, label
                ids.add(g["id"])
        # text and timestamp tokens both won, and the banned ones never did
        assert min(ids) < m.token_beg <= max(ids)
        assert not ids & {m.token_sot, m.token_solm, m.token_not}

"""Does tests/test_gpu_batch_shapes.py cover the shapes it claims, and would its numpy comparison notice a mistake?  (CPU)

The ring of decode_flow_kernel is restated from decode_flow.cu (Cfg<D>::SLOT, smemLayout, ringSlots) and its slot counts are pinned
to the table of the GPU file's docstring; the GPU file's cases must then reach every width the step kernels are instantiated for,
both column tiles at d = 128, 768 and 1280, the 7-slot ring (NS < FL_WARPS), a cross attention that ends in a partial group of K
slots, and a prompt pass whose chunks straddle the per-op kernel's 16-column tiles.

Mutations: the GPU file's run_oracle and compare, fed the mistake in place of the GPU's result, must report a failure.  Cross-K/V:
an encode of each clip at audio_ctx CROSS_KEYS, to stay fast.
- micro.en-sc (scripted): two slots' results swapped, one chunk's step token replaced by its neighbour's, and one chunk decoded on its
  neighbour's cross-K/V are all caught.
- small (random weights): the neighbour's cross-K/V is caught too, although a random encoder's output is about 95 % one constant
  vector (the rows of a clip's cross K differ from their mean by about 5 % of their magnitude).  Its largest deviation is 167 times
  its tolerance at 64 keys, and 24 times with the full 1500-key encode of both clips (measured once; that encode alone takes over a
  minute in numpy).  The GPU file's bit-for-bit check of the chunks reversed and rotated by 8 covers the same mistake again.
"""
import copy

import pytest

from oracle import whisper_np as wn
from tests.test_gpu_batch_shapes import (CALLS, CASES, FLOW_MAX_B, N_STEPS, NPOS, PCM_SEED, PROMPT_N, SKINNY_COLS, checked_slots, compare,
                                         orders, run_oracle)
from tests.test_gpu_decode_step_long_context import chunk_tokens, slot_rows
from whisper_b200 import synth

# ---- decode_flow.cu, restated -----------------------------------------------------------------------------------------------------
FL_WARPS, FL_NSMAX, FL_MAXT, FL_SMEM_MAX, MAX_REF_THREADS = 8, 32, 1536, 232448, 16
WIDTHS = (128, 384, 512, 768, 1024, 1280)           # dispatchD
NS_TABLE = {8: (12, 12, 12, 12, 11, 9), 16: (12, 11, 11, 10, 10, 7)}


def slot_bytes(d):
    """Cfg<D>::SLOT: 8 weight rows of RS = 2 d + 64 bytes, at least 16 KiB"""
    return max(8 * (2 * d + 64), 16384)


def smem_fixed(d, ncols):
    """smemLayout(SLOT, RS, 0, ncols).total: activations, reduction buffer, scores, bias, residual, partials, and the rest"""
    rs = 2 * d + 64
    return (ncols * rs + 4 * FL_WARPS * 8 * ncols * 4 + FL_MAXT * 4 + 256 * 4 + 16 * 16 * 4 + MAX_REF_THREADS * 64 * 4 + 64 + 3 * 128
            + 2 * FL_NSMAX * 8)


def ring_slots(d, ncols):
    return min(FL_NSMAX, (FL_SMEM_MAX - smem_fixed(d, ncols)) // slot_bytes(d))


def ncols(B):
    return 16 if B > 8 else 8


def cross_groups(n_keys, d, B):
    """the sizes of the groups of K slots the cross attention of n_keys keys is scored in (GS = min(FL_WARPS, NS))"""
    cr = slot_rows(d)
    nkc = -(-n_keys // cr)
    gs = min(FL_WARPS, ring_slots(d, ncols(B)))
    return [min(gs, nkc - c0) for c0 in range(0, nkc, gs)]


def width(model):
    return synth.MODELS[model[:-3] if model.endswith("-sc") else model].n_text_state


def test_ring_slots_table():
    """the slot counts of the GPU file's table, and every one of them holds a round of V slots (flowSupported: NS >= 5)"""
    for nc, row in NS_TABLE.items():
        assert tuple(ring_slots(d, nc) for d in WIDTHS) == row, nc
    assert all(slot_rows(d) == (slot_bytes(d) // 128) & ~7 for d in WIDTHS)
    assert min(min(r) for r in NS_TABLE.values()) >= 5
    assert [d for d in WIDTHS for nc in (8, 16) if ring_slots(d, nc) < FL_WARPS] == [1280]
    assert cross_groups(1500, 1280, 16) == [7, 3] and cross_groups(1121, 1280, 9) == [7, 1] and cross_groups(1500, 1280, 1) == [8, 2]


def test_cases_cover_the_shapes():
    cases = [(width(model), B, threads, n) for model, B, threads, n in CASES]
    assert {d for d, *_ in cases} == set(WIDTHS)
    for d in (128, 768, 1280):
        assert {ncols(B) for dd, B, *_ in cases if dd == d} == {8, 16}, d
    assert any(B == FLOW_MAX_B for d, B, *_ in cases)
    # the 7-slot ring, and its cross attention ending in a partial group
    narrow = [(d, B, n) for d, B, _, n in cases if ring_slots(d, ncols(B)) < FL_WARPS]
    assert narrow and any(cross_groups(n, d, B)[-1] < min(FL_WARPS, ring_slots(d, ncols(B))) for d, B, n in narrow)
    assert any(cross_groups(n, d, B) == [7, 1] for d, B, n in narrow)
    # a prompt chunk that straddles two 16-column tiles of the per-op skinny GEMM
    assert any((PROMPT_N * b) // SKINNY_COLS != (PROMPT_N * b + PROMPT_N - 1) // SKINNY_COLS
               for d, B, *_ in cases for b in range(B)) and SKINNY_COLS % PROMPT_N
    # the numpy slots reach both edges of each n-tile; the permutations move columns 0..7 into the second tile
    assert checked_slots(768, 16) == [0, 7, 8, 15] and checked_slots(1280, 9) == [0, 7, 8]
    perm = dict(orders(16))["rotated by 8"]
    assert sorted(perm) == list(range(16)) and all(perm.index(k) >= 8 for k in range(8))
    assert CALLS[0] == (0, PROMPT_N) and len(CALLS) == 1 + N_STEPS and NPOS == sum(n for _, n in CALLS)


# ---- mutations ----------------------------------------------------------------------------------------------------------------------
CROSS_KEYS = 64
THREADS = 4
_cache = {}


def short_cross(m, seed, n=CROSS_KEYS):
    """whisper_np.encode of a clip at audio_ctx n: the window's first 2n mel frames and positional rows [0, n)"""
    mm = copy.copy(m)
    mm.t = dict(m.t)
    mm.n_audio_ctx = n
    mm.t["encoder.positional_embedding"] = m["encoder.positional_embedding"][:n]
    _, ck, cv = wn.encode(mm, wn.log_mel(synth.synth_pcm(seed), m.filters))
    return ck, cv


def setup(name):
    """two chunks' NpModel, cross-K/V, tokens and unmutated oracle results"""
    if name not in _cache:
        m = wn.NpModel(synth.model_path(name))
        cross = {b: short_cross(m, PCM_SEED + b) for b in range(2)}
        tokens = [t[:CALLS[-1][0] + 1] for t in chunk_tokens(m.token_sot, m.token_eot, 2, 3002)]
        _cache[name] = (m, cross, tokens, run_oracle(m, cross, tokens, THREADS))
    return _cache[name]


def deviation(got, want):
    """(failures, largest error / tolerance) of the GPU file's comparison of slot 0"""
    return compare(got, want, "slot 0")


def test_unmutated_passes():
    m, cross, tokens, want = setup("micro.en-sc")
    again = run_oracle(m, cross, tokens, THREADS)
    for b in range(2):
        bad, worst = deviation(again[b], want[b])
        assert not bad and worst == 0.0


def mutated(name, mut):
    m, cross, tokens, want = setup(name)
    if mut == "swap":                                    # the oracles of slots 0 and 1 exchanged
        return want[1]
    if mut == "token":                                   # chunk 0's third step fed chunk 1's token
        p = PROMPT_N + 2
        assert tokens[0][p] != tokens[1][p]
        t = [list(tokens[0])]
        t[0][p] = tokens[1][p]
        return run_oracle(m, {0: cross[0]}, t, THREADS)[0]
    if mut == "cross":                                   # chunk 0 decoded on chunk 1's cross-K/V
        return run_oracle(m, {0: cross[1]}, tokens, THREADS)[0]
    raise ValueError(mut)


@pytest.mark.parametrize("mut", ["swap", "token", "cross"])
def test_mutation_is_caught(mut):
    _, _, _, want = setup("micro.en-sc")
    bad, worst = deviation(mutated("micro.en-sc", mut), want[0])
    assert bad, "%s: not caught (largest deviation %.3g of its tolerance)" % (mut, worst)


def test_cross_swap_is_caught_on_small():
    """the random-weight small model (d = 768), whose encoder output barely depends on the clip"""
    _, _, _, want = setup("small")
    bad, worst = deviation(mutated("small", "cross"), want[0])
    assert bad, "not caught (largest deviation %.3g of its tolerance)" % worst

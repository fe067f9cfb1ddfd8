#!/usr/bin/env python
"""Generate tests/golden/chunks_eot.npz from oracle/_ref — the reference's own CPU implementation — for wsp_run_chunks_until_eot: every
chunk of a batch decoded greedily until its first EOT or a cap of CAP tokens.

Each chunk runs through the reference on its own, with the prompt and first-step rules of make_golden.py's chunk fixtures: the prompt
of prompt_of(), the first token by whisper_sample_timestamp(initial), then whisper_sample_best until the sampled token is EOT or CAP
tokens have been sampled.  Stored per chunk: the tokens (EOT included), the EOT step (n_out; 0 in "eot_step" = no EOT before the cap)
and the reference's top-2 logit margin at every step but the forced first one.

On the scripted models (whisper_b200/synth.py) a 30 s clip follows its script to EOT after 45 tokens.  A clip a little shorter than
30 s is zero-padded up to the window: the encoder's response to the silent tail moves the decoder off its script, so such clips end at
other steps or never (they repeat a short loop up to the cap).  Candidates are (PCM chunk id, clip length) pairs, tried in a fixed order;
a candidate is kept when its margin is >= GAP_SAFE at every step of its output at every thread count of the case.  A batch must hold
at least two distinct EOT steps and at least one chunk that reaches the cap; the generator fails instead of writing a weaker batch.

base.en-sc and medium-sc are not cases here: their 30 s clips rarely keep the margin over 45 steps, and the CPU reference needs about
a minute per medium candidate.  tests/test_gpu_chunks_eot.py runs both against the GPU's own fixed-length decode instead.

    python tests/golden/make_chunks_eot_golden.py [case ...]   # rewrites tests/golden/chunks_eot.npz (a few minutes)
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

from tests.golden.make_golden import GAP_SAFE, prompt_of, top2_gap  # noqa: E402
from whisper_b200 import synth  # noqa: E402

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "chunks_eot.npz")

CAP = 72                                           # max_decode of every case
# clip lengths tried for each chunk id, in this order (samples at 16 kHz); where a model leaves its script depends on the model
LENGTHS = (440000, 420000, 480000, 400000, 430000, 410000, 390000, 360000)
CHUNK_TRIES = 24
CASES = {
    # name: (model, reference threads, batch)
    "micro_en": ("micro.en-sc", (1, 4), 4),
    "micro_ml": ("micro-sc", (1, 4), 4),           # multilingual specials: EOT is 50257
}


def until_eot(o, prompt, cap):
    """o: a RefOracle with the chunk encoded.  Returns the tokens up to and including the first EOT (at most cap) and the top-2
    margins of steps 2..n."""
    eot = o.special["eot"]
    o.decode(prompt, 0)
    toks, gaps = [o.sample(initial=True, force_timestamp=True)["id"]], []
    while toks[-1] != eot and len(toks) < cap:
        lg, _ = o.decode([toks[-1]], len(prompt) + len(toks) - 1)
        gaps.append(top2_gap(lg[0]))
        toks.append(o.sample()["id"])
    return np.array(toks, np.int32), np.array(gaps, np.float32)


def candidates():
    for ch in range(CHUNK_TRIES):
        for n in LENGTHS:
            yield ch, n


def batch_ok(runs, eot, cap):
    """the properties a case's batch must have, at every thread count: >= 2 distinct EOT steps, >= 1 chunk at the cap, clean margins"""
    for toks, gaps in runs:
        ends = [len(t) for t in toks if t[-1] == eot]
        if len(set(ends)) < 2 or not any(len(t) == cap and t[-1] != eot for t in toks):
            return False
        if min(float(g.min()) for g in gaps) < GAP_SAFE:
            return False
    return True


def make_case(name):
    from oracle.ref import RefOracle
    model, threads, batch = CASES[name]
    path = synth.model_path(model)
    oracles = {th: RefOracle(path, threads=th) for th in threads}
    o0 = oracles[threads[0]]
    eot, prompt = o0.special["eot"], prompt_of(o0)
    kept = []        # (chunk, n_samples, {th: (tokens, gaps)})
    for ch, n in candidates():
        mel = o0.pcm_to_mel(synth.synth_pcm(ch, n))
        rs = {}
        for th, o in oracles.items():
            o.set_mel(mel)
            o.encode(0)
            rs[th] = until_eot(o, prompt, CAP)
        gap = min(float(g.min()) for _t, g in rs.values())
        ends = sorted({len(t) if t[-1] == eot else 0 for t, _g in rs.values()})
        ok = gap >= GAP_SAFE
        print("  %s chunk %d, %d samples: n_out %s, min gap %.3f %s" % (name, ch, n, ends, gap, "keep" if ok else "skip"), flush=True)
        if ok:
            kept.append((ch, n, rs))
        chosen = choose(kept, eot, batch, threads)
        if chosen:
            break
    else:
        raise RuntimeError("%s: no batch of %d clean chunks with two EOT steps and one chunk at the cap in %d candidates"
                           % (name, batch, CHUNK_TRIES * len(LENGTHS)))
    out = {name + "_chunks": np.array([c[0] for c in chosen], np.int32),
           name + "_n_samples": np.array([c[1] for c in chosen], np.int32),
           name + "_prompt": np.array(prompt, np.int32), name + "_eot": np.int32(eot), name + "_cap": np.int32(CAP),
           name + "_threads": np.array(threads, np.int32)}
    for th in threads:
        toks = np.full((batch, CAP), -1, np.int32)
        gaps = np.full((batch, CAP - 1), np.nan, np.float32)
        n_out = np.zeros(batch, np.int32)
        eot_step = np.zeros(batch, np.int32)
        for b, (_ch, _n, rs) in enumerate(chosen):
            t, g = rs[th]
            toks[b, :t.size] = t
            gaps[b, :g.size] = g
            n_out[b] = t.size
            eot_step[b] = t.size if t[-1] == eot else 0
        pre = "%s_t%d_" % (name, th)
        out[pre + "tokens"], out[pre + "gap"], out[pre + "n_out"], out[pre + "eot_step"] = toks, gaps, n_out, eot_step
    return out


def choose(kept, eot, batch, threads):
    """a batch from the kept candidates: one that reaches the cap and one per EOT step first, the rest in the order they were found"""
    if len(kept) < batch:
        return None
    th = threads[0]
    picked, steps = [], set()
    for k in kept:
        t = k[2][th][0]
        if t[-1] != eot and not any(p[2][th][0][-1] != eot for p in picked):
            picked.append(k)
        elif t[-1] == eot and t.size not in steps:
            steps.add(t.size)
            picked.append(k)
    picked = picked[:batch]
    picked += [k for k in kept if not any(k is p for p in picked)][:batch - len(picked)]
    runs = [([k[2][t][0] for k in picked], [k[2][t][1] for k in picked]) for t in threads]
    return picked if batch_ok(runs, eot, CAP) else None


if __name__ == "__main__":
    names = sys.argv[1:] or list(CASES)       # a subset of the cases is merged into the existing file
    new = {}
    for nm in names:
        new.update(make_case(nm))
    data = dict(np.load(OUT)) if os.path.exists(OUT) and len(names) < len(CASES) else {}
    data.update(new)
    np.savez_compressed(OUT, **data)
    print("chunks_eot %.0f KB" % (os.path.getsize(OUT) / 1024), flush=True)

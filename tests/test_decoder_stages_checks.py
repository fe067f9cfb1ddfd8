"""The checks of tests/test_gpu_decoder_stages.py have teeth: on micro.en (random weights) a decoder pass simulated with the stage
restatements themselves meets every check exactly, and each plausible kernel bug, applied to it, fails the check of the op it hits.
Also pins the restatements to the reference: the f16-table exp by the reference's rule (double -> f32 -> f16) at every input the
vocabulary softmax can see, and the side-by-side V^T·P chains to wn.pv_mad_f16."""
import copy

import numpy as np

from oracle import whisper_np as wn
from tests.test_gpu_decoder_stages import (N_TEXT_CTX, SCALE, Check, DecWeights, check_attention, check_embedding, check_layer, check_logits,
                                           check_probs, pv_chains, ref_attention, ref_cross_q, ref_embedding, ref_fc1, ref_logits,
                                           ref_qkv, ref_resid, table_exp, table_row)
from whisper_b200 import synth

F16, F32, F64 = np.float16, np.float32, np.float64
B, N, N_PAST, THREADS, T = 2, 5, 400, 4, 40


def cross_memories(W, seed):
    """per chunk (K, V) [L][H][T][64] of f16 values"""
    rng = np.random.default_rng(seed)
    return [tuple(wn.r16(rng.standard_normal((W.L, W.H, T, 64)) * s).astype(F64) for s in (0.7, 1.0)) for _ in range(B)]


def sim_run(W, tokens, ck):
    """What a correct pass returns: per layer the tensors check_layer reads, built from the op restatements themselves."""
    d, H, L = W.d, W.H, W.L
    rng = np.random.default_rng(5)
    caches = []
    for _ in range(B):
        # small cached keys and values around 6: nearly uniform probabilities over long chains whose sums grow to where the f16
        # rounding of every step shows how the threads split the keys
        kv = [np.zeros((L, H, N_TEXT_CTX, 64)) for _ in range(2)]
        for a, s, mean in zip(kv, (0.05, 1.0), (0.0, 6.0)):
            a[:, :, :N_PAST] = wn.r16(rng.standard_normal((L, H, N_PAST, 64)) * s + mean)
        caches.append(tuple(kv))
    nkv = N_PAST + np.arange(N) + 1
    x = np.stack([ref_embedding(W, tokens[b], N_PAST)[0] for b in range(B)])
    run = {"emb": x, "layers": []}
    for il in range(L):
        t = {"x_in": x, "kv_before": caches}
        caches = copy.deepcopy(caches)
        q0 = []
        for b in range(B):
            (q, _), (k, _), (v, _) = ref_qkv(W, il, x[b])
            q0.append(q)
            for cache, rows in zip(caches[b], (k, v)):
                cache[il, :, N_PAST:N_PAST + N] = rows.reshape(N, H, 64).transpose(1, 0, 2)
        t["kv_after"] = caches
        t["q0"] = np.stack(q0)
        t["attn1"] = ref_attention(t["q0"], np.stack([c[0][il] for c in caches]), np.stack([c[1][il] for c in caches]), nkv, N_PAST + N,
                                   THREADS)[0]
        t["x2"] = np.stack([ref_resid(W.blk(il, "attn.out.weight"), W.blk(il, "attn.out.bias"), x[b], t["attn1"][b])[0] for b in range(B)])
        t["q3"] = np.stack([ref_cross_q(W, il, t["x2"][b])[0] for b in range(B)])
        t["attn4"] = ref_attention(t["q3"], np.stack([k[il] for k, _ in ck]), np.stack([v[il] for _, v in ck]), np.full(N, T), T, THREADS)[0]
        t["x5"] = np.stack([ref_resid(W.blk(il, "cross_attn.out.weight"), W.blk(il, "cross_attn.out.bias"), t["x2"][b], t["attn4"][b])[0]
                            for b in range(B)])
        t["h6"] = np.stack([ref_fc1(W, il, t["x5"][b])[0] for b in range(B)])
        t["x7"] = np.stack([ref_resid(W.blk(il, "mlp.2.weight"), W.blk(il, "mlp.2.bias"), t["x5"][b], t["h6"][b])[0] for b in range(B)])
        x = t["x7"]
        run["layers"].append(t)
    run["x"] = x
    run["logits"] = np.stack([ref_logits(W, x[b, N - 1:])[0] for b in range(B)])
    run["all_logits"] = np.stack([ref_logits(W, x[b])[0] for b in range(B)])
    lg = run["all_logits"].reshape(B * N, -1).astype(F32)
    run["probs"] = wn.softmax_rows(lg)
    return run


def check_run(W, run, tokens, ck):
    chk = Check(record=False)
    check_embedding(W, chk, tokens, N_PAST, run["emb"])
    for il, t in enumerate(run["layers"]):
        check_layer(W, chk, t, il, il - 1, N_PAST, N)
    check_attention(chk, [(il, t, tuple(np.stack([m[i][il] for m in ck]) for i in (0, 1))) for il, t in enumerate(run["layers"])],
                    N_PAST, N, THREADS)
    check_logits(W, chk, "logits", run["x"][:, N - 1:], run["logits"])
    check_logits(W, chk, "all logits", run["x"], run["all_logits"])
    check_probs(chk, run["all_logits"].reshape(B * N, -1), run["probs"])
    return chk


def test_table_exp_follows_the_reference_rule():
    """wn.softmax_rows rounds exp in double straight to f16, the reference's table goes through f32 first (ggml.c:1382): at all
    31 744 finite f16 inputs <= 0 the two agree, and the exhaustive row of the GPU test is that table scaled by 1 / sum."""
    x = np.arange(0x8000, 0xFC00, dtype=np.uint16).view(F16).astype(F64)
    e = np.exp(x)
    assert np.array_equal(e.astype(F16), e.astype(F32).astype(F16))
    row = table_row(51864)
    tab = table_exp(row.astype(F64))
    want = (tab * (1.0 / tab.sum()).astype(F32)).astype(F32)
    assert np.array_equal(wn.softmax_rows(row), want)


def test_stage_checks_catch_mutations():
    W = DecWeights(synth.model_path("micro.en"))
    H, d, L = W.H, W.d, W.L
    rng = np.random.default_rng(3)
    tokens = rng.integers(0, 50256, (B, N))
    ck = cross_memories(W, 4)
    run = sim_run(W, tokens, ck)
    nkv = N_PAST + np.arange(N) + 1

    # the side-by-side chains are wn.pv_mad_f16's, key by key
    t = run["layers"][1]
    for q, K, V, keys, n_all in ((t["q0"][0], t["kv_after"][0][0][1], t["kv_after"][0][1][1], nkv, N_PAST + N),
                                 (t["q3"][1], ck[1][0][1], ck[1][1][1], np.full(N, T), T)):
        S = np.einsum("hqd,hkd->hqk", wn.r16(q).reshape(N, H, 64).transpose(1, 0, 2), K[:, :n_all].astype(F32)).astype(F32)
        valid = np.arange(n_all)[None, :] < keys[:, None]
        P = wn.softmax_rows(np.where(valid[None], S, -np.inf).astype(F32))
        for threads in (1, 3, THREADS, 16):
            got = pv_chains(P[None].astype(F64), np.zeros((1,) + P.shape), V[None, :, :n_all], valid, threads, -(-n_all // threads))[0][0]
            assert np.array_equal(got, wn.r16(wn.pv_mad_f16(P, V[:, :n_all], threads)))

    chk = check_run(W, run, tokens, ck)
    assert not chk.fails, [f[2] for f in chk.fails]

    def mutated(fn):
        r = copy.deepcopy(run)
        fn(r)
        return check_run(W, r, tokens, ck)

    def attn(r, il, b, q, **kw):
        t = r["layers"][il]
        a = dict(keys=nkv, n_all=N_PAST + N, threads=THREADS)
        a.update(kw)
        if "per_query" in kw:
            return np.concatenate([ref_attention(q[None, i:i + 1], t["kv_after"][b][0][il][None], t["kv_after"][b][1][il][None],
                                                 a["keys"][i:i + 1], int(a["keys"][i]), THREADS)[0][0] for i in range(N)])
        return ref_attention(q[None], t["kv_after"][b][0][il][None], t["kv_after"][b][1][il][None], a["keys"], a["n_all"], a["threads"])[0][0]

    last = N_PAST + N - 1

    def wrong_position(r):          # the embedding adds the positional row of the next position
        r["emb"][1] = r["emb"][1] + W["decoder.positional_embedding"][N_PAST + 1:N_PAST + N + 1] - W["decoder.positional_embedding"][N_PAST:N_PAST + N]
    assert mutated(wrong_position).failed("embedding", 1)

    def q_bias_band(r):             # Q columns 32..63 of head 0 without their bias
        r["layers"][0]["q0"][0][:, 32:64] -= W.blk(0, "attn.query.bias")[32:64] * SCALE
    assert mutated(q_bias_band).failed("qkv", 0)

    def k_unscaled(r):              # head 1's K rows stored without the 64^-0.25
        Ka = r["layers"][3]["kv_after"][0][0]
        Ka[3, 1, N_PAST:N_PAST + N] = wn.r16(Ka[3, 1, N_PAST:N_PAST + N] / SCALE)
    assert mutated(k_unscaled).failed("qkv", 0)

    def k_next_position(r):         # the last token's K row written at position + 1
        Ka = r["layers"][1]["kv_after"][1][0]
        Ka[1, :, last + 1] = Ka[1, :, last]
        Ka[1, :, last] = r["layers"][1]["kv_before"][1][0][1, :, last]
    chk = mutated(k_next_position)
    assert chk.failed("qkv", 1) and chk.failed("kv-cache", 1)

    def v_into_chunk0(r):           # chunk 1's V rows written into chunk 0
        t = r["layers"][2]
        t["kv_after"][0][1][2, :, N_PAST:N_PAST + N] = t["kv_after"][1][1][2, :, N_PAST:N_PAST + N]
    chk = mutated(v_into_chunk0)
    assert chk.failed("qkv", 0) and not chk.failed("qkv", 1)

    def v_previous_position(r):     # the first token's V row also written one position early
        Va = r["layers"][2]["kv_after"][1][1]
        Va[2, :, N_PAST - 1] = Va[2, :, N_PAST]
    assert mutated(v_previous_position).failed("kv-cache", 1)

    def mask_off_by_one(r):         # every query sees one key more
        t = r["layers"][0]
        t["attn1"][1] = wn.r16(attn(r, 0, 1, t["q0"][1], keys=nkv + 1))
    assert mutated(mask_off_by_one).failed("self attention", 1)

    def split_per_query(r):         # the threads split each query's own keys instead of the call's
        for il in range(L):
            t = r["layers"][il]
            t["attn1"][0] = wn.r16(attn(r, il, 0, t["q0"][0], per_query=True))
    assert mutated(split_per_query).failed("self attention", 0)

    def self_out_bias(r):           # the self-attention out-projection without bias on columns 64..95
        r["layers"][2]["x2"][1][:, 64:96] -= W.blk(2, "attn.out.bias")[64:96]
    assert mutated(self_out_bias).failed("self-out", 1)

    def cross_q_unscaled(r):        # the cross query without the 64^-0.25
        r["layers"][1]["q3"][0] /= SCALE
    assert mutated(cross_q_unscaled).failed("cross q", 0)

    def cross_other_chunk(r):       # chunk 0 attends over chunk 1's cross memory
        t = r["layers"][3]
        t["attn4"][0] = wn.r16(ref_attention(t["q3"][None, 0], ck[1][0][None, 3], ck[1][1][None, 3], np.full(N, T), T, THREADS)[0][0])
    chk = mutated(cross_other_chunk)
    assert chk.failed("cross attention", 0) and not chk.failed("cross attention", 1)

    def cross_out_from_input(r):    # the cross out-projection added to the layer's input instead of the self-attention's output
        t = r["layers"][0]
        t["x5"][0] = ref_resid(W.blk(0, "cross_attn.out.weight"), W.blk(0, "cross_attn.out.bias"), t["x_in"][0], t["attn4"][0])[0]
    assert mutated(cross_out_from_input).failed("cross-out", 0)

    def ln_swapped_block(r):        # the MLP LayerNorm's gamma and beta exchanged on columns 0..127
        t = r["layers"][2]
        g, b = W.blk(2, "mlp_ln.weight").copy(), W.blk(2, "mlp_ln.bias").copy()
        W2 = copy.copy(W)
        W2.m = copy.copy(W.m)
        W2.m.t = dict(W.m.t)
        W2.m.t["decoder.blocks.2.mlp_ln.weight"], W2.m.t["decoder.blocks.2.mlp_ln.bias"] = b, g
        t["h6"][1] = ref_fc1(W2, 2, t["x5"][1])[0]
    assert mutated(ln_swapped_block).failed("fc1", 1)

    def fc2_bias(r):                # fc2 without bias on columns 0..31
        r["layers"][3]["x7"][0][:, :32] -= W.blk(3, "mlp.2.bias")[:32]
    assert mutated(fc2_bias).failed("fc2", 0)

    def first_column(r):            # the logits of chunk b from column b N instead of b N + N - 1
        r["logits"][1] = ref_logits(W, r["x"][1, :1])[0]
    assert mutated(first_column).failed("logits", 1)

    def rows_swapped(r):            # all-logits rows of chunk 0 in the wrong order
        r["all_logits"][0] = r["all_logits"][0][::-1]
    assert mutated(rows_swapped).failed("all logits", 0)

    def prob_ulp(r):                # one probability one ulp off
        p = r["probs"]
        p[3, 77] = np.nextafter(p[3, 77], F32(1))
    assert mutated(prob_ulp).failed("probs", 3)

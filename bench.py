#!/usr/bin/env python
"""bench.py — audio-seconds per wall-second of the Whisper hot path on H100 (BASELINE.json metric).

    python bench.py [--gpus N] [--steps K] [--warmup W] [--dump-outputs DIR]   # this engine
    python bench.py --impl reference [--gpus N] [--steps K] [--warmup W] # the reference's own CPU path on the host cores
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N ... bench.py --gpus N ...   # N > 1, one rank per GPU

One "step" = one pass of the hot path over one batch of synthetic input per GPU: `batch` independent 30 s chunks of 16 kHz
PCM -> log-mel -> encoder -> cross-KV -> prompt + n_decode greedy decoder steps (timestamp rules, tokens fed back on the device).
Workload = BASELINE.json configs[2]: ggml-medium shapes (synthetic "scripted" weights, seed 1234: whisper_b200/synth.py), batch 8 per GPU, beam 1,
100 tokens.  Every rank's chunks are those of the committed parity fixture of this configuration (the reference's greedy tokens at the
reference thread count the decoder reproduces), and the line says whether the tokens of every rank matched.

  value : whole-job audio-s/s with the PCM already resident in HBM (wsp_upload_pcm + wsp_run_chunks_resident) — the log-mel
          front end, encoder and decoder all run inside the timed region; device time from CUDA events on the launching stream.
  e2e   : the same through the public C-ABI call with HOST buffers (wsp_run_chunks): pinned PCM -> H2D every step, tokens D2H.
  roofline: the dominant kernel (decode_flow_kernel: the single-launch dataflow decoder step) against the HBM peak
          (MEASURED_PEAKS.json when present, else the H100 SXM data sheet's 3.35 TB/s); its per-launch duration is measured live by an
          instrumented decoder pass (CUDA event pair around every launch).
  cpu_baseline: oracle/_ref (the reference's unmodified ggml.c + whisper.cpp) on this box's host cores, bounded sample.

--dump-outputs DIR: after the timed steps, rank 0 writes what the last timed step returned — tokens.npy ([batch, n_decode] token ids
as float64) and last_logits.npy ([batch, n_vocab] float32 logits of the final decoder step).  Inputs are seeded, so two builds run with
the same arguments can be compared output for output.

Multi-GPU: chunks are independent, so ranks shard the batch with no data-path collective ("weak" scaling: batch per GPU fixed).
The only collective is the NCCL broadcast of the ggml file image at load (rank 0 reads the file once).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

METRIC = "audio-sec/s (RTF) medium 30s chunks @1/2/4/8 H100 vs reference CPU path"
UNIT = "audio-s/s"
CHUNK_SECONDS = 30.0


def parse_args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--model", default="medium-sc", help="synthetic model (whisper_b200/synth.py); -sc = scripted weights, same shapes and arithmetic")
    ap.add_argument("--batch", type=int, default=8, help="chunks per GPU per step")
    ap.add_argument("--n-decode", type=int, default=100, help="greedy tokens per chunk (BASELINE.md §2)")
    ap.add_argument("--ref-threads", type=int, default=0, help="reference arm: CPU threads (0 = min(cores, 16))")
    ap.add_argument("--arith-threads", type=int, default=0,
                    help="reference thread count whose V^T*P arithmetic the decoder reproduces (the reference's result depends on its thread count, "
                         "ggml.c:4680-4722).  0 = 16 — what the reference arm and the cpu_baseline leg run with on this box — when the parity "
                         "fixture of the configuration is pinned at 16 threads, else 4 (the reference's default)")
    ap.add_argument("--chunk-base", type=int, default=-1, help="debug: use synthetic chunks base .. base+B-1 instead of the fixture's (no token check)")
    ap.add_argument("--no-cpu-baseline", action="store_true", help="skip the reference CPU leg (model sweeps; the default run keeps it)")
    ap.add_argument("--ref-tokens", type=int, default=12, help="reference arm: decoder tokens actually run per sample")
    ap.add_argument("--dump-outputs", default=None, metavar="DIR", help="write the last timed step's outputs to DIR/<name>.npy")
    return ap.parse_args()


def workload_name(a):
    return "ggml-%s shapes (synthetic weights seed 1234), batch=%d independent 30 s chunks per GPU, greedy beam=1, n_decode=%d" % (a.model, a.batch, a.n_decode)


def decoder_weight_bytes(m):
    d, L = m.n_text_state, m.n_text_layer
    return L * 14 * d * d * 2 + m.n_vocab * d * 2   # SURVEY.md §8(d): read once per step regardless of batch


def hbm_peak():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        try:
            return float(json.load(open(p))["hbm_gbs"]), "measured (MEASURED_PEAKS.json)"
        except Exception:
            pass
    return 3350.0, "H100 SXM data sheet (not measured)"


def _jsonable(o):
    if isinstance(o, dict):
        return {k: _jsonable(v) for k, v in o.items()}
    if isinstance(o, (list, tuple)):
        return [_jsonable(v) for v in o]
    if isinstance(o, np.generic):
        return o.item()
    return o


class ClockSampler:
    """nvidia-smi clocks / throttle reasons DURING the timed region."""

    def __init__(self, index):
        self.index, self.rows, self.proc = index, [], None

    def start(self):
        q = "clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"
        try:
            self.proc = subprocess.Popen(["nvidia-smi", "-i", str(self.index), "--query-gpu=" + q, "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.rows.append([x.strip() for x in line.split(",")])

    def stop(self):
        if not self.proc:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            self.proc.kill()
        sm, mx, reasons = [], [], set()
        names = ["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"]
        for r in self.rows:
            try:
                sm.append(float(r[0])); mx.append(float(r[1]))
                for n, v in zip(names, r[3:7]):
                    if v.lower().startswith("active"):
                        reasons.add(n)
            except Exception:
                pass
        return {"sm_mhz": float(np.median(sm)) if sm else None, "sm_max_mhz": max(mx) if mx else None, "reasons": sorted(reasons), "samples": len(sm)}


# ---------------------------------------------------------------------------------------------------------------------
def reference_sample(model_name, threads, n_tokens, n_decode):
    """One sample of the workload on the host: one chunk — log-mel + encoder + prompt + (n_tokens-1) decoder steps with the reference's own
    code.  n_tokens == n_decode: everything is MEASURED; n_tokens < n_decode (only the numpy-port fallback does that): the decode time is
    scaled to n_decode tokens and the detail says so.  Returns (audio_s_per_s, detail dict)."""
    from whisper_b200 import synth
    from oracle import ref
    path = synth.model_path(model_name)
    if ref.available():
        o = _REF_CACHE.get("o")
        if o is None:
            o = ref.RefOracle(path, threads=threads)
            _REF_CACHE["o"] = o
        prompt = [o.special["sot"]] + ([o.special["sot"] + 1, o.special["transcribe"]] if o.n_vocab == 51865 else [])
        wall, toks, st = o.bench_chunk(synth.synth_pcm(0), prompt, n_tokens, threads=threads)
        kind = "reference"
    else:
        # oracle port (numpy restatement), only when the reference library did not travel
        from oracle import whisper_np as wn
        m = _REF_CACHE.get("m") or wn.NpModel(path)
        _REF_CACHE["m"] = m
        pcm = synth.synth_pcm(0)
        t0 = time.time(); mel = wn.log_mel(pcm, m.filters)
        t1 = time.time(); out, ck, cv = wn.encode(m, mel)
        t2 = time.time()
        dec = wn.NpDecoder(m, ck, cv, pv_threads=4)
        prompt = [m.token_sot] + ([m.token_sot + 1, 50359] if m.n_vocab == 51865 else [])
        cur, n_past = prompt, 0
        for _ in range(n_tokens):
            lg, pr = dec.decode(cur, n_past)
            n_past += len(cur)
            cur = [wn.sample_best(m, pr[-1])["id"]]
        t3 = time.time()
        st = [(t1 - t0) * 1e3, (t2 - t1) * 1e3, (t3 - t2) * 1e3]
        kind = "port"
    per_tok = st[2] / n_tokens
    total_s = (st[0] + st[1] + per_tok * n_decode) / 1e3
    return CHUNK_SECONDS / total_s, dict(kind=kind, mel_ms=st[0], encode_ms=st[1], decode_ms_per_token=per_tok, sampled_tokens=n_tokens,
                                         extrapolated=n_tokens != n_decode, threads=threads)


_REF_CACHE = {}


def reference_thread_candidates(cores):
    """SURVEY.md §8(d): ggml spawns and joins its threads for every graph and spin-waits between ops, so more threads are not reliably
    faster — try the reference's default (4), 16 and all cores, keep the fastest."""
    return sorted({min(4, cores), min(16, cores), cores})


def run_reference(a):
    rank = int(os.environ.get("RANK", "0"))
    if rank != 0:
        return 0
    from oracle import ref
    from whisper_b200 import synth
    synth.model_path(a.model)
    cores = os.cpu_count() or 1
    budget_s = 240.0
    t_begin = time.time()
    full = ref.available()                       # the real reference is fast enough to run the whole workload: nothing is extrapolated
    n_tok = a.n_decode if full else a.ref_tokens
    # calibration = warm-up: one full sample per candidate thread count (the fastest one is used for the timed steps)
    cands = [a.ref_threads] if a.ref_threads else reference_thread_candidates(cores)
    calib = {}
    for th in cands:
        v, det = reference_sample(a.model, th, n_tok, a.n_decode)
        calib[th] = v
        if time.time() - t_begin > budget_s / 2:
            break
    threads = max(calib, key=calib.get)
    vals, det = [], None
    steps_done = 0
    t0 = time.time()
    while steps_done < a.steps:
        v, det = reference_sample(a.model, threads, n_tok, a.n_decode)
        vals.append(v)
        steps_done += 1
        one = (time.time() - t0) / steps_done
        if time.time() - t_begin + one > budget_s:
            break
    value = float(np.mean(vals))
    sample = ("1 chunk/step, MEASURED end to end: log-mel + full encoder + prompt + %d decoder tokens with the reference's whisper_pcm_to_mel / "
              "whisper_encode / whisper_decode / whisper_sample_best%s; %d of %d requested steps fit the %.0f s budget; thread counts tried "
              "(audio-s/s): %s" % (n_tok - 1, "" if not det["extrapolated"] else " (numpy port: decode time scaled to n_decode=%d)" % a.n_decode,
                                  steps_done, a.steps, budget_s, ", ".join("%d: %.2f" % (k, calib[k]) for k in sorted(calib))))
    line = {
        "impl": "reference", "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": a.gpus, "steps": steps_done, "warmup": len(calib),
        "ms_per_step": 1e3 * CHUNK_SECONDS / value, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f16 weights x f16-rounded activations, f32 accumulate (ggml CPU)",
        "data": "synthetic",
        "config": {"workload": workload_name(a), "l2": "inputs larger than L2 (n/a on CPU)",
                   "reference_arm": "ONE CPU process on this box's host cores whatever --gpus says (the reference's CPU path has no multi-GPU notion); "
                                    "a step is 1 chunk here vs %d chunks per GPU in the engine's arm — the metric (audio-s/s) is per-audio, so the lines compare" % a.batch},
        "cpu_baseline": {"value": value, "unit": UNIT, "cores": threads, "kind": det["kind"], "sample": sample,
                         "mel_ms": det["mel_ms"], "encode_ms": det["encode_ms"], "decode_ms_per_token": det["decode_ms_per_token"], "host_cores": cores},
        "e2e": {"value": value, "unit": UNIT, "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
    }
    print(json.dumps(_jsonable(line)), flush=True)
    return 0


# ---------------------------------------------------------------------------------------------------------------------
def run_ours(a):
    # stdout carries ONE JSON line: whatever libraries print to file descriptor 1 meanwhile (NCCL prints its version banner there)
    # is sent to stderr, and the line itself is written to the saved descriptor at the end
    sys.stdout.flush()
    real_stdout = os.dup(1)
    os.dup2(2, 1)
    try:
        return _run_ours(a, real_stdout)
    finally:
        sys.stdout.flush()
        os.dup2(real_stdout, 1)
        os.close(real_stdout)


def _run_ours(a, real_stdout):
    import torch
    import torch.distributed as dist
    from whisper_b200 import capi, synth

    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.cuda.set_device(local)
        dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    L = capi.lib()
    if L.wsp_device_count() < 1:
        raise SystemExit("bench.py: no CUDA device — whisper_b200 has no CPU fallback")

    # ---- load: rank 0 reads the ggml file once; peers get the host meta blob + the file image over NCCL (NVLink) ----
    t_load = time.time()
    if world == 1:
        model = capi.Model(synth.model_path(a.model))
        engine = capi.Engine(model, local)
        bcast_ms = 0.0
    else:
        from whisper_b200 import dist as wdist
        model, engine, bcast_ms = wdist.load_broadcast(a.model, rank, local, world)
    load_s = time.time() - t_load
    ctx = capi.Context(engine, a.batch)
    prompt = model.prompt_init()
    B, K, W = a.batch, a.steps, a.warmup

    # ---- inputs: distinct synthetic chunks per rank, pinned host memory for the e2e leg ----
    # rank 0 runs the very chunks of the committed parity fixture of this configuration (tests/golden/real_shapes.npz: the reference's
    # greedy tokens for 8 chunks x 32 steps of medium-sc), so the measured run is checked against the reference while it is measured
    chunk_ids = [rank * B + i for i in range(B)]
    fixture_tokens = None
    arith = a.arith_threads or 4
    try:
        fx = np.load(os.path.join(ROOT, "tests", "golden", "real_shapes.npz"))
        key = a.model.replace(".", "_").replace("-", "_")
        if key + "_chunks" in fx and len(fx[key + "_chunks"]) == B:
            if not a.arith_threads and key + "_t16_tokens" in fx:
                arith = 16
            pre = key + ("" if arith == 4 else "_t%d" % arith)
            # EVERY rank runs the chunks of the pinned configuration and is checked against the fixture (replicas: the chunks of
            # different GPUs are independent either way).  Chunks outside the calibrated family can throw the scripted decoder off its
            # script into rows whose top probability is shared, and every such row costs the sampler its exact std::partial_sort
            # emulation
            chunk_ids = [int(x) for x in fx[key + "_chunks"]]
            fixture_tokens = fx[pre + "_tokens"] if pre + "_tokens" in fx else None
    except Exception:
        pass
    if a.chunk_base >= 0:
        chunk_ids = [a.chunk_base + i for i in range(B)]
        fixture_tokens = None
    ctx.set_reference_threads(arith)
    pcms = [synth.synth_pcm(cid) for cid in chunk_ids]
    n_samp = pcms[0].size
    pinned = []
    for p in pcms:
        ptr = L.wsp_host_alloc(p.nbytes)
        if not ptr:
            raise SystemExit("wsp_host_alloc failed")
        C.memmove(ptr, p.ctypes.data, p.nbytes)
        pinned.append(ptr)
    ptrs = (C.POINTER(C.c_float) * B)(*[C.cast(p, C.POINTER(C.c_float)) for p in pinned])
    ns = np.full(B, n_samp, np.int32)
    for i, p in enumerate(pcms):
        ctx.upload_pcm(i, p)

    def barrier():
        if world > 1:
            dist.barrier()
        torch.cuda.synchronize()
        ctx_sync()

    def ctx_sync():
        capi.check(L.wsp_synchronize(ctx.h))

    def max_over_ranks(x):
        if world == 1:
            return x
        t = torch.tensor([x], dtype=torch.float64, device="cuda")
        dist.all_reduce(t, op=dist.ReduceOp.MAX)
        return float(t.item())

    # ---- warm-up (both paths) ----
    toks = None
    for _ in range(max(W, 3)):
        toks, _ = ctx.run_chunks_ptrs(ptrs, ns, B, prompt, a.n_decode)
    ctx.run_chunks_resident(B, prompt, a.n_decode)

    # ---- e2e leg: host PCM in, tokens out, through the public C-ABI call ----
    barrier()
    t0 = time.time()
    ctx.timer_start()
    for _ in range(K):
        toks, _ = ctx.run_chunks_ptrs(ptrs, ns, B, prompt, a.n_decode)
    e2e_ms_dev = ctx.timer_stop()
    barrier()
    e2e_wall = time.time() - t0
    e2e_ms = max_over_ranks(max(e2e_ms_dev, 0.0))
    e2e_wall = max_over_ranks(e2e_wall)

    # ---- value leg: PCM resident in HBM; clocks sampled during this region ----
    sampler = ClockSampler(local)     # every rank watches its own GPU; rank 0's sample goes into "clocks", the others into "per_rank"
    sampler.start()
    time.sleep(0.15)
    launches0 = L.wsp_launch_count()
    stage = np.zeros(3)
    barrier()
    ctx.timer_start()
    for _ in range(K):
        toks_r, st = ctx.run_chunks_resident(B, prompt, a.n_decode)
        stage += st
    val_ms_dev = ctx.timer_stop()
    barrier()
    launches = int(L.wsp_launch_count() - launches0)
    clocks = sampler.stop()
    val_ms = max_over_ranks(val_ms_dev)
    match_fixture = None
    if fixture_tokens is not None:
        match_fixture = bool((np.asarray(toks_r)[:, :fixture_tokens.shape[1]] == fixture_tokens[:, :a.n_decode]).all())
        match_fixture = max_over_ranks(0.0 if match_fixture else 1.0) == 0.0      # true only if every rank matched
    per_rank = None
    if world > 1:
        mine = torch.tensor([val_ms_dev / K, stage[0] / K, stage[1] / K, stage[2] / K, float(clocks.get("sm_mhz") or 0.0)], dtype=torch.float64, device="cuda")
        allr = [torch.zeros_like(mine) for _ in range(world)]
        dist.all_gather(allr, mine)
        per_rank = [{"rank": i, "ms_per_step": float(t[0]), "mel_ms": float(t[1]), "encode_ms": float(t[2]), "decode_ms": float(t[3]), "sm_mhz": float(t[4])}
                    for i, t in enumerate(allr)]
    same_tokens = bool((toks_r == toks).all())
    if a.dump_outputs and rank == 0:
        # what the last timed step returned; read back before the instrumented decoder pass below overwrites the logits
        os.makedirs(a.dump_outputs, exist_ok=True)
        np.save(os.path.join(a.dump_outputs, "tokens.npy"), np.asarray(toks_r, np.float64))
        np.save(os.path.join(a.dump_outputs, "last_logits.npy"), np.asarray(ctx.logits(B), np.float32))

    # ---- roofline of the dominant kernel: instrumented decoder pass (event pair around every launch) ----
    n_prof = 6
    ms_kind, n_kind = ctx.profile_decode(B, n_prof)
    wbytes = decoder_weight_bytes(model)
    peak, peak_src = hbm_peak()
    per_step = n_kind[0] / n_prof
    if per_step <= 1.5:
        # persistent decoder-step kernel: one launch = one token step for B chunks.  Algorithmic bytes (SURVEY.md §8d): decoder weights once
        # + per chunk the cross-KV memories (L*2*T*d*2) and the self-KV rows written so far.
        d, Ld, T = model.n_text_state, model.n_text_layer, model.n_audio_ctx
        n_past_avg = len(prompt) + a.n_decode + n_prof / 2.0
        cross_bytes = Ld * 2 * T * d * 2
        self_bytes = Ld * 2 * n_past_avg * d * 2
        bytes_per_launch = wbytes + B * (cross_bytes + self_bytes)
        ms_per_launch = ms_kind[0] / max(1, n_kind[0])
        kernel = "kern::decode_flow_kernel<%d> (dataflow decoder step: embedding + %d decoder layers + logits for %d chunks, one launch per token step)" % (d, Ld, B)
        detail = {"weights_bytes": wbytes, "cross_kv_bytes_per_chunk": cross_bytes, "self_kv_bytes_per_chunk": self_bytes}
    else:
        bytes_per_launch = wbytes / per_step
        ms_per_launch = ms_kind[0] / max(1, n_kind[0])
        kernel = "kern::skinny_gemm_kernel (decoder weight-streaming GEMM, 6 per layer + logits)"
        detail = {"launches_per_decoder_step": per_step}
    achieved = bytes_per_launch / (ms_per_launch * 1e-3) / 1e9
    roofline = {
        "kernel": kernel, "bound": "hbm", "achieved": achieved, "peak": peak, "unit": "GB/s", "frac": achieved / peak,
        "peak_source": peak_src, "bytes_per_launch": bytes_per_launch, "ms_per_launch": ms_per_launch,
        "decoder_step_ms_by_kind": {"decoder_kernel": ms_kind[0] / n_prof, "cross_attention": ms_kind[1] / n_prof, "self_attention": ms_kind[2] / n_prof, "sampler": ms_kind[3] / n_prof},
        "how": "wsp_profile_decode: %d un-graphed decoder steps, cudaEvent pair around every launch on the launching stream" % n_prof,
    }
    roofline.update(detail)

    total_audio = CHUNK_SECONDS * B * world * K
    value = total_audio / (val_ms * 1e-3)
    e2e_value = total_audio / (e2e_ms * 1e-3)

    cpu = None
    if rank == 0 and world == 1 and not a.no_cpu_baseline:
        cores = os.cpu_count() or 1
        threads = a.ref_threads or min(cores, 16)
        try:
            from oracle import ref as _ref
            n_tok = a.n_decode if _ref.available() else a.ref_tokens
            v, det = reference_sample(a.model, threads, n_tok, a.n_decode)
            cpu = {"value": v, "unit": UNIT, "cores": threads, "kind": det["kind"], "host_cores": cores,
                   "sample": "1 chunk of the same workload, measured end to end: log-mel + full encoder + prompt + %d decoder tokens%s" % (
                       n_tok - 1, " (decode time scaled to n_decode=%d)" % a.n_decode if det["extrapolated"] else ""),
                   "mel_ms": det["mel_ms"], "encode_ms": det["encode_ms"], "decode_ms_per_token": det["decode_ms_per_token"]}
        except Exception as ex:   # the bench line must still be printed
            cpu = {"value": None, "unit": UNIT, "cores": threads, "kind": "reference", "sample": "failed: %r" % (ex,)}

    if rank == 0:
        line = {
            "metric": METRIC, "value": value, "unit": UNIT, "n_gpus": world, "steps": K, "warmup": max(W, 3), "ms_per_step": val_ms / K,
            "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f16 (f16 weights x f16-rounded activations, f32 accumulate; KV f16)",
            "data": "synthetic",
            "config": {"workload": workload_name(a), "parallelism": "replicas x%d (independent chunks, no step-loop collective)" % world,
                       "chunks_per_step": B * world, "l2": "inputs larger than L2: every step streams 0.81 GB of decoder weights per token x %d tokens + 0.71 GB encoder weights" % a.n_decode,
                       "reference_threads_arithmetic": arith},
            "e2e": {"value": e2e_value, "unit": UNIT, "h2d_bytes_per_step": int(B * n_samp * 4 + B * len(prompt) * 4), "d2h_bytes_per_step": int(B * model.n_text_ctx * 4),
                    "ms_per_step": e2e_ms / K, "wall_ms_per_step": 1e3 * e2e_wall / K},
            "gpu_launches": launches,
            "roofline": roofline,
            "cpu_baseline": cpu,
            "clocks": clocks, "per_rank": per_rank,
            "stage_ms_per_step": {"mel": stage[0] / K, "encode": stage[1] / K, "decode": stage[2] / K},
            "load": {"seconds": load_s, "nccl_broadcast_ms": bcast_ms, "weight_bytes": engine.weight_bytes()},
            "tokens_equal_e2e_vs_resident": same_tokens,
            "tokens_match_reference_fixture": match_fixture,
        }
        os.write(real_stdout, (json.dumps(_jsonable(line)) + "\n").encode())
    for p in pinned:
        L.wsp_host_free(p)
    if world > 1:
        dist.barrier()
        dist.destroy_process_group()
    return 0


def main():
    a = parse_args()
    if a.impl == "reference":
        return run_reference(a)
    return run_ours(a)


if __name__ == "__main__":
    sys.exit(main())

"""ctypes binding of libwhisper_b200.so — the C ABI declared in include/whisper_b200.h.

This module is host-side plumbing for tests and bench.py (the reference is a C++ DLL; its real clients bind the COM
layer, see INTEGRATION.md).  There is no fallback: if the shared library is missing, importing the symbols fails loudly.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libwhisper_b200.so")

WSP_OK = 0
WSP_S_FALSE = 1
TOKEN_LANGUAGE_AUTO = -1   # WSP_TOKEN_LANGUAGE_AUTO: the prompt slot of each chunk's detected language (run_chunks*)
DECODE_FORCE_TIMESTAMP = 1
DECODE_INITIAL = 2
DECODE_ALL_LOGITS = 4
DECODE_DEVICE_TOKENS = 8
DECODE_NO_SAMPLE = 16


class TokenData(C.Structure):
    _fields_ = [("id", C.c_int32), ("tid", C.c_int32), ("p", C.c_float), ("pt", C.c_float), ("ptsum", C.c_float)]


class WindowParams(C.Structure):
    _fields_ = [("max_tokens", C.c_int32), ("single_segment", C.c_int32)]


class WindowResult(C.Structure):
    _fields_ = [("n_sampled", C.c_int32), ("n_tokens", C.c_int32), ("seek_delta", C.c_int32), ("failed", C.c_int32)]


class WindowSpan(C.Structure):
    _fields_ = [("slot", C.c_int32), ("offset_ms", C.c_int32), ("duration_ms", C.c_int32)]


class Segment(C.Structure):
    _fields_ = [("t0", C.c_int64), ("t1", C.c_int64), ("i0", C.c_int32), ("i1", C.c_int32)]


class TokenTime(C.Structure):
    _fields_ = [("t0", C.c_int64), ("t1", C.c_int64), ("vlen", C.c_float)]


class TokenTimeParams(C.Structure):
    _fields_ = [("thold_pt", C.c_float), ("thold_ptsum", C.c_float), ("max_len", C.c_int32)]


SEGMENT_SINGLE = 1          # wsp_window_segments flags
SEGMENT_PRINT_SPECIAL = 2
SEGMENT_SPEED_UP = 4

SPEAKER_UNSURE = 0          # wsp_chunk_speakers answers (iContext::detectSpeaker's eSpeakerChannel)
SPEAKER_LEFT = 1
SPEAKER_RIGHT = 2
SPEAKER_NO_STEREO = 255
SPEAKER_OUT_OF_RANGE = -1   # the segment starts outside the clip (the reference's E_BOUNDS)


class ReplicaStats(C.Structure):
    _fields_ = [("device", C.c_int32), ("batches_done", C.c_int32), ("chunks_done", C.c_int32), ("failed", C.c_int32), ("busy_ms", C.c_float), ("load_ms", C.c_float)]


# every symbol include/whisper_b200.h declares (tests/test_abi.py checks the .so exports each one)
EXPORTS = [
    "wsp_version", "wsp_last_error", "wsp_device_count", "wsp_device_name", "wsp_launch_count",
    "wsp_model_open", "wsp_model_close", "wsp_model_hparams", "wsp_model_special_tokens", "wsp_model_token_text",
    "wsp_model_is_multilingual", "wsp_model_file_data", "wsp_model_meta_serialize", "wsp_model_from_meta",
    "wsp_engine_create", "wsp_engine_create_from_image", "wsp_engine_destroy", "wsp_engine_weight_bytes",
    "wsp_context_create", "wsp_context_destroy", "wsp_synchronize",
    "wsp_context_device_bytes", "wsp_pcm_to_mel", "wsp_pcm_to_mel_window", "wsp_set_mel", "wsp_mel_len", "wsp_get_mel", "wsp_encode", "wsp_set_audio_ctx", "wsp_set_speed_up", "wsp_decode", "wsp_get_logits", "wsp_get_probs",
    "wsp_detect_language", "wsp_run_chunks", "wsp_run_chunks_resident", "wsp_run_chunks_until_eot", "wsp_get_chunk_languages", "wsp_run_chunks_window", "wsp_run_spans_window", "wsp_window_segments", "wsp_set_token_timestamps", "wsp_window_token_times", "wsp_upload_pcm", "wsp_upload_pcm_stereo", "wsp_chunk_speakers", "wsp_timer_start", "wsp_timer_stop", "wsp_profile_decode", "wsp_get_tensor", "wsp_debug_set_encoder_layers", "wsp_debug_set_decoder_stop", "wsp_debug_set_graph", "wsp_debug_set_step_mode", "wsp_debug_enable_step_timing", "wsp_debug_step_timing", "wsp_set_reference_threads",
    "wsp_host_alloc", "wsp_host_free", "wsp_timings",
    "wsp_replicas_create", "wsp_replicas_count", "wsp_replicas_run_chunks", "wsp_replicas_debug_fail_next", "wsp_replicas_destroy",
    "wsp_test_gemm", "wsp_test_attention", "wsp_test_skinny", "wsp_test_layernorm", "wsp_test_sample", "wsp_test_softmax_rows", "wsp_test_window_rule", "wsp_test_token_times", "wsp_test_signal_energy",
    "wsp_test_speakers",
]

_lib = None


class WspError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("wsp_status %d: %s" % (status, msg))
        self.status = status


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError("whisper_b200: %s is missing — build it with __graft_entry__.build() (no CPU fallback exists)" % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i32, u32, u64, sz = C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, C.c_size_t
    fp, ip, u16p = C.POINTER(C.c_float), C.POINTER(C.c_int32), C.POINTER(C.c_uint16)

    def sig(name, res, args):
        f = getattr(L, name)
        f.restype = res
        f.argtypes = args

    sig("wsp_version", C.c_char_p, [])
    sig("wsp_last_error", C.c_char_p, [])
    sig("wsp_device_count", i32, [])
    sig("wsp_device_name", i32, [i32, C.c_char_p, sz])
    sig("wsp_launch_count", u64, [])
    sig("wsp_model_open", i32, [C.c_char_p, C.POINTER(vp)])
    sig("wsp_model_close", None, [vp])
    sig("wsp_model_hparams", i32, [vp, ip])
    sig("wsp_model_special_tokens", i32, [vp, ip])
    sig("wsp_model_token_text", C.c_char_p, [vp, i32])
    sig("wsp_model_is_multilingual", i32, [vp])
    sig("wsp_model_file_data", vp, [vp, C.POINTER(u64)])
    sig("wsp_model_meta_serialize", i32, [vp, vp, u64, C.POINTER(u64)])
    sig("wsp_model_from_meta", i32, [vp, u64, C.POINTER(vp)])
    sig("wsp_engine_create", i32, [vp, i32, C.POINTER(vp)])
    sig("wsp_engine_create_from_image", i32, [vp, i32, vp, u64, C.POINTER(vp)])
    sig("wsp_engine_destroy", None, [vp])
    sig("wsp_engine_weight_bytes", u64, [vp])
    sig("wsp_context_create", i32, [vp, i32, C.POINTER(vp)])
    sig("wsp_context_destroy", None, [vp])
    sig("wsp_synchronize", i32, [vp])
    sig("wsp_context_device_bytes", u64, [vp])
    sig("wsp_pcm_to_mel", i32, [vp, i32, fp, i32])
    sig("wsp_pcm_to_mel_window", i32, [vp, i32, fp, i32, i32, fp, fp])
    sig("wsp_set_mel", i32, [vp, i32, fp, i32])
    sig("wsp_mel_len", i32, [vp, i32])
    sig("wsp_get_mel", i32, [vp, i32, fp, sz])
    sig("wsp_encode", i32, [vp, ip, i32])
    sig("wsp_set_audio_ctx", i32, [vp, i32])
    sig("wsp_set_speed_up", i32, [vp, i32])
    sig("wsp_decode", i32, [vp, ip, i32, i32, i32, u32, C.POINTER(TokenData)])
    sig("wsp_get_logits", i32, [vp, fp, sz])
    sig("wsp_get_probs", i32, [vp, fp, sz])
    sig("wsp_run_chunks", i32, [vp, C.POINTER(fp), ip, i32, ip, i32, i32, ip, fp])
    sig("wsp_run_chunks_resident", i32, [vp, i32, ip, i32, i32, ip, fp])
    sig("wsp_run_chunks_until_eot", i32, [vp, C.POINTER(fp), ip, i32, ip, i32, i32, ip, ip, fp])
    sig("wsp_get_chunk_languages", i32, [vp, i32, ip, fp, sz])
    sig("wsp_run_chunks_window", i32, [vp, C.POINTER(fp), ip, i32, ip, i32, C.POINTER(WindowParams), C.POINTER(TokenData), i32,
                                       C.POINTER(WindowResult), fp])
    sig("wsp_run_spans_window", i32, [vp, C.POINTER(WindowSpan), i32, ip, i32, C.POINTER(WindowParams), C.POINTER(TokenData), i32,
                                      C.POINTER(WindowResult), fp])
    sig("wsp_window_segments", i32, [vp, C.POINTER(TokenData), C.POINTER(WindowResult), i32, u32, C.POINTER(Segment), i32, ip])
    sig("wsp_test_window_rule", i32, [ip, i32, i32, i32, ip, i32, ip, ip])
    sig("wsp_set_token_timestamps", i32, [vp, i32])
    sig("wsp_window_token_times", i32, [vp, i32, C.POINTER(TokenData), C.POINTER(WindowResult), u32, C.POINTER(TokenTimeParams),
                                        C.POINTER(Segment), i32, ip, C.POINTER(TokenTime)])
    sig("wsp_test_signal_energy", i32, [i32, C.POINTER(fp), ip, i32, C.POINTER(fp), i32, fp])
    sig("wsp_test_token_times", i32, [C.POINTER(TokenData), fp, i32, C.c_int64, C.c_int64, ip, fp, i32, C.c_float, C.c_float,
                                      C.POINTER(C.c_int64), C.POINTER(TokenTime)])
    sig("wsp_upload_pcm", i32, [vp, i32, fp, i32])
    sig("wsp_upload_pcm_stereo", i32, [vp, i32, fp, i32])
    sig("wsp_chunk_speakers", i32, [vp, i32, ip, C.POINTER(Segment), ip])
    sig("wsp_test_speakers", i32, [fp, i32, C.POINTER(Segment), i32, ip])
    sig("wsp_timer_start", i32, [vp])
    sig("wsp_timer_stop", i32, [vp, fp])
    sig("wsp_profile_decode", i32, [vp, i32, i32, fp, ip])
    sig("wsp_get_tensor", i32, [vp, C.c_char_p, i32, fp, sz, C.POINTER(sz)])
    sig("wsp_debug_set_encoder_layers", i32, [vp, i32])
    sig("wsp_debug_set_decoder_stop", i32, [vp, i32, i32])
    sig("wsp_debug_set_graph", i32, [vp, i32])
    sig("wsp_set_reference_threads", i32, [vp, i32])
    sig("wsp_debug_set_step_mode", i32, [vp, i32])
    sig("wsp_debug_enable_step_timing", i32, [vp, i32])
    sig("wsp_debug_step_timing", i32, [vp, C.POINTER(C.c_uint64), i32])
    sig("wsp_host_alloc", vp, [sz])
    sig("wsp_host_free", None, [vp])
    sig("wsp_timings", i32, [vp, fp, ip, i32])
    sig("wsp_detect_language", i32, [vp, i32, i32, fp, ip])
    sig("wsp_replicas_create", i32, [vp, ip, i32, i32, C.POINTER(vp)])
    sig("wsp_replicas_count", i32, [vp])
    sig("wsp_replicas_run_chunks", i32, [vp, C.POINTER(fp), ip, i32, ip, i32, i32, ip, C.POINTER(ReplicaStats)])
    sig("wsp_replicas_debug_fail_next", i32, [vp, i32])
    sig("wsp_replicas_destroy", None, [vp])
    sig("wsp_test_sample", i32, [i32, i32, i32, fp, ip, i32, i32, fp, C.POINTER(TokenData)])
    sig("wsp_test_softmax_rows", i32, [i32, i32, i32, fp, fp])
    sig("wsp_test_gemm", i32, [i32, i32, i32, i32, u16p, u16p, fp, i32, i32, fp])
    sig("wsp_test_attention", i32, [i32, i32, i32, u16p, u16p, u16p, fp, i32, fp])
    sig("wsp_test_skinny", i32, [i32, i32, i32, i32, u16p, u16p, fp, i32, fp])
    sig("wsp_test_layernorm", i32, [i32, i32, i32, fp, fp, fp, u16p])
    _lib = L
    return L


def check(status):
    if status < 0:
        raise WspError(status, lib().wsp_last_error().decode(errors="replace"))
    return status


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _i(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def _u16(a):
    return a.ctypes.data_as(C.POINTER(C.c_uint16))


class Model:
    """Parsed ggml model file (host)."""

    def __init__(self, path: str = None, _handle=None):
        self.L = lib()
        if _handle is not None:
            self.h = _handle
        else:
            h = C.c_void_p()
            check(self.L.wsp_model_open(path.encode(), C.byref(h)))
            self.h = h
        hp = np.zeros(11, np.int32)
        check(self.L.wsp_model_hparams(self.h, _i(hp)))
        (self.n_vocab, self.n_audio_ctx, self.n_audio_state, self.n_audio_head, self.n_audio_layer,
         self.n_text_ctx, self.n_text_state, self.n_text_head, self.n_text_layer, self.n_mels, self.f16) = [int(x) for x in hp]
        st = np.zeros(8, np.int32)
        check(self.L.wsp_model_special_tokens(self.h, _i(st)))
        self.special = dict(zip(["eot", "sot", "prev", "solm", "not", "beg", "translate", "transcribe"], [int(x) for x in st]))

    @classmethod
    def from_meta(cls, blob: bytes):
        L = lib()
        h = C.c_void_p()
        buf = C.create_string_buffer(blob, len(blob))
        check(L.wsp_model_from_meta(C.cast(buf, C.c_void_p), len(blob), C.byref(h)))
        return cls(_handle=h)

    def meta(self) -> bytes:
        n = C.c_uint64()
        check(self.L.wsp_model_meta_serialize(self.h, None, 0, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        check(self.L.wsp_model_meta_serialize(self.h, C.cast(buf, C.c_void_p), n.value, C.byref(n)))
        return buf.raw[: n.value]

    def file_image(self):
        """(address, size) of the mapped file image."""
        n = C.c_uint64()
        p = self.L.wsp_model_file_data(self.h, C.byref(n))
        return p, n.value

    def window_segments(self, tokens, result: dict, seek: int = 0, flags: int = 0):
        """whisper_full's segments of one window (wsp_window_segments): tokens = list of token dicts (at least result["n_tokens"]),
        result = the window's result dict.  Returns [dict(t0, t1, i0, i1, text)], times in 10 ms units; the text follows the
        reference's rule (special tokens, id >= eot, only with SEGMENT_PRINT_SPECIAL)."""
        n = max(len(tokens), 1)
        td = (TokenData * n)(*[TokenData(t["id"], t["tid"], t["p"], t["pt"], t["ptsum"]) for t in tokens])
        res = WindowResult(result["n_sampled"], result["n_tokens"], result["seek_delta"], result["failed"])
        segs = (Segment * (result["n_tokens"] + 1))()
        n_segs = np.zeros(1, np.int32)
        check(self.L.wsp_window_segments(self.h, td, C.byref(res), seek, flags, segs, len(segs), _i(n_segs)))
        eot = self.special["eot"]
        out = []
        for s in segs[:int(n_segs[0])]:
            ids = [tokens[i]["id"] for i in range(s.i0, s.i1)]
            text = "".join(self.token_text(i) or "" for i in ids if (flags & SEGMENT_PRINT_SPECIAL) or i < eot)
            out.append(dict(t0=int(s.t0), t1=int(s.t1), i0=int(s.i0), i1=int(s.i1), text=text))
        return out

    def token_text(self, i: int):
        t = self.L.wsp_model_token_text(self.h, i)
        return None if t is None else t.decode(errors="replace")

    def token_bytes(self, i: int) -> bytes:
        return self.L.wsp_model_token_text(self.h, i) or b""

    @property
    def multilingual(self):
        return bool(self.L.wsp_model_is_multilingual(self.h))

    def close(self):
        if self.h:
            self.L.wsp_model_close(self.h)
            self.h = None

    def prompt_init(self, language_id: int | str = 0, translate: bool = False):
        """[sot, (lang, task)] as whisper_full builds it (whisper.cpp:2839-2848).  language_id="auto" puts TOKEN_LANGUAGE_AUTO in the
        language slot: run_chunks* then detect each chunk's language (Context.chunk_languages)."""
        p = [self.special["sot"]]
        if self.multilingual:
            p.append(TOKEN_LANGUAGE_AUTO if language_id == "auto" else self.special["sot"] + 1 + language_id)
            p.append(self.special["translate"] if translate else self.special["transcribe"])
        return p


class Engine:
    def __init__(self, model: Model, device: int = 0, dev_image: int = None, image_size: int = 0):
        self.L = lib()
        self.model = model
        h = C.c_void_p()
        if dev_image is None:
            check(self.L.wsp_engine_create(model.h, device, C.byref(h)))
        else:
            check(self.L.wsp_engine_create_from_image(model.h, device, C.c_void_p(dev_image), image_size, C.byref(h)))
        self.h = h

    def weight_bytes(self):
        return int(self.L.wsp_engine_weight_bytes(self.h))

    def close(self):
        if self.h:
            self.L.wsp_engine_destroy(self.h)
            self.h = None


class Context:
    def __init__(self, engine: Engine, max_batch: int = 1):
        self.L = lib()
        self.engine = engine
        self.model = engine.model
        self.max_batch = max_batch
        self.speed_up = False
        h = C.c_void_p()
        check(self.L.wsp_context_create(engine.h, max_batch, C.byref(h)))
        self.h = h

    def close(self):
        if self.h:
            self.L.wsp_context_destroy(self.h)
            self.h = None

    def pcm_to_mel(self, slot: int, pcm: np.ndarray):
        pcm = np.ascontiguousarray(pcm, np.float32)
        check(self.L.wsp_pcm_to_mel(self.h, slot, _f(pcm), pcm.size))

    def pcm_to_mel_window(self, slot: int, pcm: np.ndarray, n_frames: int, forced_max: float | None = None) -> float:
        """Streamed flavour of the log-mel (one window, normalised by its own maximum); returns that maximum."""
        pcm = np.ascontiguousarray(pcm, np.float32)
        fm = None if forced_max is None else C.c_float(forced_max)
        out = C.c_float(0)
        check(self.L.wsp_pcm_to_mel_window(self.h, slot, _f(pcm), pcm.size, n_frames, None if fm is None else C.byref(fm), C.byref(out)))
        return float(out.value)

    def set_mel(self, slot: int, mel: np.ndarray):
        mel = np.ascontiguousarray(mel, np.float32)
        assert mel.shape[0] == 80
        check(self.L.wsp_set_mel(self.h, slot, _f(mel), mel.shape[1]))

    def get_mel(self, slot: int) -> np.ndarray:
        n = self.L.wsp_mel_len(self.h, slot)
        out = np.empty((80, n), np.float32)
        check(self.L.wsp_get_mel(self.h, slot, _f(out), out.size))
        return out

    def encode(self, batch: int = 1, offsets=None):
        off = None if offsets is None else _i(np.ascontiguousarray(offsets, np.int32))
        check(self.L.wsp_encode(self.h, off, batch))

    def set_audio_ctx(self, n: int):
        """sFullParams::audio_ctx: the next encode covers only the first n audio positions (2n mel frames); n <= 0 = the model's
        n_audio_ctx.  Decodes attend over the n of the last encode."""
        check(self.L.wsp_set_audio_ctx(self.h, int(n)))

    def set_speed_up(self, on):
        """whisper_full_params::speed_up: whole-clip log-mels (pcm_to_mel, run_chunks*) through the reference's 2x phase vocoder,
        n_samples // 320 frames, so a 3000-frame window holds 60 s of audio.  Takes 0 or 1 (bools are accepted)."""
        check(self.L.wsp_set_speed_up(self.h, int(on)))
        self.speed_up = bool(on)

    def decode(self, tokens, n_past: int, batch: int = 1, flags: int = 0):
        """tokens: [batch][n_tokens] (or None with DECODE_DEVICE_TOKENS).  Returns list of sampled dicts (or None)."""
        if tokens is None:
            tp, n = None, 1
        else:
            t = np.ascontiguousarray(tokens, np.int32).reshape(batch, -1)
            tp, n = _i(t), t.shape[1]
        out = (TokenData * batch)()
        check(self.L.wsp_decode(self.h, tp, n, n_past, batch, flags, out))
        if flags & (DECODE_ALL_LOGITS | DECODE_NO_SAMPLE):
            return None
        return [dict(id=o.id, tid=o.tid, p=o.p, pt=o.pt, ptsum=o.ptsum) for o in out]

    def logits(self, rows: int) -> np.ndarray:
        out = np.empty((rows, self.model.n_vocab), np.float32)
        check(self.L.wsp_get_logits(self.h, _f(out), out.size))
        return out

    def probs(self, rows: int) -> np.ndarray:
        out = np.empty((rows, self.model.n_vocab), np.float32)
        check(self.L.wsp_get_probs(self.h, _f(out), out.size))
        return out

    def run_chunks(self, pcms, prompt, n_decode: int):
        """pcms: list of float32 arrays (host).  Returns (tokens[batch][n_decode], stage_ms[3])."""
        batch = len(pcms)
        arrs = [np.ascontiguousarray(p, np.float32) for p in pcms]
        ptrs = (C.POINTER(C.c_float) * batch)(*[_f(a) for a in arrs])
        ns = np.array([a.size for a in arrs], np.int32)
        pr = np.ascontiguousarray(prompt, np.int32)
        toks = np.zeros((batch, n_decode), np.int32)
        st = np.zeros(3, np.float32)
        check(self.L.wsp_run_chunks(self.h, ptrs, _i(ns), batch, _i(pr), pr.size, n_decode, _i(toks), _f(st)))
        return toks, st

    def run_chunks_ptrs(self, ptrs, ns, batch, prompt, n_decode: int):
        """Same as run_chunks but with caller-owned (e.g. pinned) host buffers: ptrs = ctypes array of float*."""
        pr = np.ascontiguousarray(prompt, np.int32)
        toks = np.zeros((batch, n_decode), np.int32)
        st = np.zeros(3, np.float32)
        check(self.L.wsp_run_chunks(self.h, ptrs, _i(ns), batch, _i(pr), pr.size, n_decode, _i(toks), _f(st)))
        return toks, st

    def run_chunks_resident(self, batch: int, prompt, n_decode: int):
        pr = np.ascontiguousarray(prompt, np.int32)
        toks = np.zeros((batch, n_decode), np.int32)
        st = np.zeros(3, np.float32)
        check(self.L.wsp_run_chunks_resident(self.h, batch, _i(pr), pr.size, n_decode, _i(toks), _f(st)))
        return toks, st

    def run_chunks_until_eot(self, pcms, prompt, max_decode: int, batch: int | None = None):
        """Each chunk's greedy tokens up to and including its first EOT (at most max_decode).  pcms: list of float32 arrays, or
        None to run `batch` chunks from the slots' resident PCM (upload_pcm).  Returns (list of token arrays, stage_ms[3])."""
        ptrs, ns = None, None
        if pcms is not None:
            batch = len(pcms)
            arrs = [np.ascontiguousarray(p, np.float32) for p in pcms]
            ptrs = (C.POINTER(C.c_float) * batch)(*[_f(a) for a in arrs])
            ns = np.array([a.size for a in arrs], np.int32)
        pr = np.ascontiguousarray(prompt, np.int32)
        toks = np.zeros((batch, max_decode), np.int32)
        n_out = np.zeros(batch, np.int32)
        st = np.zeros(3, np.float32)
        check(self.L.wsp_run_chunks_until_eot(self.h, ptrs, None if ns is None else _i(ns), batch, _i(pr), pr.size, max_decode, _i(toks), _i(n_out), _f(st)))
        return [toks[b, :n_out[b]].copy() for b in range(batch)], st

    def set_token_timestamps(self, on):
        """whisper_full_params::token_timestamps: run_chunks_window and pcm_to_mel compute each chunk's signal energy on the device
        (get_tensor("energy", b)), which run_chunks_window(token_times=...) needs.  Takes 0 or 1 (bools are accepted)."""
        check(self.L.wsp_set_token_timestamps(self.h, int(on)))

    def run_chunks_window(self, pcms, prompt, max_tokens: int = 0, single_segment: bool = False, print_special: bool = False,
                          batch: int | None = None, token_times: dict | None = None, speakers: bool = False):
        """Each chunk decoded as whisper_full's first window (wsp_run_chunks_window).  pcms: list of float32 arrays, or None to run
        `batch` chunks from the slots' resident PCM (upload_pcm).  Returns (list per chunk of dict(tokens=[token dicts], result=dict,
        segments=[dict(t0, t1, i0, i1, text)]), stage_ms[3]); segment times are doubled while speed-up is on.
        token_times=dict(thold_pt=0.01, thold_ptsum=0.01, max_len=0) (token timestamps must be on): the segments are whisper_full's
        with token_timestamps (wsp_window_token_times), wrapped at max_len characters when max_len > 0; the window's result tokens
        then carry t0, t1 and vlen, and every segment holds its tokens as `tokens`.
        speakers=True: pcms may hold (n, 2) stereo arrays; every chunk is uploaded to its slot (upload_pcm_stereo, or upload_pcm for
        a mono one), the batch runs from the resident PCM, and every segment gets "speaker", detectSpeaker's answer for it
        (chunk_speakers; SPEAKER_NO_STEREO for a mono chunk)."""
        if speakers and pcms is not None:
            for b, p in enumerate(pcms):
                p = np.asarray(p)
                if p.ndim == 2:
                    self.upload_pcm_stereo(b, p)
                else:
                    self.upload_pcm(b, p)
            batch, pcms = len(pcms), None
        ptrs, ns = None, None
        if pcms is not None:
            batch = len(pcms)
            arrs = [np.ascontiguousarray(p, np.float32) for p in pcms]
            ptrs = (C.POINTER(C.c_float) * batch)(*[_f(a) for a in arrs])
            ns = np.array([a.size for a in arrs], np.int32)
        pr = np.ascontiguousarray(prompt, np.int32)
        cap = self.model.n_text_ctx // 2 - 4
        toks = (TokenData * (batch * cap))()
        res = (WindowResult * batch)()
        st = np.zeros(3, np.float32)
        prm = WindowParams(int(max_tokens), int(bool(single_segment)))
        check(self.L.wsp_run_chunks_window(self.h, ptrs, None if ns is None else _i(ns), batch, _i(pr), pr.size, C.byref(prm), toks, cap,
                                           res, _f(st)))
        out = self._windows(toks, cap, res, list(range(batch)), [0] * batch, single_segment, print_special, token_times, speakers)
        return out, st

    def run_spans_window(self, spans, prompt, max_tokens: int = 0, single_segment: bool = False, print_special: bool = False,
                         token_times: dict | None = None, speakers: bool = False):
        """Row b decoded as the first window of whisper_full( clip of slot spans[b][0], offset_ms, duration_ms ) (wsp_run_spans_window):
        spans = [(slot, offset_ms, duration_ms)] over the slots' resident PCM (upload_pcm / upload_pcm_stereo).  Returns what
        run_chunks_window returns, one entry per row, with segment times absolute in the clip (doubled while speed-up is on).
        speakers=True: every segment gets "speaker", detectSpeaker's answer for it against its row's slot's stereo."""
        batch = len(spans)
        sp = (WindowSpan * max(batch, 1))(*[WindowSpan(int(s), int(o), int(d)) for s, o, d in spans])
        pr = np.ascontiguousarray(prompt, np.int32)
        cap = self.model.n_text_ctx // 2 - 4
        toks = (TokenData * (max(batch, 1) * cap))()
        res = (WindowResult * max(batch, 1))()
        st = np.zeros(3, np.float32)
        prm = WindowParams(int(max_tokens), int(bool(single_segment)))
        check(self.L.wsp_run_spans_window(self.h, sp, batch, _i(pr), pr.size, C.byref(prm), toks, cap, res, _f(st)))
        out = self._windows(toks, cap, res, [int(s) for s, _o, _d in spans], [int(o) // 10 for _s, o, _d in spans], single_segment,
                            print_special, token_times, speakers)
        return out, st

    def _windows(self, toks, cap, res, slots, seeks, single_segment, print_special, token_times, speakers):
        """the per-row dicts of a window call: row b's window ran at seeks[b] over slots[b]'s clip"""
        flags = ((SEGMENT_SINGLE if single_segment else 0) | (SEGMENT_PRINT_SPECIAL if print_special else 0)
                 | (SEGMENT_SPEED_UP if self.speed_up else 0))
        out = []
        for b, seek in enumerate(seeks):
            r = res[b]
            result = dict(n_sampled=r.n_sampled, n_tokens=r.n_tokens, seek_delta=r.seek_delta, failed=r.failed)
            tk = [dict(id=t.id, tid=t.tid, p=t.p, pt=t.pt, ptsum=t.ptsum) for t in toks[b * cap:b * cap + r.n_sampled]]
            if token_times is None:
                segs = self.model.window_segments(tk, result, seek, flags)
            else:
                segs = self._token_times(b, toks, b * cap, res[b], tk, flags, print_special, token_times)
            out.append(dict(tokens=tk, result=result, segments=segs))
        if speakers:
            # wsp_chunk_speakers reads chunk k's segments against slot k's stereo: the rows' segments grouped by slot
            by_slot = [[] for _ in range(max(slots) + 1)]
            for o, s in zip(out, slots):
                by_slot[s] += o["segments"]
            for segs, sp in zip(by_slot, self.chunk_speakers(by_slot)):
                for seg, k in zip(segs, sp):
                    seg["speaker"] = k
        return out

    def _token_times(self, b, toks, first, res, tk, flags, print_special, params):
        p = dict(thold_pt=0.01, thold_ptsum=0.01, max_len=0)
        p.update(params)
        prm = TokenTimeParams(p["thold_pt"], p["thold_ptsum"], int(p["max_len"]))
        n = res.n_tokens
        times = (TokenTime * max(n, 1))()
        n_segs = np.zeros(1, np.int32)
        td = C.cast(C.byref(toks, first * C.sizeof(TokenData)), C.POINTER(TokenData))
        st = self.L.wsp_window_token_times(self.h, b, td, C.byref(res), flags, C.byref(prm), None, 0, _i(n_segs), times)
        if st != -7:                                     # WSP_E_BOUNDS: *n_segs holds the count
            check(st)
        segs = (Segment * max(int(n_segs[0]), 1))()
        check(self.L.wsp_window_token_times(self.h, b, td, C.byref(res), flags, C.byref(prm), segs, len(segs), _i(n_segs), times))
        for i in range(n):
            tk[i].update(t0=int(times[i].t0), t1=int(times[i].t1), vlen=float(times[i].vlen))
        eot = self.model.special["eot"]
        out = []
        for s in segs[:int(n_segs[0])]:
            ids = [tk[i]["id"] for i in range(s.i0, s.i1)]
            if p["max_len"] > 0:                         # a wrapped segment's text: its non-special tokens' bytes
                text = b"".join(self.model.token_bytes(i) for i in ids if i < eot).decode(errors="replace")
            else:                                        # as window_segments makes it
                text = "".join(self.model.token_text(i) or "" for i in ids if print_special or i < eot)
            out.append(dict(t0=int(s.t0), t1=int(s.t1), i0=int(s.i0), i1=int(s.i1), text=text, tokens=tk[s.i0:s.i1]))
        return out

    def chunk_languages(self, batch: int):
        """The languages the last run_chunks* call detected for chunks [0, batch) (its prompt held TOKEN_LANGUAGE_AUTO): (ids[batch],
        probs[batch][n_langs]), ids as detect_language reports them (0 = en).  None if that call had no sentinel."""
        n_langs = self.model.special["translate"] - self.model.special["sot"] - 1
        ids = np.zeros(batch, np.int32)
        probs = np.zeros((batch, n_langs), np.float32)
        if check(self.L.wsp_get_chunk_languages(self.h, batch, _i(ids), _f(probs), probs.size)) == WSP_S_FALSE:
            return None
        return ids, probs

    def upload_pcm(self, slot: int, pcm: np.ndarray):
        pcm = np.ascontiguousarray(pcm, np.float32)
        check(self.L.wsp_upload_pcm(self.h, slot, _f(pcm), pcm.size))

    def upload_pcm_stereo(self, slot: int, lr: np.ndarray):
        """Interleaved stereo lr[n][2] (left, right) into the slot: kept on the device, and its downmix (l + r) * 0.5 becomes the
        slot's resident mono PCM (get_tensor("pcm") / "pcm_stereo")."""
        lr = np.ascontiguousarray(lr, np.float32)
        if lr.ndim != 2 or lr.shape[1] != 2:
            raise ValueError("stereo PCM must have shape (n, 2)")
        check(self.L.wsp_upload_pcm_stereo(self.h, slot, _f(lr), lr.shape[0]))

    def chunk_speakers(self, segments_per_chunk):
        """detectSpeaker's answer for every segment of chunks [0, len(segments_per_chunk)) against the slots' stereo, in one call of
        wsp_chunk_speakers: segments are dicts (or objects) with t0 / t1 in 10 ms units.  Returns a list of answer lists (SPEAKER_*)."""
        counts = [len(s) for s in segments_per_chunk]
        start = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        flat = [seg for s in segments_per_chunk for seg in s]
        tt = [(seg["t0"], seg["t1"]) if isinstance(seg, dict) else (seg.t0, seg.t1) for seg in flat]
        segs = (Segment * max(len(flat), 1))(*[Segment(int(a), int(b), 0, 0) for a, b in tt])
        out = np.zeros(max(len(flat), 1), np.int32)
        check(self.L.wsp_chunk_speakers(self.h, len(counts), _i(start), segs, _i(out)))
        return [out[start[b]:start[b + 1]].tolist() for b in range(len(counts))]

    def timer_start(self):
        check(self.L.wsp_timer_start(self.h))

    def timer_stop(self) -> float:
        ms = C.c_float(0)
        check(self.L.wsp_timer_stop(self.h, C.byref(ms)))
        return ms.value

    def profile_decode(self, batch: int, n_steps: int):
        """-> (ms_by_kind[4], launches_by_kind[4]) for kinds (skinny GEMM, cross-attn, self-attn, other)."""
        ms = np.zeros(4, np.float32)
        n = np.zeros(4, np.int32)
        check(self.L.wsp_profile_decode(self.h, batch, n_steps, _f(ms), _i(n)))
        return ms, n

    def get_tensor(self, name: str, slot: int = 0) -> np.ndarray:
        n = C.c_size_t()
        check(self.L.wsp_get_tensor(self.h, name.encode(), slot, None, 0, C.byref(n)))
        out = np.empty(n.value, np.float32)
        check(self.L.wsp_get_tensor(self.h, name.encode(), slot, _f(out), out.size, C.byref(n)))
        return out

    def detect_language(self, offset_frames: int = 0, n_langs: int = 99):
        probs = np.zeros(n_langs, np.float32)
        lid = np.zeros(1, np.int32)
        check(self.L.wsp_detect_language(self.h, offset_frames, n_langs, _f(probs), _i(lid)))
        return int(lid[0]), probs

    def set_encoder_layers(self, n: int):
        check(self.L.wsp_debug_set_encoder_layers(self.h, n))

    def set_decoder_stop(self, layer: int, op: int):
        """End every decoder pass after op `op` (0 QKV, 1 self attention, 2 self-out, 3 cross Q, 4 cross attention, 5 cross-out,
        6 fc1, 7 fc2) of layer `layer`; layer -1 = after the embedding, (-1, -1) = no stop.  Stopped passes run kernel by kernel and
        must not sample (DECODE_NO_SAMPLE or DECODE_ALL_LOGITS)."""
        check(self.L.wsp_debug_set_decoder_stop(self.h, int(layer), int(op)))

    def set_reference_threads(self, n: int):
        check(self.L.wsp_set_reference_threads(self.h, n))

    def set_step_mode(self, mode: int):
        """2 = dataflow decoder-step kernel (default), 1 = round 1's barrier kernel, 0 = one kernel per op."""
        check(self.L.wsp_debug_set_step_mode(self.h, int(mode)))

    def step_timing(self, enable=None, cap=4608):
        """enable=True/False switches the %globaltimer marks on/off; enable=None reads the marks of the last step (ns)."""
        if enable is not None:
            check(self.L.wsp_debug_enable_step_timing(self.h, int(bool(enable))))
            return None
        buf = np.zeros(cap, np.uint64)
        check(self.L.wsp_debug_step_timing(self.h, buf.ctypes.data_as(C.POINTER(C.c_uint64)), cap))
        return buf

    def set_graph(self, on: bool):
        check(self.L.wsp_debug_set_graph(self.h, int(on)))

    def timings(self, reset=False):
        ms = np.zeros(4, np.float32)
        calls = np.zeros(4, np.int32)
        check(self.L.wsp_timings(self.h, _f(ms), _i(calls), int(reset)))
        return ms, calls


# ---- kernel-level test hooks ---------------------------------------------------------------------------------------
def test_gemm(A16: np.ndarray, B16: np.ndarray, bn: int = 256, iters: int = 0, device: int = 0):
    """A16 [M][K], B16 [N][K] float16 -> (D [M][N] float32, ms)."""
    A16 = np.ascontiguousarray(A16, np.float16)
    B16 = np.ascontiguousarray(B16, np.float16)
    M, K = A16.shape
    N = B16.shape[0]
    D = np.zeros((M, N), np.float32)
    ms = C.c_float(0)
    check(lib().wsp_test_gemm(device, M, N, K, _u16(A16.view(np.uint16)), _u16(B16.view(np.uint16)), _f(D), bn, iters, C.byref(ms)))
    return D, ms.value


def test_attention(Q, K, V, iters: int = 0, device: int = 0):
    """Q,K,V [BH][T][64] float16 -> (out [BH][T][64] float32, ms)."""
    Q = np.ascontiguousarray(Q, np.float16)
    K = np.ascontiguousarray(K, np.float16)
    V = np.ascontiguousarray(V, np.float16)
    BH, T, _ = Q.shape
    out = np.zeros((BH, T, 64), np.float32)
    ms = C.c_float(0)
    check(lib().wsp_test_attention(device, BH, T, _u16(Q.view(np.uint16)), _u16(K.view(np.uint16)), _u16(V.view(np.uint16)), _f(out), iters, C.byref(ms)))
    return out, ms.value


def test_skinny(W16, X16, iters: int = 0, device: int = 0):
    """W16 [nOut][K], X16 [cols][K] float16 -> (out [cols][nOut] float32, ms)."""
    W16 = np.ascontiguousarray(W16, np.float16)
    X16 = np.ascontiguousarray(X16, np.float16)
    nOut, K = W16.shape
    cols = X16.shape[0]
    out = np.zeros((cols, nOut), np.float32)
    ms = C.c_float(0)
    check(lib().wsp_test_skinny(device, nOut, K, cols, _u16(W16.view(np.uint16)), _u16(X16.view(np.uint16)), _f(out), iters, C.byref(ms)))
    return out, ms.value


def test_window_rule(ids, eot: int, beg: int, max_tokens: int = 0, single_segment: bool = False, n_max: int = 220, seek: int = 0,
                     seek_end: int = 3000):
    """csrc/window_rule.h on the host over a token sequence from step 0 -> (dict(has_ts, seek_delta, result_len, failed, ended),
    tokens consumed)"""
    a = np.ascontiguousarray(ids, np.int32)
    rule = np.array([eot, beg, max_tokens, int(bool(single_segment))], np.int32)
    out = np.zeros(5, np.int32)
    n = np.zeros(1, np.int32)
    check(lib().wsp_test_window_rule(_i(rule), n_max, seek, seek_end, _i(a), a.size, _i(out), _i(n)))
    return dict(zip(["has_ts", "seek_delta", "result_len", "failed", "ended"], [int(x) for x in out])), int(n[0])


def test_token_times(tokens, vlen, t0: int, t1: int, beg: int, eot: int, energy, thold_pt: float = 0.01, thold_ptsum: float = 0.01,
                     state=(0, 0, 0), times=None):
    """csrc/token_times.h on the host for one segment: tokens = dicts (id, tid, p, pt, ptsum), vlen = floats, energy = float32 array,
    state = (t_beg, t_last, tid_last), times = [[t0, t1, vlen]] on entry (default all -1, 0).  -> (times as [[t0, t1, vlen]], state,
    whether there was energy)"""
    n = len(tokens)
    td = (TokenData * max(n, 1))(*[TokenData(t["id"], t["tid"], t.get("p", 0.0), t["pt"], t["ptsum"]) for t in tokens])
    vl = np.ascontiguousarray(vlen if n else [0.0], np.float32)
    tt = (TokenTime * max(n, 1))(*[TokenTime(int(a), int(b_), float(v)) for a, b_, v in (times or [[-1, -1, 0.0]] * n)])
    en = np.ascontiguousarray(energy if len(energy) else [0.0], np.float32)
    st = (C.c_int64 * 3)(*[int(x) for x in state])
    sp = np.array([beg, eot], np.int32)
    rc = check(lib().wsp_test_token_times(td, _f(vl), n, t0, t1, _i(sp), _f(en), len(energy), thold_pt, thold_ptsum, st, tt))
    return [[int(t.t0), int(t.t1), float(t.vlen)] for t in tt[:n]], [int(x) for x in st], rc == WSP_OK


def test_speakers(lr, segments):
    """csrc/speaker.h on the host: detectSpeaker's answer for each (t0, t1) of `segments` over stereo lr[n][2] (None or an empty
    array: no stereo)"""
    a = np.ascontiguousarray(np.zeros((0, 2)) if lr is None else lr, np.float32).reshape(-1, 2)
    segs = (Segment * max(len(segments), 1))(*[Segment(int(t0), int(t1), 0, 0) for t0, t1 in segments])
    out = np.zeros(max(len(segments), 1), np.int32)
    check(lib().wsp_test_speakers(_f(a) if a.size else None, a.shape[0], segs, len(segments), _i(out)))
    return out[:len(segments)].tolist()


def test_signal_energy(pcms, iters: int = 0, device: int = 0):
    """signal_energy_kernel alone over a batch of float32 clips -> (energies, ms of one launch averaged over iters launches)"""
    arrs = [np.ascontiguousarray(p, np.float32) for p in pcms]
    outs = [np.empty_like(a) for a in arrs]
    ins = (C.POINTER(C.c_float) * len(arrs))(*[_f(a) for a in arrs])
    dst = (C.POINTER(C.c_float) * len(arrs))(*[_f(o) for o in outs])
    ns = np.array([a.size for a in arrs], np.int32)
    ms = C.c_float(0)
    check(lib().wsp_test_signal_energy(device, ins, _i(ns), len(arrs), dst, iters, C.byref(ms)))
    return outs, ms.value


def test_layernorm(x, gamma, beta, device: int = 0):
    x = np.ascontiguousarray(x, np.float32)
    rows, d = x.shape
    g = np.ascontiguousarray(gamma, np.float32)
    b = np.ascontiguousarray(beta, np.float32)
    out = np.zeros((rows, d), np.uint16)
    check(lib().wsp_test_layernorm(device, rows, d, _f(x), _f(g), _f(b), _u16(out)))
    return out.view(np.float16).astype(np.float32)


def test_sample(logits: np.ndarray, special4, force_timestamp=False, is_initial=False, device: int = 0):
    """rows of logits -> (probs [rows][n_vocab], list of token dicts) from the GPU sampler alone"""
    lg = np.ascontiguousarray(logits, np.float32)
    rows, nv = lg.shape
    probs = np.empty_like(lg)
    out = (TokenData * rows)()
    sp = np.ascontiguousarray(special4, np.int32)
    check(lib().wsp_test_sample(device, rows, nv, _f(lg), _i(sp), int(force_timestamp), int(is_initial), _f(probs), out))
    return probs, [dict(id=t.id, tid=t.tid, p=t.p, pt=t.pt, ptsum=t.ptsum) for t in out]


def test_softmax_rows(logits: np.ndarray, device: int = 0):
    """rows of logits -> probs [rows][n] from softmaxRows alone (the all-logits vocabulary softmax)"""
    lg = np.ascontiguousarray(logits, np.float32)
    rows, n = lg.shape
    probs = np.empty_like(lg)
    check(lib().wsp_test_softmax_rows(device, rows, n, _f(lg), _f(probs)))
    return probs


class Replicas:
    """wsp_replicas: one engine + context per listed device inside this process, fed by a host work queue (csrc/replicas.cpp)."""

    def __init__(self, model: Model, devices, max_batch: int):
        self.L = lib()
        self.h = C.c_void_p()
        dv = np.ascontiguousarray(devices, np.int32)
        check(self.L.wsp_replicas_create(model.h, _i(dv), dv.size, max_batch, C.byref(self.h)))
        self.n = dv.size

    def run_chunks(self, pcms, prompt, n_decode: int):
        pcms = [np.ascontiguousarray(p, np.float32) for p in pcms]
        ptrs = (C.POINTER(C.c_float) * len(pcms))(*[_f(p) for p in pcms])
        ns = np.array([p.size for p in pcms], np.int32)
        pr = np.ascontiguousarray(prompt, np.int32)
        toks = np.zeros((len(pcms), n_decode), np.int32)
        stats = (ReplicaStats * self.n)()
        check(self.L.wsp_replicas_run_chunks(self.h, ptrs, _i(ns), len(pcms), _i(pr), pr.size, n_decode, _i(toks), stats))
        return toks, [dict(device=s.device, batches=s.batches_done, chunks=s.chunks_done, failed=s.failed, busy_ms=s.busy_ms, load_ms=s.load_ms) for s in stats]

    def fail_next(self, replica: int):
        check(self.L.wsp_replicas_debug_fail_next(self.h, replica))

    def close(self):
        if self.h:
            self.L.wsp_replicas_destroy(self.h)
            self.h = None

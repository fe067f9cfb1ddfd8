"""C-ABI surface: the shared library loads, exports every symbol include/whisper_b200.h declares, parses model files on the
host, and FAILS LOUDLY (no CPU fallback) when asked to compute without an sm_90a device.  No GPU needed."""
import os
import re

import numpy as np
import pytest

from whisper_b200 import capi, synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "whisper_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(wsp_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    L = capi.lib()
    syms = declared_symbols()
    assert len(syms) >= 35
    missing = [s for s in syms if not hasattr(L, s)]
    assert not missing, missing
    # and the Python binding lists the same set
    assert sorted(capi.EXPORTS) == syms


def test_version_and_error_text():
    L = capi.lib()
    assert b"sm_90a" in L.wsp_version()
    assert isinstance(L.wsp_last_error(), bytes)


def test_model_open_errors(tmp_path):
    with pytest.raises(capi.WspError) as e:
        capi.Model(str(tmp_path / "does-not-exist.bin"))
    assert e.value.status == -3  # WSP_E_FILE
    bad = tmp_path / "bad.bin"
    bad.write_bytes(b"\x00" * 4096)
    with pytest.raises(capi.WspError) as e:
        capi.Model(str(bad))
    assert e.value.status == -4  # WSP_E_FORMAT
    # truncated real file: header parses, tensors are cut short
    good = synth.model_path("micro.en")
    data = open(good, "rb").read()
    trunc = tmp_path / "trunc.bin"
    trunc.write_bytes(data[: len(data) // 2])
    with pytest.raises(capi.WspError) as e:
        capi.Model(str(trunc))
    assert e.value.status in (-3, -4)


@pytest.mark.parametrize("name,multilingual", [("micro.en", False), ("micro", True)])
def test_model_parse_matches_reference_conventions(name, multilingual):
    m = capi.Model(synth.model_path(name))
    hp = synth.MODELS[name]
    assert (m.n_vocab, m.n_audio_state, m.n_audio_head, m.n_audio_layer, m.n_text_ctx) == (
        hp.n_vocab, hp.n_audio_state, hp.n_audio_head, hp.n_audio_layer, hp.n_text_ctx)
    assert m.multilingual == multilingual
    sh = 1 if multilingual else 0   # whisper.cpp:575-583
    assert m.special == dict(eot=50256 + sh, sot=50257 + sh, prev=50360 + sh, solm=50361 + sh, **{"not": 50362 + sh}, beg=50363 + sh,
                             translate=50358, transcribe=50359)
    # vocabulary: file words, then the synthesised specials (whisper.cpp:585-607)
    assert m.token_text(5) == " t5"
    assert m.token_text(m.special["beg"]) == "[_BEG_]"
    assert m.token_text(m.special["beg"] + 7) == "[_TT_7]"
    assert m.token_text(m.n_vocab) is None
    assert m.prompt_init() == ([m.special["sot"]] if not multilingual else [m.special["sot"], m.special["sot"] + 1, 50359])
    m.close()


def test_meta_blob_roundtrip():
    m = capi.Model(synth.model_path("micro"))
    blob = m.meta()
    assert 100_000 < len(blob) < 2_000_000
    m2 = capi.Model.from_meta(blob)
    assert m2.special == m.special and m2.n_vocab == m.n_vocab and m2.token_text(123) == m.token_text(123)
    addr, size = m.file_image()
    assert addr and size == os.path.getsize(synth.model_path("micro"))
    addr2, size2 = m2.file_image()
    assert not addr2 and size2 == size   # a meta-only model has no tensor bytes: the engine needs a device image
    with pytest.raises(capi.WspError):
        capi.Model.from_meta(blob[:1000])


def test_no_cpu_fallback_without_gpu():
    """On a box without an H100 every compute entry point must fail with WSP_E_CUDA and say why."""
    L = capi.lib()
    if L.wsp_device_count() > 0:
        pytest.skip("a CUDA device is visible here")
    m = capi.Model(synth.model_path("micro.en"))
    with pytest.raises(capi.WspError) as e:
        capi.Engine(m, 0)
    assert e.value.status == -5 and "cuda" in str(e.value).lower()
    a = np.zeros((128, 64), np.float16)
    with pytest.raises(capi.WspError) as e:
        capi.test_gemm(a, a)
    assert e.value.status == -5


def _first_tensor_header(data: bytes):
    """byte offset of the first tensor record: magic, 11 hparams, filters, vocabulary (whisper.cpp:451-607)"""
    import struct
    pos = 4 + 44
    n_mel, n_fft = struct.unpack_from("<2i", data, pos)
    pos += 8 + n_mel * n_fft * 4
    (n_words,) = struct.unpack_from("<i", data, pos)
    pos += 4
    for _ in range(n_words):
        (ln,) = struct.unpack_from("<I", data, pos)
        pos += 4 + ln
    return pos


def test_corrupt_tensor_headers_are_rejected(tmp_path):
    """ADVICE r1: a negative dimension must not turn into a huge byte count that wraps the cursor; unknown tensor types are refused."""
    import struct
    data = bytearray(open(synth.model_path("micro.en"), "rb").read())
    pos = _first_tensor_header(data)
    n_dims, name_len, ftype = struct.unpack_from("<3i", data, pos)
    assert 1 <= n_dims <= 3 and 0 < name_len < 64 and ftype in (0, 1)
    for patch, what in (((pos + 12, struct.pack("<i", -5)), "negative ne[0]"), ((pos + 12, struct.pack("<i", 0)), "zero ne[0]"),
                        ((pos + 8, struct.pack("<i", 7)), "ftype 7")):
        bad = bytearray(data)
        bad[patch[0]:patch[0] + 4] = patch[1]
        p = tmp_path / "bad.bin"
        p.write_bytes(bytes(bad))
        with pytest.raises(capi.WspError) as e:
            capi.Model(str(p))
        assert e.value.status == -4, what  # WSP_E_FORMAT


def test_inconsistent_meta_blob_is_rejected():
    """A meta blob is not trusted: tensor offsets / sizes must stay inside the image it describes."""
    import struct
    m = capi.Model(synth.model_path("micro.en"))
    blob = bytearray(m.meta())
    size = struct.unpack_from("<Q", blob, len(blob) - 8)[0]      # imageSize is the last field
    assert size == os.path.getsize(synth.model_path("micro.en"))
    shrunk = bytearray(blob)
    shrunk[len(blob) - 8:] = struct.pack("<Q", size // 2)        # now most tensors end past the image
    with pytest.raises(capi.WspError) as e:
        capi.Model.from_meta(bytes(shrunk))
    assert e.value.status == -4
    m.close()

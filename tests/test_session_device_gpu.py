"""GPU tests of Session.extract_tensor (osm_b200_session_extract_device): audio held as a padded CUDA tensor gives, bit for bit,
the rows and offsets the host entry points give for the same samples -- extract_pcm for int16, extract_files on 32-bit float WAV
files for float32 -- for the shipped LLD and summary configurations, on ragged batches whose padding (NaN, random values) is never
read.  The work follows the caller's stream, and no host <-> device copy of the samples or the rows happens."""
import json
import os
import struct

import numpy as np
import pytest
import torch

from opensmile_b200 import Session
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm
from session_device_cases import LLD, SUMMARY, conf_path, ragged_lengths

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.isdir(os.path.dirname(conf_path(LLD["mfcc"]))),
                                 reason="reference configuration files not built (make -C oracle ref)")]
CASES = {**LLD, **SUMMARY}


def utterances(lengths, sr, nch, seed=0):
    """int16 utterances [n, nch] (mixed voiced / noise / silence content)"""
    out = []
    for u, n in enumerate(lengths):
        x = stereo_mixed_pcm(int(n), sr, seed=seed + u) if nch == 2 else mixed_pcm(int(n), sr, seed=seed + u)
        out.append(x.reshape(int(n), nch))
    return out


def padded(utts, nch, pad=17, seed=1):
    """int16 CUDA batch [B, C, L], channel-planar (C dropped for mono), its padding filled with random values"""
    rng = np.random.default_rng(seed)
    x = rng.integers(-32768, 32767, size=(len(utts), nch, max(len(y) for y in utts) + pad), dtype=np.int16)
    for u, y in enumerate(utts):
        x[u, :, :len(y)] = y.T
    return torch.from_numpy(x[:, 0] if nch == 1 else x).contiguous().cuda()


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(np.ascontiguousarray(a).view(np.uint32), np.ascontiguousarray(b).view(np.uint32))


@pytest.mark.parametrize("name", list(CASES))
def test_int16_tensor_rows_are_the_host_path_rows(name):
    conf, opts, sr, nch = CASES[name]
    s = Session(conf_path((conf,)), options=opts, device=0)
    lens = ragged_lengths(s, sr, nch)
    utts = utterances(lens, sr, nch)
    off = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    want, fo_h = s.extract_pcm(np.concatenate([x.reshape(-1) for x in utts]), off, sr, nch)
    rows, fo = s.extract_tensor(padded(utts, nch), lens, sr)
    assert rows.is_cuda and rows.dtype == torch.float32 and rows.device == torch.device("cuda", 0)
    assert list(fo) == list(fo_h) and fo.dtype == np.int64
    assert same_bits(rows.cpu().numpy(), want), name
    s.close()


def _write_float_wav(path, x, sr):
    data = np.ascontiguousarray(x, dtype="<f4").tobytes()
    nch = x.shape[1]
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 36 + len(data)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<IHHIIHH", 16, 3, nch, sr, sr * 4 * nch, 4 * nch, 32))
        f.write(b"data" + struct.pack("<I", len(data)) + data)


def _read_htk(path):
    raw = open(path, "rb").read()
    n, _, size, _ = struct.unpack(">iihh", raw[:12])
    return np.frombuffer(raw[12:], dtype=">f4").astype(np.float32).reshape(n, size // 4)


@pytest.mark.parametrize("name", ["mfcc", "plp_stereo"])
def test_float32_tensor_rows_are_those_of_float_wav_files(name, tmp_path):
    conf, opts, sr, nch = CASES[name]
    s = Session(conf_path((conf,)), options=opts, device=0)
    lens = np.array([int(1.7 * sr), 1, 399, 1103, 3 * sr], np.int64)
    utts = [(x / 32768.0).astype(np.float32) for x in utterances(lens, sr, nch, seed=4)]
    wavs = [str(tmp_path / ("u%d.wav" % u)) for u in range(len(lens))]
    htks = [str(tmp_path / ("u%d.htk" % u)) for u in range(len(lens))]
    for p, x in zip(wavs, utts):
        _write_float_wav(p, x, sr)
    frames = s.extract_files(wavs, htk_paths=htks)
    rng = np.random.default_rng(2)
    x = rng.standard_normal((len(lens), nch, int(lens.max()) + 9)).astype(np.float32)
    x[:, :, ::3] = np.nan
    for u, y in enumerate(utts):
        x[u, :, :len(y)] = y.T
    t = torch.from_numpy(x[:, 0] if nch == 1 else x).contiguous().cuda()
    rows, fo = s.extract_tensor(t, lens, sr)
    rows = rows.cpu().numpy()
    assert list(np.diff(fo)) == list(frames)
    for u, p in enumerate(htks):
        assert same_bits(rows[fo[u]:fo[u + 1]], _read_htk(p)), (name, u)
    s.close()


@pytest.mark.parametrize("name", ["mfcc", "egemaps"])
def test_caller_stream_rerun_and_single_utterances(name):
    conf, opts, sr, nch = CASES[name]
    s = Session(conf_path((conf,)), options=opts, device=0)
    lens = np.array([3 * sr, int(2.5 * sr), 0, 4 * sr + 7], np.int64)
    x = padded(utterances(lens, sr, nch, seed=9), nch)
    base, fo = s.extract_tensor(x, lens, sr)
    base = base.cpu().numpy()
    # a torch op on another stream writes the input, the extraction follows on that stream
    side = torch.cuda.Stream()
    y = torch.empty_like(x)
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(50_000_000)                    # the copy lands well after the call has returned
        y.copy_(x)
        rows, fo2 = s.extract_tensor(y, lens, sr)
    side.synchronize()
    assert list(fo2) == list(fo) and same_bits(rows.cpu().numpy(), base)
    again, _ = s.extract_tensor(x, lens, sr)
    assert same_bits(again.cpu().numpy(), base)
    for u in (0, 3):
        one, fo1 = s.extract_tensor(x[u:u + 1, :int(lens[u])].contiguous(), [int(lens[u])], sr)
        assert same_bits(one.cpu().numpy(), base[fo[u]:fo[u + 1]]), u
    s.close()


@pytest.mark.parametrize("name", ["mfcc", "egemaps"])
def test_no_host_device_copy_of_samples_or_rows(name, tmp_path):
    conf, opts, sr, nch = CASES[name]
    s = Session(conf_path((conf,)), options=opts, device=0)
    lens = np.array([3 * sr - 5 * u for u in range(16)], np.int64)
    x = padded(utterances(lens, sr, nch), nch)
    rows, _ = s.extract_tensor(x, lens, sr)                         # warm-up: plan, buffers and the batch's schedule
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]) as prof:
        rows, _ = s.extract_tensor(x, lens, sr)
        torch.cuda.synchronize()
    trace = str(tmp_path / "trace.json")
    prof.export_chrome_trace(trace)
    copies = [(e["name"], int(e.get("args", {}).get("bytes", 0))) for e in json.load(open(trace))["traceEvents"]
              if e.get("cat") == "gpu_memcpy" and ("HtoD" in e["name"] or "DtoH" in e["name"])]
    kernels = [e["name"] for e in json.load(open(trace))["traceEvents"] if e.get("cat") == "kernel"]
    assert any("pcm_pack_kernel" in k for k in kernels), kernels
    limit = 64 * (len(lens) + 1)                                     # offsets and counts: a few int64 per utterance
    assert all(b <= limit for _, b in copies), (copies, limit)
    assert limit < min(x.numel() * 2, rows.numel() * 4)
    s.close()


def test_extract_tensor_refuses_device_arguments():
    conf, opts, sr, nch = CASES["mfcc"]
    x = torch.zeros((2, 16000), dtype=torch.int16, device="cuda")
    s = Session(conf_path((conf,)), options=opts, device=0)
    with pytest.raises(ValueError, match="on the host"):
        s.extract_tensor(x, torch.tensor([16000, 10], device="cuda"), sr)
    s.close()
    d = Session(conf_path((conf,)), options=opts, device=-1)         # a description-only session runs on no device
    with pytest.raises(ValueError, match="session runs on device -1"):
        d.extract_tensor(x, [16000, 10], sr)
    d.close()

"""Python host-side wrapper over the C ABI (include/osm_b200.h).

`Plan` owns an `osm_b200_plan*`; `components_*()` build the component list the way the shipped
.conf files wire the reference's components (same instance names, levels and field values;
e.g. config/mfcc/MFCC12_0_D_A.conf).  torch is used only as the device-memory / stream
plumbing for the device-resident entry point.
"""
import ctypes as C
from collections import namedtuple

import numpy as np

from . import capi

LldLaunch = namedtuple("LldLaunch", "kernel grid n_chunks")


def _comp(ctype, name, reader, writer, **fields):
    L = capi.lib()
    c = capi.Component()
    st = L.osm_b200_component_defaults(ctype, C.byref(c))
    if st != capi.OK:
        raise ValueError(capi.last_error())
    c.name = name.encode()
    readers = [r for r in (reader.split(";") if reader else []) if r]
    c.n_inputs = len(readers)
    for i, r in enumerate(readers):
        c.reader_dmLevel[i].value = r.encode()
    c.writer_dmLevel = writer.encode()
    if "nameAppend" in fields:
        c.nameAppend = fields.pop("nameAppend").encode()
    if "copyInputName" in fields:
        c.copyInputName = int(fields.pop("copyInputName"))
    if ctype in capi.UNION_FIELD:
        u = getattr(c.u, capi.UNION_FIELD[ctype])
        for k, v in fields.items():
            if not hasattr(u, k):
                raise AttributeError("%s has no field %s" % (type(u).__name__, k))
            if isinstance(v, str):
                v = v.encode()
            setattr(u, k, v)
    return c


def components_mfcc12_0_d_a(sample_rate=16000.0, n_channels=1, pcm_format=0):
    """config/mfcc/MFCC12_0_D_A.conf (+ shared/standard_wave_input.conf.inc) as a component list.
    pcm_format: osm_b200_pcm_format of the buffers handed to run_* (0 int16, 1 float32, 2 int8, 3 packed 24 bit, 4 24 in 32, 5 int32)"""
    T = capi
    return [
        _comp(T.C_WAVESOURCE, "waveIn", "", "wave", sampleRate=float(sample_rate),
              nChannels=n_channels, monoMixdown=1, format=pcm_format),
        _comp(T.C_FRAMER, "frame", "wave", "frames", frameSize=0.025, frameStep=0.010),
        _comp(T.C_VECTORPREEMPHASIS, "pe", "frames", "framespe", k=0.97, de=0),
        _comp(T.C_WINDOWER, "win", "framespe", "winframes", winFunc=T.WIN_BY_NAME["ham"], gain=1.0, offset=0.0),
        _comp(T.C_TRANSFORMFFT, "fft", "winframes", "fft", inverse=0, zeroPadSymmetric=0),
        _comp(T.C_FFTMAGPHASE, "fftmag", "fft", "fftmag", magnitude=1, phase=0),
        _comp(T.C_MELSPEC, "melspec", "fftmag", "melspec", htkcompatible=1, nBands=26, usePower=1,
              lofreq=0.0, hifreq=8000.0),
        _comp(T.C_MFCC, "mfcc", "melspec", "ft0", firstMfcc=0, lastMfcc=12, cepLifter=22.0, htkcompatible=1),
        _comp(T.C_DELTAREGRESSION, "delta", "ft0", "ft0de", deltawin=2),
        _comp(T.C_DELTAREGRESSION, "accel", "ft0de", "ft0dede", deltawin=2),
        _comp(T.C_VECTORCONCAT, "audspec_lldconcat", "ft0;ft0de;ft0dede", "lld"),
    ]


def components_plp_0_d_a(sample_rate=16000.0, n_channels=1):
    """config/plp/PLP_0_D_A.conf (+ shared/standard_wave_input.conf.inc) as a component list."""
    T = capi
    return [
        _comp(T.C_WAVESOURCE, "waveIn", "", "wave", sampleRate=float(sample_rate),
              nChannels=n_channels, monoMixdown=1),
        _comp(T.C_FRAMER, "frame", "wave", "frames", frameSize=0.025, frameStep=0.010),
        _comp(T.C_VECTORPREEMPHASIS, "pe", "frames", "framespe", k=0.97, de=0),
        _comp(T.C_WINDOWER, "win", "framespe", "winframes", winFunc=T.WIN_BY_NAME["ham"], gain=1.0, offset=0.0),
        _comp(T.C_TRANSFORMFFT, "fft", "winframes", "fft", zeroPadSymmetric=0),
        _comp(T.C_FFTMAGPHASE, "fftmag", "fft", "fftmag"),
        _comp(T.C_MELSPEC, "melspec", "fftmag", "melspec", htkcompatible=1, nBands=26, usePower=1,
              lofreq=0.0, hifreq=8000.0),
        _comp(T.C_PLP, "plp", "melspec", "plp", firstCC=0, lpOrder=5, cepLifter=22.0, compression=0.33,
              htkcompatible=1, doIDFT=1, doLpToCeps=1, doLP=1, doInvLog=0, doAud=1, doLog=0),
        _comp(T.C_DELTAREGRESSION, "delta", "plp", "plpde", deltawin=2),
        _comp(T.C_DELTAREGRESSION, "accel", "plpde", "plpdede", deltawin=2),
        _comp(T.C_VECTORCONCAT, "audspec_lldconcat", "plp;plpde;plpdede", "lld"),
    ]


def comp(type_name, name, reader, writer, **fields):
    """One `[name:cType]` section -> osm_b200_component (type by the reference's component name).
    List-valued cSpectral options: bands=[(lo,hi),...], slopes=[...], rollOff=[...]."""
    ctype = capi.TYPE_BY_NAME[type_name]
    bands = fields.pop("bands", None)
    slopes = fields.pop("slopes", None)
    rolloff = fields.pop("rollOff", None)
    freq_range = fields.pop("freqRange", None)
    c = _comp(ctype, name, reader, writer, **fields)
    if ctype == capi.C_SPECTRAL:
        sp = c.u.spectral
        if bands is not None:
            sp.nBands = len(bands)
            for i, (a, b) in enumerate(bands):
                sp.bandLo[i], sp.bandHi[i] = a, b
        if slopes is not None:
            sp.nSlopes = len(slopes)
            for i, (a, b) in enumerate(slopes):
                sp.slopeLo[i], sp.slopeHi[i] = a, b
        if rolloff is not None:
            sp.nRollOff = len(rolloff)
            for i, r in enumerate(rolloff):
                sp.rollOff[i] = r
        if freq_range is not None:
            sp.freqRangeLo, sp.freqRangeHi = freq_range
    return c


def components_frontend(sample_rate, frame_size, frame_step=0.010, win="ham", sigma=0.4, preemph=None,
                        n_channels=1, prefix="", with_fft=True, zero_pad_symmetric=1):
    """wave -> framer [-> pre-emphasis] -> windower [-> FFT -> magnitude] with level names
    <prefix>frame / <prefix>pe / <prefix>win / <prefix>fft / <prefix>mag."""
    T = capi
    cs = [_comp(T.C_WAVESOURCE, "waveIn", "", "wave", sampleRate=float(sample_rate), nChannels=n_channels, monoMixdown=1),
          _comp(T.C_FRAMER, prefix + "frame", "wave", prefix + "frame", frameSize=frame_size, frameStep=frame_step)]
    last = prefix + "frame"
    if preemph is not None:
        cs.append(_comp(T.C_VECTORPREEMPHASIS, prefix + "pe", last, prefix + "pe", k=preemph))
        last = prefix + "pe"
    cs.append(_comp(T.C_WINDOWER, prefix + "win", last, prefix + "win", winFunc=T.WIN_BY_NAME[win], sigma=sigma))
    if with_fft:
        cs.append(_comp(T.C_TRANSFORMFFT, prefix + "fft", prefix + "win", prefix + "fft", zeroPadSymmetric=zero_pad_symmetric))
        cs.append(_comp(T.C_FFTMAGPHASE, prefix + "mag", prefix + "fft", prefix + "mag"))
    return cs


class Plan:
    """A compiled LLD plan bound to one CUDA device."""

    def __init__(self, components, output_level="lld", device=0):
        self._L = capi.lib()
        arr = (capi.Component * len(components))(*components)
        h = C.c_void_p()
        st = self._L.osm_b200_plan_create(arr, len(components), output_level.encode(), device, C.byref(h))
        if st != capi.OK:
            raise RuntimeError("osm_b200_plan_create failed (%d): %s" % (st, capi.last_error()))
        self._h = h
        self.device = device
        self.num_elements = self._L.osm_b200_plan_num_elements(h)
        self.sample_frame_bytes = self._L.osm_b200_plan_sample_frame_bytes(h)
        self.frame_size = self._L.osm_b200_plan_frame_size_samples(h)
        self.frame_step = self._L.osm_b200_plan_frame_step_samples(h)
        self.fft_size = self._L.osm_b200_plan_fft_size(h)
        self.frame_period = self._L.osm_b200_plan_frame_period(h)

    def close(self):
        if getattr(self, "_h", None):
            self._L.osm_b200_plan_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def element_names(self):
        return [self._L.osm_b200_plan_element_name(self._h, i).decode() for i in range(self.num_elements)]

    def num_frames(self, n_sample_frames):
        return int(self._L.osm_b200_plan_num_frames(self._h, int(n_sample_frames)))

    def num_time_frames(self, n_sample_frames):
        """distinct time stamps of those rows (see osm_b200_plan_num_time_frames)"""
        return int(self._L.osm_b200_plan_num_time_frames(self._h, int(n_sample_frames)))

    def frame_offsets(self, utt_offsets):
        utt = np.ascontiguousarray(utt_offsets, dtype=np.int64)
        fo = np.zeros(utt.size, np.int64)
        st = self._L.osm_b200_plan_frame_offsets(self._h, utt.ctypes.data_as(C.POINTER(C.c_int64)), utt.size - 1,
                                                 fo.ctypes.data_as(C.POINTER(C.c_int64)))
        if st != capi.OK:
            raise RuntimeError(capi.last_error())
        return fo

    # ---- host buffers (H2D + kernels + D2H inside the call) ----
    def run_host(self, pcm, utt_offsets, out=None, frame_offsets=None):
        """pcm: int16 numpy (or any object exposing a writable/readable buffer address via
        .ctypes / data_ptr()), utt_offsets: int64[n_utt+1] in sample frames."""
        utt = np.ascontiguousarray(utt_offsets, dtype=np.int64)
        n_utt = utt.size - 1
        fo = self.frame_offsets(utt) if frame_offsets is None else np.ascontiguousarray(frame_offsets, np.int64)
        rows = int(fo[-1])
        if out is None:
            out = np.empty((rows, self.num_elements), np.float32)
        st = self._L.osm_b200_plan_run_host(self._h, _addr(pcm), utt.ctypes.data_as(C.POINTER(C.c_int64)), n_utt,
                                            fo.ctypes.data_as(C.POINTER(C.c_int64)), _addr(out))
        if st != capi.OK:
            raise RuntimeError("osm_b200_plan_run_host failed (%d): %s" % (st, capi.last_error()))
        return out

    # ---- device resident (torch tensors) ----
    def run_device(self, d_pcm, utt_offsets, d_out=None, frame_offsets=None, stream=None):
        import torch
        utt = np.ascontiguousarray(utt_offsets, dtype=np.int64)
        n_utt = utt.size - 1
        fo = self.frame_offsets(utt) if frame_offsets is None else np.ascontiguousarray(frame_offsets, np.int64)
        rows = int(fo[-1])
        if d_out is None:
            d_out = torch.empty((rows, self.num_elements), dtype=torch.float32, device=d_pcm.device)
        s = torch.cuda.current_stream(d_pcm.device).cuda_stream if stream is None else stream
        st = self._L.osm_b200_plan_run_device(self._h, C.c_void_p(d_pcm.data_ptr()),
                                              utt.ctypes.data_as(C.POINTER(C.c_int64)), n_utt,
                                              fo.ctypes.data_as(C.POINTER(C.c_int64)),
                                              C.c_void_p(d_out.data_ptr()), C.c_void_p(s))
        if st != capi.OK:
            raise RuntimeError("osm_b200_plan_run_device failed (%d): %s" % (st, capi.last_error()))
        return d_out

    def last_launch_count(self):
        return int(self._L.osm_b200_plan_last_launch_count(self._h))

    def take_device_flags(self):
        """condition flags of the runs since the last call (bit 0: a cPitchJitter row was zeroed); synchronises the device"""
        self._L.osm_b200_plan_take_device_flags.argtypes = [C.c_void_p]
        return int(self._L.osm_b200_plan_take_device_flags(self._h))

    def last_kernel_ms(self):
        return float(self._L.osm_b200_plan_last_kernel_ms(self._h))

    def last_kernel_times(self):
        """(fused per-frame kernel ms, temporal kernel ms) of the last run, CUDA events."""
        a, b = C.c_float(0), C.c_float(0)
        st = self._L.osm_b200_plan_last_kernel_times(self._h, C.byref(a), C.byref(b))
        if st != capi.OK:
            raise RuntimeError(capi.last_error())
        return a.value, b.value

    def last_lld_launch(self):
        """(kernel instance name or None, grid, chunks) of the last per-frame kernel launch of the last run"""
        nm, grid, n_chunks = C.c_char_p(), C.c_int32(0), C.c_int64(0)
        if self._L.osm_b200_plan_last_lld_launch(self._h, C.byref(nm), C.byref(grid), C.byref(n_chunks)) != capi.OK:
            raise RuntimeError(capi.last_error())
        return LldLaunch(nm.value.decode() if nm.value else None, grid.value, n_chunks.value)

    def set_profiling(self, on):
        """per-kernel CUDA-event timing of run_device (serialises the step on one stream)"""
        self._L.osm_b200_plan_set_profiling(self._h, 1 if on else 0)

    def kernel_profile(self):
        """[(kernel name, ms)] of the last profiled run_device, in launch order"""
        out = []
        for i in range(self._L.osm_b200_plan_profile_count(self._h)):
            nm, ms = C.c_char_p(), C.c_float(0)
            if self._L.osm_b200_plan_profile_entry(self._h, i, C.byref(nm), C.byref(ms)) != capi.OK:
                raise RuntimeError(capi.last_error())
            out.append((nm.value.decode(), ms.value))
        return out


def _addr(buf):
    if hasattr(buf, "data_ptr"):
        return C.c_void_p(buf.data_ptr())
    return C.c_void_p(buf.ctypes.data)


def pack_utterances(utts, n_chan=1):
    """Concatenate int16 utterances (mono, or channel-interleaved) back to back.
    Returns (pcm int16[...], utt_offsets int64[n+1] in sample frames)."""
    lens = [len(u) // n_chan for u in utts]
    off = np.zeros(len(utts) + 1, np.int64)
    off[1:] = np.cumsum(lens)
    pcm = np.concatenate([np.asarray(u, np.int16) for u in utts]) if utts else np.zeros(0, np.int16)
    return np.ascontiguousarray(pcm), off

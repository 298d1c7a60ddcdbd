"""Session: extract with one of the reference's own .conf files (include/osm_b200_host.h).

Mirrors, for the LLD path, what `SMILExtract -C conf -I wav -O htk -csvoutput csv` and the
SMILEapi external source / sink pair do (progsrc/smilextract/SMILExtract.cpp:42-174,
progsrc/include/smileapi/SMILEapi.h); config parsing, WAV / HTK / CSV I/O are host C++ inside
libosm_b200.so, the numerics are the CUDA plan.  No CPU fallback.
"""
import ctypes as C

import numpy as np

from . import capi


class SessionError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__(msg)
        self.status = status


def _strs(items):
    arr = (C.c_char_p * max(len(items), 1))()
    for i, x in enumerate(items):
        arr[i] = None if x is None else str(x).encode()
    return arr


class Session:
    def __init__(self, conf_path, options=None, output_level=None, device=0):
        self._L = capi.lib()
        self._h = C.c_void_p()
        self._device = device
        options = dict(options or {})
        st = self._L.osm_b200_session_open(
            str(conf_path).encode(), len(options), _strs(list(options.keys())), _strs(list(options.values())),
            output_level.encode() if output_level else None, device, C.byref(self._h))
        if st != capi.OK:
            self._h = C.c_void_p()
            raise SessionError(st, self._L.osm_b200_host_last_error().decode())

    def close(self):
        if self._h:
            self._L.osm_b200_session_close(self._h)
            self._h = C.c_void_p()

    __del__ = close

    def _check(self, st):
        if st != capi.OK:
            raise SessionError(st, self._L.osm_b200_host_last_error().decode())

    def element_names(self, sample_rate=16000.0, n_channels=1):
        n = self._L.osm_b200_session_num_elements(self._h, float(sample_rate), n_channels)
        if n <= 0:
            raise SessionError(capi.ERR_INVALID, self._L.osm_b200_host_last_error().decode())
        return [self._L.osm_b200_session_element_name(self._h, i).decode() for i in range(n)]

    def lld_element_names(self, sample_rate=16000.0, n_channels=1):
        """names of the LLD part of a session whose sinks read a summary and an LLD level ([] without one)"""
        n = self._L.osm_b200_session_lld_num_elements(self._h, float(sample_rate), n_channels)
        return [self._L.osm_b200_session_lld_element_name(self._h, i).decode() for i in range(n)]

    def components(self, sample_rate=16000.0, n_channels=1):
        """the osm_b200_component list the config resolved to, and the output level"""
        p = C.POINTER(capi.Component)()
        lvl = C.c_char_p()
        n = self._L.osm_b200_session_components(self._h, float(sample_rate), n_channels, C.byref(p), C.byref(lvl))
        arr = (capi.Component * n)()
        for i in range(n):
            C.memmove(C.byref(arr[i]), C.byref(p[i]), C.sizeof(capi.Component))
        return arr, lvl.value.decode()

    def frame_offsets(self, utt_offsets, sample_rate, n_channels=1):
        off = np.ascontiguousarray(utt_offsets, dtype=np.int64)
        fo = np.zeros(len(off), dtype=np.int64)
        i64p = C.POINTER(C.c_int64)
        self._check(self._L.osm_b200_session_extract_pcm(
            self._h, None, off.ctypes.data_as(i64p), len(off) - 1, float(sample_rate), n_channels,
            fo.ctypes.data_as(i64p), None, 0))
        return fo

    def extract_pcm(self, pcm, utt_offsets, sample_rate, n_channels=1):
        """packed int16 PCM (layout of Plan.run_host) -> (rows [sum frames, n_elements], frame_offsets)"""
        pcm = np.ascontiguousarray(pcm, dtype=np.int16)
        off = np.ascontiguousarray(utt_offsets, dtype=np.int64)
        fo = self.frame_offsets(off, sample_rate, n_channels)
        n_el = self._L.osm_b200_session_num_elements(self._h, float(sample_rate), n_channels)
        out = np.empty((int(fo[-1]), n_el), dtype=np.float32)
        i64p = C.POINTER(C.c_int64)
        self._check(self._L.osm_b200_session_extract_pcm(
            self._h, pcm.ctypes.data, off.ctypes.data_as(i64p), len(off) - 1, float(sample_rate), n_channels,
            fo.ctypes.data_as(i64p), out.ctypes.data, out.shape[0]))
        return out, fo

    def extract_tensor(self, pcm, lengths, sample_rate, with_lld=False):
        """Audio already on the GPU -> (rows, frame_offsets), the pair extract_pcm returns, without a host round trip.

        pcm: a contiguous CUDA tensor on the session's device, int16 or float32, shaped [B, L] (mono) or [B, C, L]
        (channel-planar, as torch holds it); utterance b is its first lengths[b] samples, the padding is never read.
        int16 samples are those of a 16-bit WAV file.  float32 samples are taken as a 32-bit float WAV file holds them,
        e.g. torchaudio's values in [-1, 1]: they are not divided by a full scale (the reference's
        smilePcm_convertFloatSamples).  Channels are mixed down as for a WAV file.
        lengths: B sample-frame counts, a host sequence or a CPU tensor.
        The work is enqueued on torch.cuda.current_stream(pcm.device).  rows: a CUDA float32 tensor
        [frame_offsets[-1], num_elements] on pcm's device; frame_offsets: a numpy int64 array of B + 1 entries.
        with_lld=True, on a session whose sinks read a summary and an LLD level: (rows, frame_offsets, lld_rows, lld_frame_offsets),
        the summary and the LLD sinks' rows of one plan run, as the two single-level sessions give them."""
        import torch
        if not isinstance(pcm, torch.Tensor):
            raise TypeError("pcm must be a torch tensor")
        fmt = {torch.int16: 0, torch.float32: 1}.get(pcm.dtype)       # OSM_B200_PCM_S16 / OSM_B200_PCM_F32
        if fmt is None:
            raise TypeError("pcm must be int16 or float32, not %s" % pcm.dtype)
        if pcm.dim() not in (2, 3):
            raise ValueError("pcm must be shaped [B, L] or [B, C, L], not %s" % (tuple(pcm.shape),))
        if not pcm.is_contiguous():
            raise ValueError("pcm must be contiguous (call .contiguous() on it: it is not copied here)")
        n_utt, n_chan, stride = pcm.shape[0], (pcm.shape[1] if pcm.dim() == 3 else 1), pcm.shape[-1]
        if isinstance(lengths, torch.Tensor):
            if lengths.device.type != "cpu":
                raise ValueError("lengths must be on the host (a sequence or a CPU tensor), not on %s" % lengths.device)
            lengths = lengths.numpy()
        lens = np.ascontiguousarray(lengths, dtype=np.int64)
        if lens.shape != (n_utt,):
            raise ValueError("lengths must hold %d entries (one per utterance), got shape %s" % (n_utt, lens.shape))
        if n_utt and (lens.min() < 0 or lens.max() > stride):
            raise ValueError("lengths must lie in 0 .. %d (the tensor's last dimension)" % stride)
        if pcm.device.type != "cuda":
            raise ValueError("pcm must be a CUDA tensor, not on %s" % pcm.device)
        if pcm.device.index != self._device:
            raise ValueError("pcm is on %s, the session runs on device %d" % (pcm.device, self._device))
        i64p = C.POINTER(C.c_int64)
        stream = C.c_void_p(torch.cuda.current_stream(pcm.device).cuda_stream)
        fo = np.zeros(n_utt + 1, dtype=np.int64)
        lfo = np.zeros(n_utt + 1, dtype=np.int64)

        def call(d_out, max_rows, d_lld=None, max_lld=0):
            args = (self._h, C.c_void_p(pcm.data_ptr()), fmt, stride, lens.ctypes.data_as(i64p), n_utt, float(sample_rate), n_chan,
                    fo.ctypes.data_as(i64p), d_out, max_rows)
            if with_lld:
                self._check(self._L.osm_b200_session_extract_device_lld(*args, lfo.ctypes.data_as(i64p), d_lld, max_lld, stream))
            else:
                self._check(self._L.osm_b200_session_extract_device(*args, stream))
        call(None, 0)
        n_el = self._L.osm_b200_session_num_elements(self._h, float(sample_rate), n_chan)
        if n_el <= 0:
            raise SessionError(capi.ERR_INVALID, self._L.osm_b200_host_last_error().decode())
        rows = torch.empty((int(fo[-1]), n_el), dtype=torch.float32, device=pcm.device)
        if not with_lld:
            if rows.numel():
                call(C.c_void_p(rows.data_ptr()), rows.shape[0])
            return rows, fo
        n_lld = self._L.osm_b200_session_lld_num_elements(self._h, float(sample_rate), n_chan)
        lld = torch.empty((int(lfo[-1]), n_lld), dtype=torch.float32, device=pcm.device)
        if rows.numel() or lld.numel():
            call(C.c_void_p(rows.data_ptr() if rows.numel() else None), rows.shape[0],
                 C.c_void_p(lld.data_ptr() if lld.numel() else None), lld.shape[0])
        return rows, fo, lld, lfo

    def sink_options(self):
        """formatting options of the configuration's active sinks, as text (osm_b200_session_sink_options)"""
        self._L.osm_b200_session_sink_options.restype = C.c_char_p
        self._L.osm_b200_session_sink_options.argtypes = [C.c_void_p]
        return self._L.osm_b200_session_sink_options(self._h).decode()

    def write_files(self, rows, frame_offsets, sample_rate, n_channels=1, n_samples=None, htk_paths=None, csv_paths=None, arff_paths=None):
        """the sinks for rows already in host memory (osm_b200_session_write_files): file i gets rows
        [frame_offsets[i], frame_offsets[i+1]); files are formatted on host threads in parallel"""
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        fo = np.ascontiguousarray(frame_offsets, dtype=np.int64)
        ns = None if n_samples is None else np.ascontiguousarray(n_samples, dtype=np.int64)
        i64p = C.POINTER(C.c_int64)
        self._check(self._L.osm_b200_session_write_files(
            self._h, float(sample_rate), n_channels, len(fo) - 1, fo.ctypes.data_as(i64p),
            ns.ctypes.data_as(i64p) if ns is not None else None, rows.ctypes.data,
            _strs(htk_paths) if htk_paths else None, _strs(csv_paths) if csv_paths else None, _strs(arff_paths) if arff_paths else None))

    def extract_files(self, wav_paths, htk_paths=None, csv_paths=None, arff_paths=None,
                      lld_htk_paths=None, lld_csv_paths=None, lld_arff_paths=None):
        """lld_*_paths: the LLD sinks' files of a session whose sinks read a summary and an LLD level, from the same plan run"""
        n = len(wav_paths)
        frames = np.zeros(n, dtype=np.int64)
        paths = [_strs(p) if p else None for p in (htk_paths, csv_paths, arff_paths)]
        if lld_htk_paths or lld_csv_paths or lld_arff_paths:
            lld = [_strs(p) if p else None for p in (lld_htk_paths, lld_csv_paths, lld_arff_paths)]
            self._check(self._L.osm_b200_session_extract_files_lld(
                self._h, n, _strs(wav_paths), *paths, *lld, frames.ctypes.data_as(C.POINTER(C.c_int64))))
        else:
            self._check(self._L.osm_b200_session_extract_files_arff(
                self._h, n, _strs(wav_paths), *paths, frames.ctypes.data_as(C.POINTER(C.c_int64))))
        return frames


def write_htk(path, rows, period, parm_kind=9):
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    if capi.lib().osm_b200_write_htk(str(path).encode(), rows.ctypes.data, rows.shape[0], rows.shape[1], float(period), parm_kind):
        raise IOError(capi.lib().osm_b200_host_last_error().decode())


def write_csv(path, rows, names, period, instance_name=None, frame_index=True, frame_time=True, n_time_frames=0):
    """cCsvSink's file format.  n_time_frames (Plan.num_time_frames) > 0: rows past that index repeat the last time stamp,
    as the rows a window processor appends at the end of input do in the reference"""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    L = capi.lib()
    L.osm_b200_write_csv_timed.argtypes = [C.c_char_p, C.c_void_p, C.c_int64, C.c_int32, C.POINTER(C.c_char_p), C.c_double,
                                           C.c_char_p, C.c_int32, C.c_int32, C.c_int64]
    if L.osm_b200_write_csv_timed(str(path).encode(), rows.ctypes.data, rows.shape[0], rows.shape[1], _strs(names),
                                  float(period), instance_name.encode() if instance_name is not None else None,
                                  int(frame_index), int(frame_time), int(n_time_frames)):
        raise IOError(L.osm_b200_host_last_error().decode())


def write_arff(path, rows, names, period, relation="smile", instance_name=None, frame_index=True, frame_time=True,
               classes=(("class", "numeric", "?"),), append=False, n_time_frames=0):
    """cArffSink's file format; classes = (name, type, value for every row) per class attribute"""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    L = capi.lib()
    cpp = C.POINTER(C.c_char_p)
    L.osm_b200_write_arff.argtypes = [C.c_char_p, C.c_void_p, C.c_int64, C.c_int32, cpp, C.c_double, C.c_char_p, C.c_char_p,
                                      C.c_int32, C.c_int32, C.c_int32, cpp, cpp, cpp, C.c_int32, C.c_int64]
    if L.osm_b200_write_arff(str(path).encode(), rows.ctypes.data, rows.shape[0], rows.shape[1], _strs(names), float(period),
                             relation.encode(), instance_name.encode() if instance_name is not None else None,
                             int(frame_index), int(frame_time), len(classes), _strs([c[0] for c in classes]),
                             _strs([c[1] for c in classes]), _strs([c[2] for c in classes]), int(append), int(n_time_frames)):
        raise IOError(L.osm_b200_host_last_error().decode())


def _dptr(buf):
    return C.c_void_p(buf.data_ptr() if hasattr(buf, "data_ptr") else int(buf))


def write_htk_device(path, d_rows, n_rows, n_elements, period, parm_kind=9):
    """cHtkSink's file from rows resident in device memory: the big-endian payload is packed on the device (sinks.cu)"""
    L = capi.lib()
    L.osm_b200_write_htk_device.argtypes = [C.c_char_p, C.c_void_p, C.c_int64, C.c_int32, C.c_double, C.c_int32]
    if L.osm_b200_write_htk_device(str(path).encode(), _dptr(d_rows), int(n_rows), int(n_elements), float(period), parm_kind):
        raise IOError(L.osm_b200_host_last_error().decode())


def write_csv_device(path, d_rows, n_rows, names, period, instance_name=None, frame_index=True, frame_time=True, n_time_frames=0):
    """cCsvSink's file from rows resident in device memory: every value is formatted on the device (sinks.cu, text_format.cuh),
    the host adds the per-row prefix; byte-identical to write_csv"""
    L = capi.lib()
    L.osm_b200_write_csv_device.argtypes = [C.c_char_p, C.c_void_p, C.c_int64, C.c_int32, C.POINTER(C.c_char_p), C.c_double,
                                            C.c_char_p, C.c_int32, C.c_int32, C.c_int64]
    if L.osm_b200_write_csv_device(str(path).encode(), _dptr(d_rows), int(n_rows), len(names), _strs(names), float(period),
                                   instance_name.encode() if instance_name is not None else None, int(frame_index), int(frame_time),
                                   int(n_time_frames)):
        raise IOError(L.osm_b200_host_last_error().decode())

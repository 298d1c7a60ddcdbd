"""ctypes mirror of include/osm_b200.h and loader of the in-tree libosm_b200.so.

This is the reference-side binding a maintainer would add for Python callers (cf. the
reference's own ctypes wrapper progsrc/smileapi/python/opensmile/SMILEapi.py:18).  It loads
the CUDA back end and NOTHING else: if the shared library is missing the import of the
compute path fails loudly -- there is no CPU fallback.
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OSM_B200_LIB") or os.path.join(_HERE, "libosm_b200.so")   # override: A/B builds of the same library

NAME_LEN = 64
MAX_INPUTS = 8
MAX_LIST = 16

OK, ERR_INVALID, ERR_UNSUPPORTED, ERR_CUDA, ERR_NOMEM = range(5)

# component types (osm_b200_component_type)
(C_WAVESOURCE, C_FRAMER, C_VECTORPREEMPHASIS, C_WINDOWER, C_TRANSFORMFFT, C_FFTMAGPHASE,
 C_MELSPEC, C_MFCC, C_PLP, C_SPECTRAL, C_ENERGY, C_MZCR, C_ACF, C_PITCHACF,
 C_DELTAREGRESSION, C_CONTOURSMOOTHER, C_VECTORCONCAT, C_VECTOROPERATION, C_FULLINPUTMEAN, C_INTENSITY,
 C_SPECSCALE, C_PITCHSHS, C_PITCHSMOOTHERVITERBI, C_VALBASEDSELECTOR, C_PITCHJITTER,
 C_SPECRESAMPLE, C_LPC, C_FORMANTLPC, C_DATASELECTOR, C_HARMONICS, C_LSP, C_TONESPEC, C_CHROMA, C_TONEFILT, C_CENS) = range(35)

# cTonespec.filterType (osm_b200_tone_filter)
TONE_GAU, TONE_TRI, TONE_TRP, TONE_REC = range(4)

TYPE_BY_NAME = {
    "cWaveSource": C_WAVESOURCE, "cExternalAudioSource": C_WAVESOURCE, "cFramer": C_FRAMER,
    "cVectorPreemphasis": C_VECTORPREEMPHASIS, "cWindower": C_WINDOWER,
    "cTransformFFT": C_TRANSFORMFFT, "cFFTmagphase": C_FFTMAGPHASE, "cMelspec": C_MELSPEC,
    "cMfcc": C_MFCC, "cPlp": C_PLP, "cSpectral": C_SPECTRAL, "cEnergy": C_ENERGY,
    "cMZcr": C_MZCR, "cAcf": C_ACF, "cPitchACF": C_PITCHACF,
    "cDeltaRegression": C_DELTAREGRESSION, "cContourSmoother": C_CONTOURSMOOTHER,
    "cVectorConcat": C_VECTORCONCAT, "cVectorOperation": C_VECTOROPERATION,
    "cFullinputMean": C_FULLINPUTMEAN, "cIntensity": C_INTENSITY,
    "cSpecScale": C_SPECSCALE, "cPitchShs": C_PITCHSHS, "cPitchSmootherViterbi": C_PITCHSMOOTHERVITERBI,
    "cValbasedSelector": C_VALBASEDSELECTOR, "cPitchJitter": C_PITCHJITTER,
    "cSpecResample": C_SPECRESAMPLE, "cLpc": C_LPC, "cFormantLpc": C_FORMANTLPC,
    "cDataSelector": C_DATASELECTOR, "cHarmonics": C_HARMONICS, "cLsp": C_LSP,
    "cTonespec": C_TONESPEC, "cChroma": C_CHROMA, "cTonefilt": C_TONEFILT, "cCens": C_CENS,
}

WIN_BY_NAME = {"rec": 0, "han": 1, "ham": 2, "gau": 3, "sin": 4, "tri": 5, "bar": 6}

i32, f64 = C.c_int32, C.c_double


class WaveSource(C.Structure):
    _fields_ = [("sampleRate", f64), ("nChannels", i32), ("monoMixdown", i32), ("format", i32),
                ("outFieldName", C.c_char * NAME_LEN)]


class Framer(C.Structure):
    _fields_ = [("frameSize", f64), ("frameStep", f64), ("frameCenterSpecial", i32), ("frameCenterFramesSet", i32),
                ("frameCenter", f64), ("frameCenterFrames", i32), ("noPostEOIprocessing", i32)]


class VectorPreemphasis(C.Structure):
    _fields_ = [("k", f64), ("de", i32)]


class Windower(C.Structure):
    _fields_ = [("winFunc", i32), ("gain", f64), ("offset", f64), ("sigma", f64), ("alpha0", f64), ("alpha1", f64), ("alpha2", f64),
                ("alpha3", f64), ("fade", f64), ("squareRoot", i32)]


class TransformFFT(C.Structure):
    _fields_ = [("inverse", i32), ("zeroPadSymmetric", i32)]


class FFTmagphase(C.Structure):
    _fields_ = [("magnitude", i32), ("phase", i32), ("normalise", i32), ("power", i32), ("dBpsd", i32), ("dBpnorm", f64), ("mindBp", f64)]


class Melspec(C.Structure):
    _fields_ = [("nBands", i32), ("lofreq", f64), ("hifreq", f64), ("usePower", i32),
                ("htkcompatible", i32), ("specScale", i32), ("scaleParam", f64)]


class Mfcc(C.Structure):
    _fields_ = [("firstMfcc", i32), ("lastMfcc", i32), ("melfloor", f64), ("doLog", i32),
                ("cepLifter", f64), ("htkcompatible", i32)]


class Plp(C.Structure):
    _fields_ = [("lpOrder", i32), ("nCeps", i32), ("firstCC", i32), ("lastCC", i32),
                ("doLog", i32), ("doAud", i32), ("RASTA", i32), ("newRASTA", i32),
                ("doInvLog", i32), ("doIDFT", i32), ("doLP", i32), ("doLpToCeps", i32),
                ("rastaUpperCutoff", f64), ("rastaLowerCutoff", f64), ("cepLifter", f64),
                ("compression", f64), ("melfloor", f64), ("htkcompatible", i32)]


class Spectral(C.Structure):
    _fields_ = [("squareInput", i32),
                ("nBands", i32), ("bandLo", f64 * MAX_LIST), ("bandHi", f64 * MAX_LIST),
                ("nSlopes", i32), ("slopeLo", f64 * MAX_LIST), ("slopeHi", f64 * MAX_LIST),
                ("nRollOff", i32), ("rollOff", f64 * MAX_LIST),
                ("flux", i32), ("centroid", i32), ("maxPos", i32), ("minPos", i32), ("entropy", i32),
                ("standardDeviation", i32), ("variance", i32), ("skewness", i32), ("kurtosis", i32),
                ("slope", i32), ("alphaRatio", i32), ("hammarbergIndex", i32), ("sharpness", i32),
                ("harmonicity", i32), ("flatness", i32),
                ("normBandEnergies", i32), ("buggyRollOff", i32), ("oldSlopeScale", i32),
                ("useLogSpectrum", i32),
                ("freqRangeLo", f64), ("freqRangeHi", f64), ("specFloor", f64), ("logFlatness", i32)]


class Energy(C.Structure):
    _fields_ = [("htkcompatible", i32), ("rms", i32), ("energy2", i32), ("log", i32),
                ("escaleLog", f64), ("escaleRms", f64), ("escaleSquare", f64),
                ("ebiasLog", f64), ("ebiasRms", f64), ("ebiasSquare", f64)]


class MZcr(C.Structure):
    _fields_ = [("zcr", i32), ("mcr", i32), ("amax", i32), ("maxmin", i32), ("dc", i32)]


class Acf(C.Structure):
    _fields_ = [("usePower", i32), ("cepstrum", i32), ("inverse", i32), ("cosLifterCepstrum", i32),
                ("expBeforeAbs", i32), ("symmetricData", i32), ("acfCepsNormOutput", i32),
                ("oldCompatCepstrum", i32), ("absCepstrum", i32)]


class PitchACF(C.Structure):
    _fields_ = [("maxPitch", f64), ("voiceProb", i32), ("voiceQual", i32), ("HNR", i32),
                ("HNRdB", i32), ("linHNR", i32), ("F0", i32), ("F0raw", i32), ("F0env", i32),
                ("voicingCutoff", f64)]


class DeltaRegression(C.Structure):
    _fields_ = [("deltawin", i32), ("absOutput", i32), ("halfWaveRect", i32),
                ("onlyInSegments", i32), ("zeroSegBound", i32), ("relativeDelta", i32)]


class ContourSmoother(C.Structure):
    _fields_ = [("smaWin", i32), ("noZeroSma", i32)]


class VectorOperation(C.Structure):
    _fields_ = [("operation", i32), ("nameBase", C.c_char * NAME_LEN)]


class VectorConcat(C.Structure):
    _fields_ = [("processArrayFields", i32), ("includeSingleElementFields", i32)]


class FullinputMean(C.Structure):
    _fields_ = [("mvn", i32), ("meanNorm", i32), ("symmSubtract", i32), ("subtractClipToZero", i32),
                ("specEnorm", i32), ("htkLogEnorm", i32), ("excludeZeros", i32), ("multiLoopMode", i32)]


class Intensity(C.Structure):
    _fields_ = [("intensity", i32), ("loudness", i32)]


class SpecScale(C.Structure):
    _fields_ = [("scaleOctave", i32), ("sourceLin", i32), ("splineInterp", i32), ("minF", f64), ("maxF", f64),
                ("nPointsTarget", i32), ("specSmooth", i32), ("specEnhance", i32), ("auditoryWeighting", i32)]


class PitchShs(C.Structure):
    _fields_ = [("maxPitch", f64), ("minPitch", f64), ("nCandidates", i32), ("scores", i32), ("voicing", i32),
                ("F0C1", i32), ("voicingC1", i32), ("F0raw", i32), ("voicingClip", i32), ("voicingCutoff", f64),
                ("octaveCorrection", i32), ("nHarmonics", i32), ("compressionFactor", f64), ("greedyPeakAlgo", i32),
                ("lfCut", f64)]


class PitchSmootherViterbi(C.Structure):
    _fields_ = [("bufferLength", i32), ("F0final", i32), ("F0finalLog", i32), ("F0finalEnv", i32), ("F0finalEnvLog", i32),
                ("voicingFinalClipped", i32), ("voicingFinalUnclipped", i32), ("F0raw", i32), ("voicingC1", i32),
                ("voicingClip", i32), ("wLocal", f64), ("wTvv", f64), ("wTvvd", f64), ("wTvuv", f64), ("wThr", f64),
                ("wRange", f64), ("wTuu", f64)]


class ValbasedSelector(C.Structure):
    _fields_ = [("threshold", f64), ("idx", i32), ("invert", i32), ("allowEqual", i32), ("removeIdx", i32),
                ("zeroVec", i32), ("adaptiveThreshold", i32), ("outputVal", f64)]


class PitchJitter(C.Structure):
    _fields_ = [("F0reader_dmLevel", C.c_char * NAME_LEN), ("F0field", C.c_char * NAME_LEN), ("searchRangeRel", f64),
                ("jitterLocal", i32), ("jitterDDP", i32), ("jitterLocalEnv", i32), ("jitterDDPEnv", i32),
                ("shimmerLocal", i32), ("shimmerLocalDB", i32), ("shimmerLocalEnv", i32), ("shimmerLocalDBEnv", i32),
                ("harmonicERMS", i32), ("noiseERMS", i32), ("linearHNR", i32), ("logHNR", i32), ("lgHNRfloor", f64),
                ("shimmerUseRmsAmplitude", i32), ("minNumPeriods", i32), ("minCC", f64), ("refinedF0", i32),
                ("sourceQualityRange", i32), ("sourceQualityMean", i32), ("usePeakToPeakPeriodLength", i32),
                ("useBrokenJitterThresh", i32), ("onlyVoiced", i32)]


class SpecResample(C.Structure):
    _fields_ = [("targetFs", f64), ("resampleRatio", f64)]


class Lpc(C.Structure):
    _fields_ = [("method", i32), ("p", i32), ("saveLPCoeff", i32), ("lpGain", i32), ("saveRefCoeff", i32), ("residual", i32),
                ("residualGainScale", i32), ("forwardFilter", i32), ("lpSpectrum", i32)]


class FormantLpc(C.Structure):
    _fields_ = [("nFormants", i32), ("saveFormants", i32), ("saveIntensity", i32), ("saveNumberOfValidFormants", i32),
                ("saveBandwidths", i32), ("minF", f64), ("maxF", f64), ("useLpSpec", i32), ("medianFilter", i32),
                ("octaveCorrection", i32)]


class DataSelector(C.Structure):
    _fields_ = [("nSelected", i32), ("elementMode", i32), ("selected", (C.c_char * NAME_LEN) * 32),
                ("newNames", (C.c_char * NAME_LEN) * 32)]


class Harmonics(C.Structure):
    _fields_ = [("f0ElementName", C.c_char * NAME_LEN), ("magSpecFieldName", C.c_char * NAME_LEN),
                ("formantFrequencyFieldName", C.c_char * NAME_LEN), ("formantBandwidthFieldName", C.c_char * NAME_LEN),
                ("f0ElementNameIsFull", i32), ("magSpecFieldNameIsFull", i32), ("formantFrequencyFieldNameIsFull", i32),
                ("formantBandwidthFieldNameIsFull", i32), ("nHarmonics", i32), ("firstHarmonicMagnitude", i32),
                ("nHarmonicMagnitudes", i32), ("outputLogRelMagnitudes", i32), ("outputLinearMagnitudes", i32),
                ("nHarmonicDifferences", i32), ("harmonicDifferences", (C.c_char * 16) * 4), ("harmonicDifferencesLog", i32),
                ("harmonicDifferencesRatioLinear", i32), ("formantAmplitudes", i32), ("formantAmplitudesLinear", i32),
                ("formantAmplitudesLogRel", i32), ("formantAmplitudesStart", i32), ("formantAmplitudesEnd", i32),
                ("computeAcfHnrLogdB", i32), ("computeAcfHnrLinear", i32), ("logRelValueFloorUnvoiced", f64)]


class Lsp(C.Structure):
    _fields_ = [("processArrayFields", i32)]


class Tonespec(C.Structure):
    _fields_ = [("nOctaves", i32), ("firstNote", f64), ("filterType", i32), ("usePower", i32), ("dbA", i32)]


class Chroma(C.Structure):
    _fields_ = [("octaveSize", i32), ("silThresh", f64)]


class Tonefilt(C.Structure):
    _fields_ = [("nNotes", i32), ("firstNote", f64), ("decayF0", f64), ("decayFN", f64), ("outputPeriod", f64)]


class Cens(C.Structure):
    _fields_ = [("window", i32), ("winlength", i32), ("l2norm", i32), ("downsampleRatio", i32), ("winlength_sec", f64),
                ("winlength_secSet", i32)]


class _U(C.Union):
    _fields_ = [("wavesource", WaveSource), ("framer", Framer),
                ("vectorpreemphasis", VectorPreemphasis), ("windower", Windower),
                ("transformfft", TransformFFT), ("fftmagphase", FFTmagphase),
                ("melspec", Melspec), ("mfcc", Mfcc), ("plp", Plp), ("spectral", Spectral),
                ("energy", Energy), ("mzcr", MZcr), ("acf", Acf), ("pitchacf", PitchACF),
                ("deltaregression", DeltaRegression), ("contoursmoother", ContourSmoother),
                ("vectoroperation", VectorOperation), ("vectorconcat", VectorConcat), ("fullinputmean", FullinputMean), ("intensity", Intensity),
                ("specscale", SpecScale), ("pitchshs", PitchShs), ("pitchsmootherviterbi", PitchSmootherViterbi),
                ("valbasedselector", ValbasedSelector), ("pitchjitter", PitchJitter),
                ("specresample", SpecResample), ("lpc", Lpc), ("formantlpc", FormantLpc),
                ("dataselector", DataSelector), ("harmonics", Harmonics), ("lsp", Lsp),
                ("tonespec", Tonespec), ("chroma", Chroma), ("tonefilt", Tonefilt), ("cens", Cens)]


class Component(C.Structure):
    _fields_ = [("type", i32), ("name", C.c_char * NAME_LEN), ("n_inputs", i32),
                ("reader_dmLevel", (C.c_char * NAME_LEN) * MAX_INPUTS),
                ("writer_dmLevel", C.c_char * NAME_LEN),
                ("nameAppend", C.c_char * NAME_LEN), ("copyInputName", i32), ("u", _U)]


UNION_FIELD = {
    C_WAVESOURCE: "wavesource", C_FRAMER: "framer", C_VECTORPREEMPHASIS: "vectorpreemphasis",
    C_WINDOWER: "windower", C_TRANSFORMFFT: "transformfft", C_FFTMAGPHASE: "fftmagphase",
    C_MELSPEC: "melspec", C_MFCC: "mfcc", C_PLP: "plp", C_SPECTRAL: "spectral",
    C_ENERGY: "energy", C_MZCR: "mzcr", C_ACF: "acf", C_PITCHACF: "pitchacf",
    C_DELTAREGRESSION: "deltaregression", C_CONTOURSMOOTHER: "contoursmoother",
    C_VECTOROPERATION: "vectoroperation", C_VECTORCONCAT: "vectorconcat",
    C_FULLINPUTMEAN: "fullinputmean", C_INTENSITY: "intensity",
    C_SPECSCALE: "specscale", C_PITCHSHS: "pitchshs", C_PITCHSMOOTHERVITERBI: "pitchsmootherviterbi",
    C_VALBASEDSELECTOR: "valbasedselector", C_PITCHJITTER: "pitchjitter",
    C_SPECRESAMPLE: "specresample", C_LPC: "lpc", C_FORMANTLPC: "formantlpc", C_DATASELECTOR: "dataselector",
    C_HARMONICS: "harmonics", C_LSP: "lsp", C_TONESPEC: "tonespec", C_CHROMA: "chroma",
}

# every symbol include/osm_b200.h declares (tests assert the library exports all of them)
EXPORTS = [
    "osm_b200_abi_version", "osm_b200_sizeof_component", "osm_b200_last_error",
    "osm_b200_device_count", "osm_b200_component_defaults", "osm_b200_plan_create",
    "osm_b200_plan_destroy", "osm_b200_plan_num_elements", "osm_b200_plan_element_name",
    "osm_b200_plan_frame_period", "osm_b200_plan_row_time", "osm_b200_plan_frame_size_samples",
    "osm_b200_plan_frame_step_samples", "osm_b200_plan_fft_size", "osm_b200_plan_num_frames", "osm_b200_plan_num_time_frames",
    "osm_b200_plan_frame_offsets", "osm_b200_plan_run_device", "osm_b200_plan_run_host", "osm_b200_plan_run_host_resident",
    "osm_b200_window_table", "osm_b200_tone_tables", "osm_b200_plan_num_frames_first_eoi", "osm_b200_plan_num_frames_first_eoi_v", "osm_b200_plan_copy_seq_lag",
    "osm_b200_plan_run_device_padded", "osm_b200_plan_copy_seq_lag_stream", "osm_b200_plan_check_device_flags",
    # include/osm_b200_functionals.h
    "osm_b200_functionals_defaults", "osm_b200_functionals_create", "osm_b200_functionals_destroy", "osm_b200_functionals_num_values",
    "osm_b200_functionals_num_elements", "osm_b200_functionals_element_name", "osm_b200_functionals_run_device", "osm_b200_functionals_run_device_cols", "osm_b200_summary_assemble_device", "osm_b200_plan_sample_frame_bytes", "osm_b200_device_csv_slot_bytes", "osm_b200_device_format_csv", "osm_b200_device_format_rows",
    "osm_b200_device_pack_htk", "osm_b200_device_gather_rows", "osm_b200_write_csv_device", "osm_b200_write_htk_device", "osm_b200_functionals_run_host",
    "osm_b200_functionals_sizeof_spec",
    "osm_b200_plan_last_launch_count", "osm_b200_plan_take_device_flags", "osm_b200_plan_last_kernel_ms",
    "osm_b200_plan_last_kernel_times", "osm_b200_plan_set_profiling", "osm_b200_plan_profile_count", "osm_b200_plan_profile_entry",
    "osm_b200_plan_last_lld_launch",
    # include/osm_b200_host.h
    "osm_b200_session_open", "osm_b200_session_close", "osm_b200_session_num_elements",
    "osm_b200_session_element_name", "osm_b200_session_extract_files", "osm_b200_session_extract_files_arff", "osm_b200_session_sink_options",
    "osm_b200_session_write_files",
    "osm_b200_session_extract_pcm", "osm_b200_session_extract_device", "osm_b200_session_extract_device_lld", "osm_b200_session_extract_files_lld",
    "osm_b200_session_lld_num_elements", "osm_b200_session_lld_element_name", "osm_b200_session_components", "osm_b200_session_plan", "osm_b200_host_last_error",
    "osm_b200_write_htk", "osm_b200_write_csv", "osm_b200_write_csv_timed", "osm_b200_write_arff",
]

_lib = None


class BackendMissing(RuntimeError):
    pass


def lib():
    """Load libosm_b200.so (built in-tree by __graft_entry__.build()).  Fails loudly."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise BackendMissing(
            "%s not found: build the CUDA back end first (python -c 'import __graft_entry__ as g; "
            "g.build()').  opensmile_b200 has no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, i64p = C.c_void_p, C.POINTER(C.c_int64)
    L.osm_b200_abi_version.restype = i32
    L.osm_b200_sizeof_component.restype = i32
    L.osm_b200_last_error.restype = C.c_char_p
    L.osm_b200_device_count.restype = i32
    L.osm_b200_component_defaults.argtypes = [i32, C.POINTER(Component)]
    L.osm_b200_plan_create.argtypes = [C.POINTER(Component), i32, C.c_char_p, i32, C.POINTER(vp)]
    L.osm_b200_plan_destroy.argtypes = [vp]
    L.osm_b200_plan_destroy.restype = None
    L.osm_b200_plan_num_elements.argtypes = [vp]
    L.osm_b200_plan_element_name.argtypes = [vp, i32]
    L.osm_b200_plan_element_name.restype = C.c_char_p
    L.osm_b200_plan_frame_period.argtypes = [vp]
    L.osm_b200_plan_frame_period.restype = f64
    L.osm_b200_plan_row_time.argtypes = [vp, C.c_int64]
    L.osm_b200_plan_row_time.restype = f64
    for fn in ("frame_size_samples", "frame_step_samples", "fft_size", "last_launch_count"):
        getattr(L, "osm_b200_plan_" + fn).argtypes = [vp]
        getattr(L, "osm_b200_plan_" + fn).restype = i32
    L.osm_b200_plan_num_frames.argtypes = [vp, C.c_int64]
    L.osm_b200_plan_num_frames.restype = C.c_int64
    L.osm_b200_plan_num_time_frames.argtypes = [vp, C.c_int64]
    L.osm_b200_plan_num_time_frames.restype = C.c_int64
    L.osm_b200_plan_num_frames_first_eoi.argtypes = [vp, C.c_int64]
    L.osm_b200_plan_num_frames_first_eoi.restype = C.c_int64
    L.osm_b200_plan_frame_offsets.argtypes = [vp, i64p, i32, i64p]
    L.osm_b200_plan_run_device.argtypes = [vp, vp, i64p, i32, i64p, vp, vp]
    L.osm_b200_plan_run_host.argtypes = [vp, vp, i64p, i32, i64p, vp]
    L.osm_b200_plan_run_device_padded.argtypes = [vp, vp, C.c_int64, i64p, i32, i64p, vp, vp]
    L.osm_b200_plan_copy_seq_lag_stream.argtypes = [vp, C.POINTER(i32), i32, vp]
    L.osm_b200_plan_check_device_flags.argtypes = [vp, vp]
    L.osm_b200_plan_last_kernel_ms.argtypes = [vp]
    L.osm_b200_plan_last_kernel_ms.restype = C.c_float
    L.osm_b200_plan_last_kernel_times.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.osm_b200_plan_set_profiling.argtypes = [vp, i32]
    L.osm_b200_plan_set_profiling.restype = None
    L.osm_b200_plan_profile_count.argtypes = [vp]
    L.osm_b200_plan_profile_entry.argtypes = [vp, i32, C.POINTER(C.c_char_p), C.POINTER(C.c_float)]
    L.osm_b200_plan_last_lld_launch.argtypes = [vp, C.POINTER(C.c_char_p), C.POINTER(i32), i64p]
    # host front end (include/osm_b200_host.h)
    cpp = C.POINTER(C.c_char_p)
    L.osm_b200_session_open.argtypes = [C.c_char_p, i32, cpp, cpp, C.c_char_p, i32, C.POINTER(vp)]
    L.osm_b200_session_close.argtypes = [vp]
    L.osm_b200_session_close.restype = None
    L.osm_b200_session_num_elements.argtypes = [vp, f64, i32]
    L.osm_b200_session_element_name.argtypes = [vp, i32]
    L.osm_b200_session_element_name.restype = C.c_char_p
    L.osm_b200_session_extract_files.argtypes = [vp, i32, cpp, cpp, cpp, i64p]
    L.osm_b200_session_extract_files_arff.argtypes = [vp, i32, cpp, cpp, cpp, cpp, i64p]
    L.osm_b200_session_write_files.argtypes = [vp, C.c_double, i32, i32, i64p, i64p, C.c_void_p, cpp, cpp, cpp]
    L.osm_b200_session_write_files.restype = i32
    L.osm_b200_session_extract_pcm.argtypes = [vp, vp, i64p, i32, f64, i32, i64p, vp, C.c_int64]
    L.osm_b200_session_extract_device.argtypes = [vp, vp, i32, C.c_int64, i64p, i32, f64, i32, i64p, vp, C.c_int64, vp]
    L.osm_b200_session_extract_device_lld.argtypes = [vp, vp, i32, C.c_int64, i64p, i32, f64, i32, i64p, vp, C.c_int64, i64p, vp, C.c_int64, vp]
    L.osm_b200_session_extract_files_lld.argtypes = [vp, i32, cpp, cpp, cpp, cpp, cpp, cpp, cpp, i64p]
    L.osm_b200_session_lld_num_elements.argtypes = [vp, f64, i32]
    L.osm_b200_session_lld_element_name.argtypes = [vp, i32]
    L.osm_b200_session_lld_element_name.restype = C.c_char_p
    L.osm_b200_session_components.argtypes = [vp, f64, i32, C.POINTER(C.POINTER(Component)), cpp]
    L.osm_b200_host_last_error.restype = C.c_char_p
    L.osm_b200_write_htk.argtypes = [C.c_char_p, vp, C.c_int64, i32, f64, i32]
    L.osm_b200_write_csv.argtypes = [C.c_char_p, vp, C.c_int64, i32, cpp, f64, C.c_char_p, i32, i32]
    if L.osm_b200_sizeof_component() != C.sizeof(Component):
        raise RuntimeError("ABI mismatch: sizeof(osm_b200_component) = %d, ctypes mirror = %d"
                           % (L.osm_b200_sizeof_component(), C.sizeof(Component)))
    L.osm_b200_tone_tables.argtypes = [C.POINTER(Tonespec), i32, f64, vp, vp, vp, vp, vp]
    if L.osm_b200_component_defaults(C_CENS, C.byref(Component())) != 0:     # the last component type of this mirror
        raise RuntimeError("ABI mismatch: the library does not know component type %d (cCens)" % C_CENS)
    _lib = L
    return L


def last_error():
    return lib().osm_b200_last_error().decode()

"""Case table of the per-frame LLD kernels (lld512_kernel in csrc/lld_fast.cu, the lld_kernel instances in csrc/kernels.cu): test
infrastructure shared by test_lld_sweep_cpu.py and test_lld_sweep_gpu.py.  One dict per case; the plan's component list and the
oracle's configuration are both built from it, so the two cannot drift apart.  Sizes are in samples."""
import functools

import numpy as np

from opensmile_b200 import comp, components_frontend, pack_utterances
from opensmile_b200.synth import mixed_pcm, stereo_mixed_pcm, voiced_pcm
from oracle import oracle

FAST13, FAST16 = "lld512_kernel<13>", "lld512_kernel<16>"


def gen(m, f, nt, minb, vec2=True, kind="MFCC"):
    return "lld_kernel<%d,%d,%d,%d,%s,%s>" % (m, f, nt, minb, "VEC2" if vec2 else "SCALAR", kind)


G512 = gen(256, 32, 256, 2)


def case(name, expect, sr=16000, n_chan=1, frame=400, hop=160, preemph=0.97, win="ham", zps=0, op="mfcc", bands=26,
         lofreq=0.0, hifreq=8000.0, use_power=1, htk=1, first=0, last=12, lifter=22.0, windows=(2, 2), extremes=False):
    return dict(name=name, expect=expect, sr=float(sr), n_chan=n_chan, frame=frame, hop=hop, preemph=preemph, win=win, zps=zps,
                op=op, bands=bands, lofreq=lofreq, hifreq=hifreq, use_power=use_power, htk=htk, first=first, last=last,
                lifter=lifter, windows=windows, extremes=extremes)


CASES = [
    # ---- lld512_kernel: frame geometry (frames of 417..512 samples take the 16-row instance) ----
    case("fast_anchor_400_160", FAST13, extremes=True),
    case("fast_320_160_nope_hann_htk0", FAST13, frame=320, preemph=None, win="han", htk=0),
    case("fast_416_80", FAST13, frame=416, hop=80),
    case("fast_424_8", FAST16, frame=424, hop=8),
    case("fast_480_480", FAST16, frame=480, hop=480),
    case("fast_512_640_gaps", FAST16, frame=512, hop=640, zps=1),
    case("fast_8k_480_80", FAST16, sr=8000, frame=480, hop=80, hifreq=4000.0),
    # ---- lld512_kernel: band and cepstrum layouts ----
    case("fast_3_bands", FAST13, bands=3, last=2),
    case("fast_40_bands_16_coeffs", FAST13, bands=40, first=1, last=16),
    case("fast_64_bands_empty_ranges", FAST13, bands=64, last=15),
    case("fast_telephone_band_no_lifter", FAST13, bands=20, lofreq=300.0, hifreq=3400.0, lifter=0.0),
    case("fast_preemph_0_5", FAST13, preemph=0.5),
    # ---- the rules of the fast path that do not hold: lld_kernel ----
    case("gen512_17_coeffs", G512, last=16),
    case("gen512_magnitude_bands", G512, use_power=0),
    case("gen512_stereo", G512, n_chan=2),
    # ---- every other instance launch_lld can select ----
    case("gen512_hop161", gen(256, 32, 256, 2, vec2=False), hop=161),
    case("gen512_hop1", gen(256, 32, 256, 2, vec2=False), hop=1),
    case("gen512_hop3", gen(256, 32, 256, 2, vec2=False), hop=3),
    case("gen1024_16k_800", gen(512, 32, 512, 1), frame=800),
    case("gen1024_22k05", gen(512, 32, 512, 1, vec2=False), sr=22050, frame=551, hop=221, hifreq=11025.0),
    case("gen2048_48k_mono", gen(1024, 16, 512, 1), sr=48000, frame=1200, hop=480),
    case("gen2048_44k1_stereo", gen(1024, 16, 512, 1, vec2=False), sr=44100, n_chan=2, frame=1103, hop=441),
    case("gen2048_narrow_48k_stereo", gen(1024, 8, 256, 1), sr=48000, n_chan=2, frame=1200, hop=480, extremes=True),
    # 25 ms at 96 kHz takes the narrow 4096 tiles even in mono (the full tile needs more than 227 KB of shared memory);
    # short frames with an 8-sample hop fit the full width
    case("gen4096_96k_2056_8", gen(2048, 8, 256, 1), sr=96000, frame=2056, hop=8, hifreq=8000.0),
    case("gen4096_narrow_96k_mono", gen(2048, 4, 128, 1), sr=96000, frame=2400, hop=960, extremes=True),
    case("gen4096_narrow_96k_stereo", gen(2048, 4, 128, 1), sr=96000, n_chan=2, frame=2400, hop=960),
    case("plp_8k", gen(256, 32, 256, 2, kind="GEN"), op="plp", sr=8000, frame=400, hop=80, hifreq=4000.0),
    case("plp_16k", gen(256, 32, 256, 2, kind="GEN"), op="plp"),
    case("plp_44k1", gen(1024, 16, 512, 1, vec2=False, kind="GEN"), op="plp", sr=44100, frame=1103, hop=441),
]

# the regression windows (delta, delta-delta) on one tile width of each size: F = 32, 16, 8 (narrow 2048) and 4 (narrow 4096)
WINDOWS = [(1, 1), (1, 2), (2, 1), (2, 2), (3, 3), (4, 4), (5, 3), (5, 5), (6, 6)]
_WIN_BASES = [("16k", dict(expect=FAST13)),
              ("44k1", dict(expect=gen(1024, 16, 512, 1, vec2=False), sr=44100, frame=1103, hop=441)),
              ("96k", dict(expect=gen(2048, 4, 128, 1), sr=96000, frame=2400, hop=960)),
              ("48k_stereo", dict(expect=gen(1024, 8, 256, 1), sr=48000, n_chan=2, frame=1200, hop=480))]
for _b, _kw in _WIN_BASES:
    for _w in WINDOWS:
        CASES.append(case("win%d%d_%s" % (_w[0], _w[1], _b), windows=_w, extremes=(_w == (3, 3)), **_kw))
BY_NAME = {c["name"]: c for c in CASES}
assert len(BY_NAME) == len(CASES)


def tile_frames(c):
    """frames per tile of the instance the case expects"""
    k = c["expect"]
    return 32 if k.startswith("lld512") else int(k.split("<")[1].split(",")[1])


def is_fast(c):
    return c["expect"].startswith("lld512")


def expect_fused(c):
    """delta and delta-delta run inside the per-frame kernel when the halo W1 + W2 is at most 8 frames and its double fits a tile"""
    h = sum(c["windows"])
    return h <= 8 and 2 * h <= tile_frames(c)


def n_static(c):
    if c["op"] == "mfcc":
        return c["last"] - c["first"] + 1
    fe, ms, pl = oracle_cfg(c)[0]
    return int(oracle.lib().osm_or_plp_num_out(oracle.C.byref(pl), oracle.C.c_int(ms.n_bands)))


def components(c):
    sr, n, h = c["sr"], c["frame"], c["hop"]
    cs = components_frontend(sr, n / sr, h / sr, win=c["win"], preemph=c["preemph"], n_channels=c["n_chan"],
                             zero_pad_symmetric=c["zps"])
    cs.append(comp("cMelspec", "melspec", "mag", "melspec", nBands=c["bands"], lofreq=c["lofreq"], hifreq=c["hifreq"],
                   usePower=c["use_power"], htkcompatible=c["htk"]))
    if c["op"] == "mfcc":
        cs.append(comp("cMfcc", "mfcc", "melspec", "ft0", firstMfcc=c["first"], lastMfcc=c["last"], cepLifter=c["lifter"],
                       htkcompatible=c["htk"]))
    else:   # config/plp/PLP_0_D_A.conf
        cs.append(comp("cPlp", "plp", "melspec", "ft0", firstCC=0, lpOrder=5, cepLifter=22.0, compression=0.33, htkcompatible=1,
                       doIDFT=1, doLpToCeps=1, doLP=1, doInvLog=0, doAud=1, doLog=0))
    w1, w2 = c["windows"]
    cs += [comp("cDeltaRegression", "delta", "ft0", "ft0de", deltawin=w1),
           comp("cDeltaRegression", "accel", "ft0de", "ft0dede", deltawin=w2),
           comp("cVectorConcat", "lldconcat", "ft0;ft0de;ft0dede", "lld")]
    return cs


def oracle_cfg(c):
    """((Frontend, Melspec, Mfcc | Plp), (delta_win, accel_win)) of the oracle"""
    sr = c["sr"]
    fe = oracle.frontend(sr, c["frame"] / sr, c["hop"] / sr, c["win"], c["preemph"], zero_pad_symmetric=c["zps"])
    ms = oracle.Melspec(c["bands"], c["lofreq"], c["hifreq"], c["use_power"], c["htk"], 0, 0.0)
    if c["op"] == "mfcc":
        third = oracle.Mfcc(c["first"], c["last"], c["lifter"], 1e-8, c["htk"])
    else:
        third = oracle.Plp(5, 0, -1, 0, 1, 0, 1, 1, 1, 0, 0, 29.0, 1.0, 22.0, 0.33, 9.3e-10, 1)
    return (fe, ms, third), tuple(c["windows"])


def oracle_rows(c, x):
    """the oracle's [T, 3K] rows (static | delta | delta-delta) of one utterance"""
    cfg, (w1, w2) = oracle_cfg(c)
    fn = oracle.mfcc_d_a if c["op"] == "mfcc" else oracle.plp_d_a
    return fn(x, c["sr"], n_chan=c["n_chan"], cfg=cfg, delta_win=w1, accel_win=w2)


def _extremes(c, n):
    """digital silence, full-scale square wave, a run of -32768, a DC offset, an impulse on the first sample of the second tile"""
    F, h = tile_frames(c), c["hop"]
    t = np.arange(n)
    sq = np.where((t // 37) % 2 == 0, 32767, -32768)
    run = voiced_pcm(n, int(c["sr"]), seed=11).astype(np.int64)
    run[n // 3: n // 3 + 3 * c["frame"]] = -32768
    dc = voiced_pcm(n, int(c["sr"]), seed=12).astype(np.int64) // 4 + 12000
    imp = np.zeros(n, np.int64)
    imp[F * h] = 32767
    sigs = [np.zeros(n, np.int64), sq, run, dc, imp]
    return [np.repeat(s, c["n_chan"]).astype(np.int16) for s in sigs]


def utterances(c):
    """the ragged batch of a case: empty and too-short inputs, T = 1, 2, 3, H, 2H, F-1, F, F+1 frames, one chunk (16 F frames)
    -1 / +0 / +1 and + 2H -1 / +1, one utterance of more than five chunks, and with `extremes` the signals of _extremes.  Fillers
    of 1..7 samples (no frame) put the utterances' first samples on every residue mod 8."""
    N, S, F, H = c["frame"], c["hop"], tile_frames(c), sum(c["windows"])
    C = 16 * F
    frames = [1, 2, 3, H, 2 * H, F - 1, F, F + 1, C - 1, C, C + 1, C + 2 * H - 1, C + 2 * H + 1, 5 * C + 7]
    lens = [0, N - 1, N, N + S - 1] + [N + (T - 1) * S for T in frames]
    sr, nc = int(c["sr"]), c["n_chan"]
    sigs = []
    for i, n in enumerate(lens):
        if nc == 2:
            sigs.append(stereo_mixed_pcm(n, sr, seed=i) if i % 2 else voiced_pcm(n, sr, seed=i, n_chan=2))
        else:
            sigs.append(mixed_pcm(n, sr, seed=i) if i % 2 else voiced_pcm(n, sr, seed=i))
    if c["extremes"]:
        sigs += _extremes(c, N + (2 * F + 3) * S)
    out, start = [], 0
    for i, x in enumerate(sigs):
        r = (i - start) % 8
        if r:
            out.append(voiced_pcm(r, sr, seed=99, n_chan=nc))
            start += r
        out.append(x)
        start += len(x) // nc
    return out


@functools.lru_cache(maxsize=None)
def _batch(name):
    utts = utterances(BY_NAME[name])
    pcm, off = pack_utterances(utts, n_chan=BY_NAME[name]["n_chan"])
    return utts, pcm, off


def batch(c):
    """(utterances, pcm, utt_offsets), built once per case: callers do not modify them"""
    if BY_NAME.get(c["name"]) is c:
        return _batch(c["name"])
    utts = utterances(c)
    pcm, off = pack_utterances(utts, n_chan=c["n_chan"])
    return utts, pcm, off

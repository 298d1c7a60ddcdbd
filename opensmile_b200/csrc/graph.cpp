// graph.cpp -- resolves a component list (the .conf graph as handed over the C ABI) into a
// fused plan description.  This is the host-side analogue of cComponentManager's
// configure/finalise phase (src/core/componentManager.cpp:606-838) restricted to the LLD
// sub-graph: it follows reader.dmLevel / writer.dmLevel wiring, applies the per-component
// geometry rules (frame size rounding, FFT size, frameSizeSec rescale, frame counts, field
// names) and emits tables.  Citations relative to /root/reference/src.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>

#include "plan.hpp"

namespace osm {

namespace {

struct Resolver {
  const osm_b200_component *comps;
  int n;
  std::map<std::string, int> producer;  // level name -> component index

  const osm_b200_component *prod(const char *level) const {
    auto it = producer.find(level);
    return it == producer.end() ? nullptr : &comps[it->second];
  }
};

const char *type_name(int t)
{
  static const char *names[] = {"cWaveSource", "cFramer", "cVectorPreemphasis", "cWindower",
    "cTransformFFT", "cFFTmagphase", "cMelspec", "cMfcc", "cPlp", "cSpectral", "cEnergy",
    "cMZcr", "cAcf", "cPitchACF", "cDeltaRegression", "cContourSmoother", "cVectorConcat",
    "cVectorOperation", "cFullinputMean", "cIntensity", "cSpecScale", "cPitchShs", "cPitchSmootherViterbi",
    "cValbasedSelector", "cPitchJitter", "cSpecResample", "cLpc", "cFormantLpc", "cDataSelector", "cHarmonics", "cLsp",
    "cTonespec", "cChroma", "cTonefilt", "cCens"};
  return (t >= 0 && t < OSM_B200_C_COUNT_) ? names[t] : "?";
}

// default nameAppend per type (ConfigType defaults: dspcore/deltaRegression.cpp:34,
// dspcore/contourSmoother.cpp:33, lldcore/mfcc.cpp:33, dspcore/acf.cpp:46, lldcore/energy.cpp:33)
const char *default_name_append(int t)
{
  switch (t) {
    case OSM_B200_C_MFCC: return "mfcc";
    case OSM_B200_C_DELTAREGRESSION: return "de";
    case OSM_B200_C_CONTOURSMOOTHER: return "sma";
    case OSM_B200_C_ACF: return "acf";
    case OSM_B200_C_ENERGY: return "energy";
    case OSM_B200_C_TONESPEC: return "note";       // lld/tonespec.cpp:47
    case OSM_B200_C_CHROMA: return "chroma";       // lld/chroma.cpp:46
    case OSM_B200_C_TONEFILT: return "tonefilt";   // lld/tonefilt.cpp:35
    case OSM_B200_C_CENS: return "CENS";           // lld/cens.cpp:41
    default: return "";
  }
}

// cDataProcessor::addNameAppendFieldAuto (core/dataProcessor.cpp:272-325)
std::string name_append_auto(const osm_b200_component &c, const std::string &base, const char *customFixed)
{
  std::string na = c.nameAppend[0] ? c.nameAppend : default_name_append(c.type);
  std::string tail = std::string(customFixed ? customFixed : "") + na;
  if (!tail.empty()) {
    if (c.copyInputName && !base.empty()) return base + "_" + tail;
    return tail;
  }
  if (c.copyInputName && !base.empty()) return base;
  return "noname";
}

}  // namespace

// core/winToVecProcessor.cpp:868-877 (noPostEOIprocessing=1): only complete frames (frame_geom.cuh).
// A cTonefilt stream (GraphCompiler::get_tonefilt_stream) reads blocks of P samples with hop P and gets one more, padded block
// for a remainder at end of input: ceil(L / P) rows, which is this rule for a "frame" of 1 sample and a step of P.
int64_t desc_num_static_frames(const PlanDesc &d, int stream, int64_t L)
{
  const FrontEnd &fe = d.streams[stream].fe;
  return frame_count(L, fe.frameSize, fe.frameStep, fe.frameCenter);
}

int64_t desc_max_static_frames(const PlanDesc &d, int64_t L)
{
  int64_t m = 0;
  for (size_t s = 0; s < d.streams.size(); s++) m = std::max<int64_t>(m, desc_num_static_frames(d, (int)s, L));
  return m;
}

// window processors emit T + W frames at EOI (core/dataMemoryLevel.cpp:1022-1026 via
// core/windowProcessor.cpp:85-119); cVectorConcat emits min over its inputs
// (core/dataReader.cpp:375-380).
int64_t desc_num_frames(const PlanDesc &d, int64_t L)
{
  int64_t best = -1;
  for (const auto &g : d.groups) {
    int64_t t = desc_num_static_frames(d, g.stream, L);
    for (int ls : g.limitStreams) t = std::min<int64_t>(t, desc_num_static_frames(d, ls, L));
    if (t <= 0) return 0;
    for (const auto &s : g.stages) t += s.win;
    if (best < 0 || (d.padRows ? t > best : t < best)) best = t;
  }
  return best < 0 ? 0 : best;
}

// Frames of the output level that exist when a full-input reader (cFunctionals with frameMode = full) ticks for the first time
// after end of input was raised.  The reference's window processors run with blocksize 1: stage s has produced
// c0_s = max(c0_{s-1} - W_s, 0) frames before EOI (tick-order model, see post_kernel) and adds exactly one more in the first EOI
// tick before the components behind it tick; the reader then takes what is there (core/dataReader.cpp:560-585) and, having read
// once, never reads again -- so the frames the window processors append later are NOT part of the summary unless the
// configuration sets EOIlevel (the shipped IS09 / IS10 files do not).  Verified against the reference's functionals rows
// (tests/test_functionals_cpu.py).
// Levels behind the SHS pitch chain (lagKind != 0): the Viterbi smoother has written V frames when end of input is raised
// (data dependent, osm_b200_plan_copy_seq_lag); cPitchJitter does not run while end of input is set (lld/pitchJitter.cpp:593), so the
// chain's static level still holds min(V, T) frames in the first EOI tick: a smoother behind it ends at V rows, its delta at V - 2
// (pinned on the reference's ComParE_2016 functionals rows: V = 143 / 193 / 198 -> 143 | 141, 193 | 191, 198 | 196).
int64_t desc_num_frames_first_eoi(const PlanDesc &d, int64_t L, int64_t V)
{
  int64_t best = -1;
  for (const auto &g : d.groups) {
    int64_t t = desc_num_static_frames(d, g.stream, L);
    for (int ls : g.limitStreams) t = std::min<int64_t>(t, desc_num_static_frames(d, ls, L));
    if (t <= 0) return 0;
    if (g.lagKind != 0 && V >= 0) t = std::min<int64_t>(t, V);
    int64_t c0 = t, fin = t;
    for (const auto &s : g.stages) { c0 = std::max<int64_t>(c0 - s.win, 0); fin += s.win; }
    const int64_t avail = g.stages.empty() ? t : std::min<int64_t>(c0 + 1, fin);
    if (best < 0 || avail < best) best = avail;
  }
  return best < 0 ? 0 : best;
}


namespace {

struct ChainInfo {               // resolved front-end chain below a static producer
  const osm_b200_component *wav = nullptr, *frm = nullptr, *pe = nullptr, *win = nullptr, *fft = nullptr, *mag = nullptr;
};

// ---- leaves of the output level ----
// The output level is a tree: temporal stages (cDeltaRegression / cContourSmoother, one input
// level each) and cVectorConcat nodes over static producers.  Temporal stages work element by
// element, so stage(concat(a, b)) = concat(stage(a), stage(b)) as long as concat does not
// truncate (all inputs equally long); every leaf becomes one output group carrying the stages
// between it and the output level.
struct Leaf { const osm_b200_component *c; std::vector<const osm_b200_component *> stages; bool arraysOnly; };
struct ConcatCheck { size_t g0, g1, above; };          // leaves [g0, g1) sit below a concat that has stages above it
struct SelScope { const osm_b200_component *c; size_t l0, l1, above; };   // leaves [l0, l1) sit below selector c, `above` stages above it
// leaves [l0, l1) are the data levels of a cValbasedSelector (zeroVec = 1) that gates them element-wise with a column of the pitch level
struct GateScope { const osm_b200_component *c; size_t l0, l1, above; };
struct GateInfo { int col, pitchOp; };

std::string wave_name(const ChainInfo &ci)
{
  return ci.wav->u.wavesource.outFieldName[0] ? ci.wav->u.wavesource.outFieldName : "pcm";
}

void add_field(StaticOp &op, const std::string &name, int n = 1, int arrNameOffset = 0)
{
  FieldName f;
  f.name = name; f.n = n; f.arrNameOffset = arrNameOffset;
  op.fields.push_back(f);
}

int field_elements(const StaticOp &op)
{
  int n = 0;
  for (const FieldName &f : op.fields) n += f.n;
  return n;
}

// the first field of op that `match` accepts; col = its first column within the op's columns
template <class Match>
const FieldName *find_field(const StaticOp &op, Match match, int &col)
{
  col = 0;
  for (const FieldName &f : op.fields) {
    if (match(f)) return &f;
    col += f.n;
  }
  return nullptr;
}

// a field named `name`, or (full = false) whose name contains it
auto name_match(const char *name, bool full)
{
  return [name, full](const FieldName &f) { return full ? f.name == name : f.name.find(name) != std::string::npos; };
}

// element names: name (single element fields) or name[idx + arrNameOffset] (core/dataMemoryLevel.cpp:1158-1169)
void append_element_names(const FieldName &f, std::vector<std::string> &out)
{
  if (f.n == 1) { out.push_back(f.name); return; }
  char buf[512];
  for (int i = 0; i < f.n; i++) {
    snprintf(buf, sizeof buf, "%s[%d]", f.name.c_str(), i + f.arrNameOffset);
    out.push_back(buf);
  }
}

bool same_geometry(const FrontEnd &a, const FrontEnd &b)
{
  return a.frameSize == b.frameSize && a.frameStep == b.frameStep && a.frameCenter == b.frameCenter;
}

// a level of geometry x delivers at least the rows of a level of geometry ref: same frame step, frames not longer
bool delivers_rows_of(const FrontEnd &x, const FrontEnd &ref)
{
  return x.frameStep == ref.frameStep && x.frameCenter == ref.frameCenter && x.frameSize <= ref.frameSize;
}

// The phases of compile_graph, the state they hand on to each other, and one builder per static producer family.  Ops and
// streams are numbered in the order get_op / get_stream create them, so the phases and builders keep their call order.
struct GraphCompiler {
  Resolver R;
  PlanDesc &d;
  std::string &err;
  std::map<const osm_b200_component *, int> staticOpOf;   // static producer -> op index
  std::vector<Leaf> leaves;
  std::vector<std::pair<size_t, size_t>> leafGroups;   // leaf -> its groups [first, last)
  std::vector<std::vector<std::string>> leafSelNames;   // per leaf: element names as a selector above it sees them
  std::vector<ConcatCheck> concatChecks;
  std::vector<SelScope> selScopes;
  bool inSelector = false;
  std::vector<GateScope> gateScopes;
  std::vector<GateInfo> gateInfo;                      // per gate scope
  std::vector<const osm_b200_component *> segComps;     // cDeltaRegression instances with onlyInSegments=1

  GraphCompiler(const osm_b200_component *comps, int n, PlanDesc &d_, std::string &err_) : R{comps, n, {}}, d(d_), err(err_) {}

  const osm_b200_component *single_input(const osm_b200_component *c) const
  {
    if (!c || c->n_inputs != 1) return nullptr;
    return R.prod(c->reader_dmLevel[0]);
  }

  osm_b200_status index_writers(const char *outputLevel)
  {
    char buf[512];
    int nWave = 0;
    for (int i = 0; i < R.n; i++) {
      const osm_b200_component &c = R.comps[i];
      if (c.type < 0 || c.type >= OSM_B200_C_COUNT_) { err = "unknown component type"; return OSM_B200_ERR_INVALID; }
      if (c.type == OSM_B200_C_WAVESOURCE) nWave++;
      if (!c.writer_dmLevel[0]) { err = "component without writer.dmLevel"; return OSM_B200_ERR_INVALID; }
      if (R.producer.count(c.writer_dmLevel)) {
        snprintf(buf, sizeof buf, "level '%s' has more than one writer", c.writer_dmLevel);
        err = buf; return OSM_B200_ERR_INVALID;   // one writer per level (core/dataWriter.cpp)
      }
      R.producer[c.writer_dmLevel] = i;
    }
    if (nWave != 1) { err = "graph must contain exactly one cWaveSource"; return OSM_B200_ERR_INVALID; }
    if (!outputLevel || !R.prod(outputLevel)) { err = "output level has no writer"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // walk from a time-domain level (framer / pre-emphasis / windower output) down to the wave source
  bool resolve_time_chain(const osm_b200_component *x, ChainInfo &ci)
  {
    if (x && x->type == OSM_B200_C_WINDOWER) { ci.win = x; x = single_input(x); }
    if (x && x->type == OSM_B200_C_VECTORPREEMPHASIS) { ci.pe = x; x = single_input(x); }
    if (!x || x->type != OSM_B200_C_FRAMER) { err = "expected cFramer [-> cVectorPreemphasis] [-> cWindower] below this component"; return false; }
    ci.frm = x;
    ci.wav = single_input(x);
    if (!ci.wav || ci.wav->type != OSM_B200_C_WAVESOURCE) { err = "cFramer must read the cWaveSource level"; return false; }
    return true;
  }

  bool resolve_mag_chain(const osm_b200_component *mag, ChainInfo &ci, bool asOutput = false)
  {
    if (!mag || mag->type != OSM_B200_C_FFTMAGPHASE) { err = "expected a cFFTmagphase level"; return false; }
    ci.mag = mag;
    const auto &mp = mag->u.fftmagphase;
    if ((!mp.magnitude && !mp.dBpsd) || mp.phase) { err = "cFFTmagphase: only magnitude=1 without phase is supported"; return false; }
    if (!asOutput && (mp.normalise || mp.power || mp.dBpsd)) {
      err = "cFFTmagphase: normalise / power / dBpsd are supported where the level is the output level only (its consumers read the plain magnitude)"; return false;
    }
    ci.fft = single_input(mag);
    if (!ci.fft || ci.fft->type != OSM_B200_C_TRANSFORMFFT) { err = "cFFTmagphase must read a cTransformFFT level"; return false; }
    if (ci.fft->u.transformfft.inverse) { err = "cTransformFFT.inverse=1 is not supported"; return false; }
    const osm_b200_component *w = single_input(ci.fft);
    if (!w || w->type != OSM_B200_C_WINDOWER) { err = "cTransformFFT must read a cWindower level"; return false; }
    return resolve_time_chain(w, ci);
  }

  // find or create the stream of a chain; needFft extends an existing time-only stream
  osm_b200_status get_stream(const ChainInfo &ci, bool needFft, int &idx)
  {
    for (size_t s = 0; s < d.streams.size(); s++) {
      Stream &st = d.streams[s];
      // a framer-level reader may share a windowed stream (same geometry); a windowed chain needs its own window
      if (st.keyFramer == ci.frm && st.keyPe == ci.pe && (!ci.win || st.keyWin == ci.win)) {
        if (needFft && !st.hasFft) continue;
        idx = (int)s;
        return OSM_B200_OK;
      }
    }
    Stream st;
    FrontEnd &fe = st.fe;
    const auto &wp = ci.wav->u.wavesource;
    if (wp.sampleRate <= 0 || wp.nChannels < 1) { err = "cWaveSource: bad sampleRate/nChannels"; return OSM_B200_ERR_INVALID; }
    if (wp.nChannels > 1 && !wp.monoMixdown) { err = "multi-channel without monoMixdown is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    if (wp.format < OSM_B200_PCM_S16 || wp.format > OSM_B200_PCM_S32) { err = "cWaveSource: unknown sample format"; return OSM_B200_ERR_INVALID; }
    fe.sampleRate = wp.sampleRate; fe.nChan = wp.nChannels; fe.format = wp.format; fe.mixdown = true;
    // cWinToVecProcessor::configureWriter (core/winToVecProcessor.cpp:435-456)
    const auto &fp = ci.frm->u.framer;
    if (!fp.noPostEOIprocessing) { err = "cFramer: only noPostEOIprocessing=1 is supported"; return OSM_B200_ERR_UNSUPPORTED; }
    const double T = 1.0 / wp.sampleRate;
    double frameSize = fp.frameSize, frameStep = fp.frameStep;
    long fsf = (long)round(frameSize / T);
    if (frameStep == 0.0) frameStep = frameSize;
    long fstf = (long)round(frameStep / T);
    if (fstf == 0) fstf = fsf;
    if (fsf < 2) { err = "cFramer: frame too short"; return OSM_B200_ERR_INVALID; }
    fe.frameSize = (int)fsf; fe.frameStep = (int)fstf;
    fe.frameSizeSec = frameSize; fe.frameStepSec = frameStep;
    // sampling centre (core/winToVecProcessor.cpp:461-501), resolved at this stream's sample rate
    double center = 0.0;
    long cf = 0;
    if (fp.frameCenterSpecial != OSM_B200_CENTER_UNSET) {
      if (fp.frameCenterSpecial == OSM_B200_CENTER_MID) center = frameSize / 2.0;
      else if (fp.frameCenterSpecial == OSM_B200_CENTER_RIGHT) cf = fsf - 1;
      if (cf == 0) cf = (long)round(center / T);
    } else if (fp.frameCenterFramesSet) {
      cf = fp.frameCenterFrames;
      center = cf * T;
    } else {
      center = fp.frameCenter;
      cf = (long)round(center / T);
    }
    fe.frameCenter = (int)std::min(std::max(cf, 0L), fsf - 1);
    // frame times: the time of the first sample read, + frameCenter where the (unclamped) centre in samples is > 0
    // (core/winToVecProcessor.cpp:1076-1079); `right` leaves frameCenter at 0
    fe.timeOffset = cf > 0 ? center : 0.0;
    if (ci.pe) {
      fe.preemph = true;
      fe.preK = (float)ci.pe->u.vectorpreemphasis.k;     // dspcore/vectorPreemphasis.cpp:55
      fe.preDe = ci.pe->u.vectorpreemphasis.de;
    }
    if (ci.win) {
      const auto &wnp = ci.win->u.windower;
      { const double al[4] = {wnp.alpha0, wnp.alpha1, wnp.alpha2, wnp.alpha3};
        build_window(wnp.winFunc, fe.frameSize, wnp.sigma, wnp.gain, fe.window, al, wnp.squareRoot, std::min(std::max(wnp.fade, 0.0), 0.5)); }
      fe.winOffset = (float)wnp.offset;
      st.hasWindow = true;
    } else {
      fe.window.assign(fe.frameSize, 1.0f);
    }
    // cTransformFFT: next power of two >= frame size, >= 4 (dspcore/transformFft.cpp:124-129);
    // frameSizeSec *= nfft/frameSize (:78-85, SURVEY.md H2)
    int nfft = 4;
    while (nfft < fe.frameSize) nfft <<= 1;
    fe.nfft = nfft; fe.nBins = nfft / 2 + 1;
    fe.fftFrameSizeSec = frameSize;
    if (nfft != fe.frameSize) fe.fftFrameSizeSec *= (double)nfft / (double)fe.frameSize;
    if (ci.fft) fe.zeroPadSymmetric = ci.fft->u.transformfft.zeroPadSymmetric != 0;
    st.hasFft = needFft;
    st.keyFramer = ci.frm; st.keyPe = ci.pe; st.keyWin = ci.win;
    d.streams.push_back(st);
    idx = (int)d.streams.size() - 1;
    return OSM_B200_OK;
  }

  osm_b200_status expand(const std::string &lvl, std::vector<const osm_b200_component *> above, int depth, bool arraysOnly)
  {
    if (depth > 8) { err = "level graph nested too deeply (cycle?)"; return OSM_B200_ERR_INVALID; }
    const osm_b200_component *c = R.prod(lvl.c_str());
    if (!c) { err = "level '" + lvl + "' has no writer"; return OSM_B200_ERR_INVALID; }
    std::vector<const osm_b200_component *> stageComps;
    // a temporal stage reading several levels (reader.dmLevel = a;b) sees their implicit concat
    // (core/dataReader.cpp:360-444), i.e. it behaves like stage(cVectorConcat(a, b))
    bool multi = false;
    while (c && (c->type == OSM_B200_C_DELTAREGRESSION || c->type == OSM_B200_C_CONTOURSMOOTHER || c->type == OSM_B200_C_FULLINPUTMEAN)) {
      stageComps.insert(stageComps.begin(), c);
      if (c->n_inputs > 1) { multi = true; break; }
      c = single_input(c);
    }
    if (!c) { err = "broken temporal chain below level '" + lvl + "'"; return OSM_B200_ERR_INVALID; }
    stageComps.insert(stageComps.end(), above.begin(), above.end());
    if (c->type == OSM_B200_C_DATASELECTOR && !multi) {
      // cDataSelector (core/dataSelector.cpp:296-366): picks elements of its (implicitly concatenated) input levels by
      // exact name, in the order of `selected`, each as a single-element field.  Element-wise like the temporal
      // stages, so stage(select(x)) = select(stage(x)): the leaves below carry the stages, the selection is applied
      // to the output groups afterwards (selector scopes).
      const auto &q = c->u.dataselector;
      if (!q.elementMode) { err = "cDataSelector.elementMode=0 is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      if (q.nSelected < 1) { err = "cDataSelector: no elements selected"; return OSM_B200_ERR_INVALID; }
      if (arraysOnly) { err = "cDataSelector below a cVectorConcat that drops single-element fields is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      if (inSelector) { err = "nested cDataSelector levels are not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      if (c->n_inputs < 1) { err = "cDataSelector without inputs"; return OSM_B200_ERR_INVALID; }
      const size_t l0 = leaves.size();
      inSelector = true;
      for (int i = 0; i < c->n_inputs; i++) {
        osm_b200_status s2 = expand(c->reader_dmLevel[i], stageComps, depth + 1, false);
        if (s2 != OSM_B200_OK) { inSelector = false; return s2; }
      }
      inSelector = false;
      if (!stageComps.empty() && c->n_inputs > 1) concatChecks.push_back({l0, leaves.size(), stageComps.size()});
      selScopes.push_back(SelScope{c, l0, leaves.size(), stageComps.size()});
      return OSM_B200_OK;
    }
    if (c->type == OSM_B200_C_VALBASEDSELECTOR && !multi &&
        !(c->n_inputs == 2 && R.prod(c->reader_dmLevel[1]) && R.prod(c->reader_dmLevel[1])->type == OSM_B200_C_PITCHSMOOTHERVITERBI)) {
      // cValbasedSelector over [selector level ; data levels ...] with zeroVec = 1 (GeMAPSv01b_core.lld.conf.inc:395-433: formants /
      // spectral parameters of the voiced resp. unvoiced frames): every frame is written, its elements either copied or set to
      // outputVal, so the gate works element by element like the temporal stages above it.  The pitch chain's own selector
      // ([energy ; cPitchSmootherViterbi level]) is part of the SHS pitch op (build_pitch_chain_op).
      const auto &q = c->u.valbasedselector;
      if (c->n_inputs < 2) { err = "cValbasedSelector must read at least two levels: selector;data"; return OSM_B200_ERR_UNSUPPORTED; }
      if (q.idx != 0 || !q.removeIdx || !q.zeroVec || q.adaptiveThreshold) { err = "cValbasedSelector: only idx=0, removeIdx=1, zeroVec=1, adaptiveThreshold=0 are supported"; return OSM_B200_ERR_UNSUPPORTED; }
      if (arraysOnly) { err = "cValbasedSelector below a cVectorConcat that drops single-element fields is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      for (const GateScope &gs : gateScopes) if (gs.l1 == (size_t)-1) { err = "nested cValbasedSelector levels are not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      const size_t l0 = leaves.size();
      gateScopes.push_back(GateScope{c, l0, (size_t)-1, stageComps.size()});
      const size_t me = gateScopes.size() - 1;
      for (int i = 1; i < c->n_inputs; i++) {
        osm_b200_status s2 = expand(c->reader_dmLevel[i], stageComps, depth + 1, false);
        if (s2 != OSM_B200_OK) return s2;
      }
      gateScopes[me].l1 = leaves.size();
      for (size_t l = l0; l < leaves.size(); l++)
        if (leaves[l].stages.size() != stageComps.size()) { err = "cValbasedSelector reading an already smoothed level is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      if (!stageComps.empty() && c->n_inputs > 2) concatChecks.push_back({l0, leaves.size(), stageComps.size()});
      return OSM_B200_OK;
    }
    if (c->type == OSM_B200_C_VECTORCONCAT || multi) {
      if (c->n_inputs < 1) { err = "cVectorConcat without inputs"; return OSM_B200_ERR_INVALID; }
      // a real cVectorConcat is a cVectorProcessor: with processArrayFields=1 it drops single-element
      // fields unless includeSingleElementFields=1 (core/vectorProcessor.cpp:196-243)
      if (!multi && c->u.vectorconcat.processArrayFields == 1 && !c->u.vectorconcat.includeSingleElementFields) arraysOnly = true;
      if (!multi && c->u.vectorconcat.processArrayFields == 2) { err = "cVectorConcat.processArrayFields=2 is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      const size_t g0 = leaves.size();
      for (int i = 0; i < c->n_inputs; i++) {
        osm_b200_status s2 = expand(c->reader_dmLevel[i], stageComps, depth + 1, arraysOnly);
        if (s2 != OSM_B200_OK) return s2;
      }
      if (!stageComps.empty()) concatChecks.push_back({g0, leaves.size(), stageComps.size()});
      return OSM_B200_OK;
    }
    leaves.push_back(Leaf{c, stageComps, arraysOnly});
    return OSM_B200_OK;
  }

  // static feature producer of component c (created on first use)
  osm_b200_status get_op(const osm_b200_component *c, int &opIdx)
  {
    auto it = staticOpOf.find(c);
    if (it != staticOpOf.end()) { opIdx = it->second; return OSM_B200_OK; }
    StaticOp op;
    osm_b200_status s;
    switch (c->type) {
      case OSM_B200_C_MELSPEC: case OSM_B200_C_MFCC: case OSM_B200_C_PLP: s = build_band_op(c, op); break;
      case OSM_B200_C_SPECTRAL: s = build_spectral_op(c, op); break;
      case OSM_B200_C_PITCHACF: s = build_pitch_acf_op(c, op); break;
      case OSM_B200_C_ENERGY: case OSM_B200_C_MZCR: case OSM_B200_C_INTENSITY: s = build_time_op(c, op); break;
      case OSM_B200_C_FFTMAGPHASE: s = build_mag_op(c, op); break;
      case OSM_B200_C_VECTOROPERATION: s = build_vecop(c, op); break;
      case OSM_B200_C_FORMANTLPC: s = build_formant_op(c, op); break;
      case OSM_B200_C_LPC: case OSM_B200_C_LSP: s = build_lpc_op(c, op); break;
      case OSM_B200_C_HARMONICS: s = build_harmonics_op(c, op); break;
      case OSM_B200_C_VALBASEDSELECTOR: case OSM_B200_C_PITCHSMOOTHERVITERBI: case OSM_B200_C_PITCHSHS: s = build_pitch_chain_op(c, op); break;
      case OSM_B200_C_PITCHJITTER: s = build_jitter_op(c, op); break;
      case OSM_B200_C_TONESPEC: case OSM_B200_C_CHROMA: s = build_tone_op(c, op); break;
      case OSM_B200_C_TONEFILT: s = build_tonefilt_op(c, op); break;
      case OSM_B200_C_CENS: s = build_cens_op(c, op); break;
      default: {
        char buf[512];
        snprintf(buf, sizeof buf, "component '%s' (%s) is not a supported static LLD producer", c->name, type_name(c->type));
        err = buf; return OSM_B200_ERR_UNSUPPORTED;
      }
    }
    if (s != OSM_B200_OK) return s;
    if (op.kind != SOP_TONEFILT && op.kind != SOP_VECOP && op.kind != SOP_CENS && d.streams[op.stream].fe.frameCenter != 0 && !centred_ok(op)) {
      char buf[512];
      snprintf(buf, sizeof buf, "component '%s' (%s) on a centred cFramer level (frameCenterSpecial / frameCenter / "
               "frameCenterFrames) is not supported", c->name, type_name(c->type));
      err = buf; return OSM_B200_ERR_UNSUPPORTED;
    }
    op.nOut = field_elements(op);
    op.outCol = d.nStatic;
    d.nStatic += op.nOut;
    d.ops.push_back(op);
    opIdx = (int)d.ops.size() - 1;
    staticOpOf[c] = opIdx;
    return OSM_B200_OK;
  }

  // Consumers whose rows on a centred stream (frames that start with copies of sample 0) are pinned on the reference's output
  // (tests/test_centred_frames_gpu.py: emo_large.conf and tests/configs/centred_frames.conf): cMfcc, cMelspec, cPlp without
  // RASTA filtering, cSpectral, cAcf / cPitchACF, cEnergy and cMZcr.
  static bool centred_ok(const StaticOp &op)
  {
    switch (op.kind) {
      case SOP_MFCC: case SOP_MELSPEC: case SOP_SPECTRAL: case SOP_PITCHACF: case SOP_ENERGY: case SOP_MZCR:
        return true;
      case SOP_PLP: return op.plp.rasta == 0;
      default: return false;
    }
  }

  // cMelspec's filter bank on the bins of fe, appended to d.mels
  bool add_mel_bank(const osm_b200_melspec &melp, const FrontEnd &fe)
  {
    if (melp.nBands < 1 || melp.nBands > 64 || melp.nBands >= fe.nBins) { err = "cMelspec.nBands out of range"; return false; }
    MelBank mb;
    build_mel(melp, fe.nBins, fe.fftFrameSizeSec, mb);
    d.mels.push_back(mb);
    return true;
  }

  // cMfcc / cPlp on a cMelspec level, or the band level itself as an output
  osm_b200_status build_band_op(const osm_b200_component *c, StaticOp &op)
  {
    const osm_b200_component *mel = c;
    if (c->type != OSM_B200_C_MELSPEC) {
      mel = single_input(c);
      if (!mel || mel->type != OSM_B200_C_MELSPEC) { err = "cMfcc / cPlp must read a cMelspec level"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    ChainInfo ci;
    if (!resolve_mag_chain(single_input(mel), ci)) return OSM_B200_ERR_UNSUPPORTED;
    osm_b200_status s2 = get_stream(ci, true, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    const FrontEnd &fe = d.streams[op.stream].fe;
    // field base name: outFieldName -> (pe/win/fft keep) -> fftMag -> melspec keeps (no default nameAppend, lldcore/melspec.cpp:175-178)
    const std::string magName = name_append_auto(*ci.mag, wave_name(ci), "fftMag");        // dspcore/fftmagphase.cpp:154
    const std::string melName = name_append_auto(*mel, magName, nullptr);
    const auto &melp = mel->u.melspec;
    if (!add_mel_bank(melp, fe)) return OSM_B200_ERR_UNSUPPORTED;
    const int melIdx = (int)d.mels.size() - 1;
    if (c->type == OSM_B200_C_MELSPEC) {
      // the band level itself as an output (log-mel spectrogram style graphs): the band values behind the kernel's filterbank
      // phase, i.e. the cPlp back end with every stage switched off (doLog = doAud = doInvLog = doIDFT = doLP = doLpToCeps = 0
      // hands the bands through, lldcore/plp.cpp:416-593) -- the band sums and the htk scaling are cMelspec's own (a-7)
      osm_b200_plp off;
      memset(&off, 0, sizeof off);
      off.firstCC = 0; off.lastCC = -1; off.nCeps = -1; off.compression = 1.0;
      op.kind = SOP_PLP;
      if (!build_plp(off, d.mels.back(), fe.frameStepSec, op.plp, err)) return OSM_B200_ERR_UNSUPPORTED;
      op.plp.melIdx = melIdx;
      if (op.plp.nOut != melp.nBands) { err = "internal: cMelspec pass-through width"; return OSM_B200_ERR_INVALID; }
      add_field(op, melName, op.plp.nOut);
    } else if (c->type == OSM_B200_C_MFCC) {
      op.kind = SOP_MFCC;
      const auto &mfp = c->u.mfcc;
      if (mfp.lastMfcc < mfp.firstMfcc || mfp.firstMfcc < 0 || mfp.lastMfcc >= melp.nBands) { err = "cMfcc: bad firstMfcc/lastMfcc"; return OSM_B200_ERR_INVALID; }
      build_mfcc(mfp, melp.nBands, op.mfcc);
      op.mfcc.melIdx = melIdx;
      add_field(op, name_append_auto(*c, melName, nullptr), op.mfcc.nMfcc, op.mfcc.first);   // lldcore/mfcc.cpp:120-128
    } else {
      op.kind = SOP_PLP;
      if (!build_plp(c->u.plp, d.mels.back(), fe.frameStepSec, op.plp, err)) return OSM_B200_ERR_UNSUPPORTED;
      op.plp.melIdx = melIdx;
      // lldcore/plp.cpp:232-267 replaces the field name, then cVectorProcessor appends nameAppend
      const int ra = op.plp.rasta;
      const char *fixed = op.plp.doLpToCeps ? (ra ? "RASTAPlpCC" : "PlpCC")
                        : (op.plp.doLP ? (ra == 1 ? "RASTAPlpc" : (ra == 2 ? "newRASTAPlpc" : "Plpc"))
                        : (op.plp.doIDFT ? "audAutoCor" : "audSpec"));
      add_field(op, name_append_auto(*c, fixed, nullptr), op.plp.nOut);
    }
    return OSM_B200_OK;
  }

  osm_b200_status build_spectral_op(const osm_b200_component *c, StaticOp &op)
  {
    ChainInfo ci;
    if (!resolve_mag_chain(single_input(c), ci)) return OSM_B200_ERR_UNSUPPORTED;
    osm_b200_status s2 = get_stream(ci, true, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    const FrontEnd &fe = d.streams[op.stream].fe;
    op.kind = SOP_SPECTRAL;
    if (!build_spectral(c->u.spectral, fe.nBins, fe.fftFrameSizeSec, op.spectral, err)) return OSM_B200_ERR_UNSUPPORTED;
    const std::string base = name_append_auto(*ci.mag, wave_name(ci), "fftMag");
    // element names, lldcore/spectral.cpp:378-584
    const auto &sc = c->u.spectral;
    const bool lg = sc.useLogSpectrum != 0;
    char buf[512];
    auto add = [&](const std::string &suffix) { add_field(op, base + "_" + suffix); };
    for (int i = 0; i < sc.nBands; i++)
      if ((long)sc.bandLo[i] >= 0 && (long)sc.bandHi[i] > 0) { snprintf(buf, sizeof buf, "%s%ld-%ld", lg ? "logFband" : "fband", (long)sc.bandLo[i], (long)sc.bandHi[i]); add(buf); }
    for (int i = 0; i < sc.nSlopes; i++)
      if ((long)sc.slopeLo[i] >= 0 && (long)sc.slopeHi[i] > 0) { snprintf(buf, sizeof buf, "%s%ld-%ld", lg ? "logSpectralSlopeOfBand" : "spectralSlopeOfBand", (long)sc.slopeLo[i], (long)sc.slopeHi[i]); add(buf); }
    if (sc.alphaRatio) add(lg ? "alphaRatioDB" : "alphaRatio");
    if (sc.hammarbergIndex) add(lg ? "hammarbergIndexDB" : "hammarbergIndex");
    for (size_t i = 0; i < op.spectral.rollOff.size(); i++) { snprintf(buf, sizeof buf, "spectralRollOff%.1f", op.spectral.rollOff[i] * 100.0); add(buf); }
    if (sc.flux) add("spectralFlux");
    if (sc.centroid) add(lg ? "logSpectralCentroid" : "spectralCentroid");
    if (sc.maxPos) add("spectralMaxPos");
    if (sc.minPos) add("spectralMinPos");
    if (sc.entropy) add(lg ? "logSpectralEntropy" : "spectralEntropy");
    if (sc.standardDeviation) add(lg ? "logSpectralStdDev" : "spectralStdDev");
    if (sc.variance) add(lg ? "logSpectralVariance" : "spectralVariance");
    if (sc.skewness) add(lg ? "logSpectralSkewness" : "spectralSkewness");
    if (sc.kurtosis) add(lg ? "logSpectralKurtosis" : "spectralKurtosis");
    if (sc.slope) add(lg ? "logSpectralSlope" : "spectralSlope");
    if (sc.sharpness) add("psySharpness");
    if (sc.harmonicity) add(lg ? "logSpectralHarmonicity" : "spectralHarmonicity");
    if (sc.flatness) add(lg ? "logSpectralFlatness" : "spectralFlatness");
    if (field_elements(op) != op.spectral.nOut) { err = "internal: cSpectral name/element mismatch"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // reader.dmLevel = <acf level>;<cepstrum level> (lldcore/pitchACF.cpp:148-152), both cAcf instances on the same magnitude level
  osm_b200_status build_pitch_acf_op(const osm_b200_component *c, StaticOp &op)
  {
    if (c->n_inputs != 2) { err = "cPitchACF must read two levels: acf;cepstrum"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *a = R.prod(c->reader_dmLevel[0]), *b = R.prod(c->reader_dmLevel[1]);
    if (!a || !b || a->type != OSM_B200_C_ACF || b->type != OSM_B200_C_ACF) { err = "cPitchACF inputs must be cAcf levels"; return OSM_B200_ERR_UNSUPPORTED; }
    if (a->u.acf.cepstrum || !b->u.acf.cepstrum) { err = "cPitchACF expects [acf ; cepstrum] in this order"; return OSM_B200_ERR_UNSUPPORTED; }
    for (const osm_b200_component *x : {a, b}) {
      const auto &q = x->u.acf;
      if (q.inverse || q.cosLifterCepstrum || !q.symmetricData) { err = "cAcf: inverse / cosLifterCepstrum / symmetricData=0 are not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    // oldCompatCepstrum only changes the cepstrum's input stage; on the ACF instance it has no effect (dspcore/acf.cpp:103-109,276)
    if (single_input(a) != single_input(b)) { err = "both cAcf instances must read the same cFFTmagphase level"; return OSM_B200_ERR_UNSUPPORTED; }
    ChainInfo ci;
    if (!resolve_mag_chain(single_input(a), ci)) return OSM_B200_ERR_UNSUPPORTED;
    osm_b200_status s2 = get_stream(ci, true, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    const FrontEnd &fe = d.streams[op.stream].fe;
    op.kind = SOP_PITCHACF;
    PitchAcfOp &po = op.pitch;
    po.acfUsePower = a->u.acf.usePower != 0; po.cepUsePower = b->u.acf.usePower != 0;
    po.oldCompatCepstrum = b->u.acf.oldCompatCepstrum != 0;
    po.absCepstrum = b->u.acf.absCepstrum != 0 || po.oldCompatCepstrum;                  // oldCompatCepstrum forces absCepstrum = 1
    po.normOutput = a->u.acf.acfCepsNormOutput != 0;
    const bool cepNorm = b->u.acf.acfCepsNormOutput != 0 && !po.oldCompatCepstrum;     // ... and acfCepsNormOutput = 0
    if (cepNorm != po.normOutput) { err = "cAcf.acfCepsNormOutput must agree on both instances"; return OSM_B200_ERR_UNSUPPORTED; }
    const auto &pp = c->u.pitchacf;
    po.maxPitch = pp.maxPitch < 0.0 ? 0.0 : pp.maxPitch;                       // lldcore/pitchACF.cpp:101-102
    po.voicingCutoff = pp.voicingCutoff > 1.0 ? 1.0 : (pp.voicingCutoff < 0.0 ? 0.0 : pp.voicingCutoff);
    po.fsSec = (float)fe.fftFrameSizeSec;                                       // :107-110
    po.voiceProb = pp.voiceProb != 0; po.voiceQual = pp.voiceQual != 0; po.HNR = pp.HNR != 0; po.HNRdB = pp.HNRdB != 0;
    po.linHNR = pp.linHNR != 0; po.F0 = pp.F0 != 0; po.F0raw = pp.F0raw != 0; po.F0env = pp.F0env != 0;
    const std::pair<bool, const char *> outputs[] = {                           // :112-121
      {po.voiceProb, "voiceProb"}, {po.HNR, "HNR"}, {po.HNRdB, "HNRdBacf"}, {po.linHNR, "linearHNRacf"},
      {po.voiceQual, "voiceQual"}, {po.F0, "F0"}, {po.F0raw, "F0raw"}, {po.F0env, "F0env"}};
    for (const auto &o : outputs) if (o.first) add_field(op, o.second);
    po.nOut = (int)op.fields.size();
    if (po.nOut < 1) { err = "cPitchACF produces no output"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // cEnergy, cMZcr, cIntensity on a time-domain frame level
  osm_b200_status build_time_op(const osm_b200_component *c, StaticOp &op)
  {
    ChainInfo ci;
    if (!resolve_time_chain(single_input(c), ci)) return OSM_B200_ERR_UNSUPPORTED;
    op.windowed = ci.win != nullptr;
    if (ci.pe && !ci.win) { err = "cEnergy / cMZcr reading a pre-emphasised, un-windowed level is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    osm_b200_status s2 = get_stream(ci, false, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    const std::string base = wave_name(ci);
    if (c->type == OSM_B200_C_ENERGY) {
      op.kind = SOP_ENERGY;
      build_energy(c->u.energy, op.energy);
      // lldcore/energy.cpp:97-125: addNameAppendFieldAuto(name, "RMS"|"SQUARED"|"LOG")
      if (op.energy.rms) add_field(op, name_append_auto(*c, base, "RMS"));
      if (op.energy.energy2) add_field(op, name_append_auto(*c, base, "SQUARED"));
      if (op.energy.lg) add_field(op, name_append_auto(*c, base, "LOG"));
    } else if (c->type == OSM_B200_C_INTENSITY) {
      op.kind = SOP_INTENSITY;
      IntensityOp &io = op.intensity;
      io.intensity = c->u.intensity.intensity != 0; io.loudness = c->u.intensity.loudness != 0;
      io.nOut = (io.intensity ? 1 : 0) + (io.loudness ? 1 : 0);
      // Hamming window of the frame length (smileutil/smileUtil.c:1291-1303), summed in index order
      const int N = d.streams[op.stream].fe.frameSize;
      io.winSum = 0.0;
      for (int j = 0; j < N; j++) {
        const double w = 0.54 - 0.46 * cos((2.0 * M_PI * (double)j) / ((double)N - 1.0));
        if (j < 2) io.w[j] = w;
        io.winSum += w;
      }
      if (io.winSum <= 0.0) io.winSum = 1.0;
      if (io.intensity) add_field(op, name_append_auto(*c, base, "intensity"));   // lldcore/intensity.cpp:91-92
      if (io.loudness) add_field(op, name_append_auto(*c, base, "loudness"));
    } else {
      op.kind = SOP_MZCR;
      build_mzcr(c->u.mzcr, op.mzcr);
      auto add = [&](const char *suffix) { add_field(op, base + "_" + suffix); };   // lldcore/mzcr.cpp:68-100
      if (op.mzcr.zcr) add("zcr");
      if (op.mzcr.mcr) add("mcr");
      if (op.mzcr.amax) add("absmax");
      if (op.mzcr.maxmin) { add("max"); add("min"); }
      if (op.mzcr.dc) add("dc");
    }
    if (op.fields.empty()) { err = "component produces no output"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // the magnitude level itself as an output (config/spectrum/spectrogram.conf): nBins elements
  osm_b200_status build_mag_op(const osm_b200_component *c, StaticOp &op)
  {
    ChainInfo ci;
    if (!resolve_mag_chain(c, ci, true)) return OSM_B200_ERR_UNSUPPORTED;
    osm_b200_status s2 = get_stream(ci, true, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    op.kind = SOP_MAG;
    const auto &mp = c->u.fftmagphase;
    const bool norm = mp.normalise || mp.dBpsd;                          // dBpsd implies normalise (:92)
    op.magMode = mp.dBpsd ? 4 : (norm && mp.power ? 3 : (mp.power ? 2 : (norm ? 1 : 0)));
    op.magDbNorm = (float)mp.dBpnorm;
    op.magMinDb = (float)mp.mindBp;
    if (op.magMinDb - op.magDbNorm < -120.0f) op.magMinDb = -120.0f + op.magDbNorm;      // :95-98
    const char *fixed = mp.dBpsd ? "fftMag_dBsplPSD" : (mp.power && !norm ? "fftMag_PowSpec" : (mp.power ? "fftMag_PowSpecDens" : (norm ? "fftMag_SpecDens" : "fftMag")));   // :141-155
    add_field(op, name_append_auto(*c, wave_name(ci), fixed), d.streams[op.stream].fe.nBins);
    return OSM_B200_OK;
  }

  // n -> 1 reduction of another static level (other/vectorOperation.cpp:475-481, names :226-249)
  osm_b200_status build_vecop(const osm_b200_component *c, StaticOp &op)
  {
    if (c->u.vectoroperation.operation != 0) { err = "cVectorOperation: only operation=ll1 is supported"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *in = single_input(c);
    if (!in) { err = "cVectorOperation must read exactly one level"; return OSM_B200_ERR_UNSUPPORTED; }
    int src = -1;
    osm_b200_status s2 = get_op(in, src);
    if (s2 != OSM_B200_OK) return s2;
    if (d.ops[src].fields.size() != 1) { err = "cVectorOperation: the input level must hold exactly one field"; return OSM_B200_ERR_UNSUPPORTED; }
    op.kind = SOP_VECOP;
    op.srcOp = src;
    op.stream = d.ops[src].stream;
    osm_b200_component named = *c;
    if (!named.nameAppend[0]) snprintf(named.nameAppend, sizeof named.nameAppend, "%s", "lengthL1norm");
    const std::string inName = c->u.vectoroperation.nameBase[0] ? std::string(c->u.vectoroperation.nameBase) : d.ops[src].fields[0].name;
    add_field(op, name_append_auto(named, inName, nullptr));
    return OSM_B200_OK;
  }

  // cCens on a cChroma level of either chroma front end (cTonespec or cTonefilt): a row-wise op on the chroma op's static columns
  // (cens.cu).  Every input row gives an output row; downsampleRatio scales the level's period only (lld/cens.cpp:107-114,178).
  osm_b200_status build_cens_op(const osm_b200_component *c, StaticOp &op)
  {
    const auto &q = c->u.cens;
    if (c->n_inputs > 1) { err = std::string("cCens '") + c->name + "': a multi-field input (more than one input level) is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *in = single_input(c);
    if (!in || in->type != OSM_B200_C_CHROMA) {
      err = std::string("cCens '") + c->name + "' must read a cChroma level (it quantises chroma energies)"; return OSM_B200_ERR_UNSUPPORTED;
    }
    if (q.winlength_secSet) {
      // lld/cens.cpp:91-100 reads the input level's period in myFetchConfig, before the reader's level is configured: the reference
      // dereferences a null level configuration and crashes, so there is no behaviour to reproduce
      err = std::string("cCens '") + c->name + "': winlength_sec is not supported (set winlength in frames)"; return OSM_B200_ERR_UNSUPPORTED;
    }
    const int W = q.winlength < 1 ? 1 : q.winlength;                    // :103
    if (W > kCensMaxTaps) {
      err = std::string("cCens '") + c->name + "': winlength " + std::to_string(W) + " is above " + std::to_string(kCensMaxTaps) + " taps";
      return OSM_B200_ERR_UNSUPPORTED;
    }
    int src = -1;
    osm_b200_status s2 = get_op(in, src);
    if (s2 != OSM_B200_OK) return s2;
    if (d.ops[src].fields.size() != 1) { err = std::string("cCens '") + c->name + "': the chroma level must hold exactly one field"; return OSM_B200_ERR_UNSUPPORTED; }
    op.kind = SOP_CENS;
    op.srcOp = src;
    op.stream = d.ops[src].stream;
    CensOp &co = op.cens;
    co.N = d.ops[src].fields[0].n;
    co.W = W;
    co.l2norm = q.l2norm != 0;
    co.ratio = q.downsampleRatio < 1 ? 1 : q.downsampleRatio;        // :102
    const int win = q.window == OSM_B200_WIN_HAMMING || q.window == OSM_B200_WIN_BARTLETT ? q.window : OSM_B200_WIN_HANNING;
    build_window(win, W, 0.0, 1.0, co.win);                             // (FLOAT_DMEM)_win[j], :123-128,185
    co.unit = (float)(1.0 / std::sqrt((float)co.N));                    // :203, the float overload of sqrt
    add_field(op, name_append_auto(*c, d.ops[src].fields[0].name, nullptr), co.N);
    return OSM_B200_OK;
  }

  // cFormantLpc <- cLpc <- cSpecResample <- cTransformFFT <- cWindower chain (GeMAPSv01b_core.lld.conf.inc:250-286)
  osm_b200_status build_formant_op(const osm_b200_component *c, StaticOp &op)
  {
    const osm_b200_component *lpc = single_input(c);
    if (!lpc || lpc->type != OSM_B200_C_LPC) { err = "cFormantLpc must read a cLpc level"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *rsm = single_input(lpc);
    if (!rsm || rsm->type != OSM_B200_C_SPECRESAMPLE) { err = "cLpc must read a cSpecResample level"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *fft = single_input(rsm);
    if (!fft || fft->type != OSM_B200_C_TRANSFORMFFT || fft->u.transformfft.inverse) { err = "cSpecResample must read a (forward) cTransformFFT level"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *w = single_input(fft);
    if (!w || w->type != OSM_B200_C_WINDOWER) { err = "cTransformFFT must read a cWindower level"; return OSM_B200_ERR_UNSUPPORTED; }
    ChainInfo ci;
    if (!resolve_time_chain(w, ci)) return OSM_B200_ERR_UNSUPPORTED;
    op.windowed = true;
    osm_b200_status s2 = get_stream(ci, false, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    op.kind = SOP_FORMANT;
    if (!build_formant(rsm->u.specresample, lpc->u.lpc, c->u.formantlpc, d.streams[op.stream].fe,
                       fft->u.transformfft.zeroPadSymmetric != 0, op.formant, err)) return OSM_B200_ERR_UNSUPPORTED;
    // lld/formantLpc.cpp:113-136: fixed field names, array indices start at 1
    if (op.formant.saveNValid) add_field(op, "nFormants");
    if (op.formant.saveFormants) add_field(op, "formantFreqLpc", op.formant.nFormants, 1);
    if (op.formant.saveBandwidths) add_field(op, "formantBandwidthLpc", op.formant.nFormants, 1);
    if (field_elements(op) != op.formant.nOut) { err = "internal: cFormantLpc name/element mismatch"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // stand-alone cLpc (method acf) on a time-domain frame level [framer -> pre-emphasis -> window], and cLsp on such a
  // cLpc level (config/emobase/emobase.conf: cVectorPreemphasis -> cLpc p = 8 -> cLsp).  Both are cVectorProcessors
  // that keep the frame count of the level they read.
  osm_b200_status build_lpc_op(const osm_b200_component *c, StaticOp &op)
  {
    const osm_b200_component *lpc = c;
    if (c->type == OSM_B200_C_LSP) {
      if (c->u.lsp.processArrayFields != 0) { err = "cLsp.processArrayFields=1 is not supported (the reference's cLsp finds its input field only with processArrayFields=0)"; return OSM_B200_ERR_UNSUPPORTED; }
      lpc = single_input(c);
      if (!lpc || lpc->type != OSM_B200_C_LPC || !lpc->u.lpc.saveLPCoeff) { err = "cLsp must read a level with an lpcCoeff field (a cLpc level with saveLPCoeff=1)"; return OSM_B200_ERR_UNSUPPORTED; }
      // lld/lsp.cpp:289-292: with more input elements than lspFreq outputs (Ndst < Nsrc) the reference's cLsp writes nothing
      if (lpc->u.lpc.lpGain) { err = "cLsp reading a cLpc level that also holds lpGain is not supported (Ndst < Nsrc: the reference's cLsp returns without output, lld/lsp.cpp:292)"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    const auto &q = lpc->u.lpc;
    if (q.method != 0) { err = "cLpc: only method=acf is supported (burg is not)"; return OSM_B200_ERR_UNSUPPORTED; }
    if (q.saveRefCoeff || q.residual || q.forwardFilter || q.lpSpectrum) { err = "cLpc: saveRefCoeff / residual / forwardFilter / lpSpectrum are not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    if (q.p < 1 || q.p > 16) { err = "cLpc.p must be in 1..16"; return OSM_B200_ERR_UNSUPPORTED; }
    if (!q.saveLPCoeff && !q.lpGain) { err = "cLpc produces no output"; return OSM_B200_ERR_INVALID; }
    const osm_b200_component *in = single_input(lpc);
    if (in && in->type == OSM_B200_C_SPECRESAMPLE) {
      err = c->type == OSM_B200_C_LSP ? "cLsp behind the formant chain's cSpecResample -> cLpc is not supported"
                                      : "cLpc on a cSpecResample level is supported only in front of cFormantLpc";
      return OSM_B200_ERR_UNSUPPORTED;
    }
    ChainInfo ci;
    if (!resolve_time_chain(in, ci)) { err = "cLpc: " + err; return OSM_B200_ERR_UNSUPPORTED; }
    op.windowed = ci.win != nullptr;
    osm_b200_status s2 = get_stream(ci, false, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    op.kind = SOP_LPC;
    op.lpc.p = q.p;
    if (c->type == OSM_B200_C_LSP) {                                     // lld/lsp.cpp:272-287
      op.lpc.lpc = false; op.lpc.lsp = true;
      add_field(op, "lspFreq", q.p);
    } else {                                                             // lld/lpc.cpp:118-146
      op.lpc.lpc = q.saveLPCoeff != 0; op.lpc.gain = q.lpGain != 0;
      if (op.lpc.lpc) add_field(op, "lpcCoeff", q.p);
      if (op.lpc.gain) add_field(op, "lpGain");
    }
    return OSM_B200_OK;
  }

  // cHarmonics reads [pitch level ; formant level ; magnitude level] through one multi-level reader
  // (GeMAPSv01b_core.lld.conf.inc:289-318) and looks its inputs up by name (lld/harmonics.cpp:258-300)
  osm_b200_status build_harmonics_op(const osm_b200_component *c, StaticOp &op)
  {
    const auto &q = c->u.harmonics;
    const osm_b200_component *pit = nullptr, *fmt = nullptr, *mg = nullptr;
    for (int i = 0; i < c->n_inputs; i++) {
      const osm_b200_component *x = R.prod(c->reader_dmLevel[i]);
      if (!x) { err = std::string("level '") + c->reader_dmLevel[i] + "' has no writer"; return OSM_B200_ERR_INVALID; }
      if (x->type == OSM_B200_C_VALBASEDSELECTOR || x->type == OSM_B200_C_PITCHSMOOTHERVITERBI) pit = x;
      else if (x->type == OSM_B200_C_FORMANTLPC) fmt = x;
      else if (x->type == OSM_B200_C_FFTMAGPHASE) mg = x;
      else { err = "cHarmonics: inputs must be a Viterbi-smoothed pitch level, a cFormantLpc level and a cFFTmagphase level"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    if (!pit || !mg || c->n_inputs > 3) { err = "cHarmonics needs a pitch level and a magnitude level (and optionally a formant level)"; return OSM_B200_ERR_UNSUPPORTED; }
    if (q.nHarmonicMagnitudes > 0 || q.outputLinearMagnitudes || q.harmonicDifferencesRatioLinear || q.formantAmplitudesLinear || q.computeAcfHnrLinear) {
      err = "cHarmonics: harmonic magnitudes / linear outputs are not supported (log differences, log formant amplitudes, HNR in dB only)"; return OSM_B200_ERR_UNSUPPORTED;
    }
    ChainInfo ci;
    if (!resolve_mag_chain(mg, ci)) return OSM_B200_ERR_UNSUPPORTED;
    HarmonicsOp &ho = op.harmonics;
    osm_b200_status s3 = get_op(pit, ho.pitchOp);
    if (s3 != OSM_B200_OK) return s3;
    if (fmt) { s3 = get_op(fmt, ho.formantOp); if (s3 != OSM_B200_OK) return s3; }
    osm_b200_status s2 = get_stream(ci, true, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    const FrontEnd &fe = d.streams[op.stream].fe;
    if (!same_geometry(d.streams[d.ops[ho.pitchOp].stream].fe, fe)) { err = "cHarmonics: the pitch level and the magnitude level must share the frame geometry"; return OSM_B200_ERR_UNSUPPORTED; }
    if (fmt && !delivers_rows_of(d.streams[d.ops[ho.formantOp].stream].fe, fe)) { err = "cHarmonics: the formant level must have the same frame step and frames no longer than the magnitude level's"; return OSM_B200_ERR_UNSUPPORTED; }
    // the magnitude field (name of the cFFTmagphase level, dspcore/fftmagphase.cpp:154)
    {
      const std::string magName = name_append_auto(*mg, wave_name(ci), "fftMag");
      const bool ok = q.magSpecFieldNameIsFull ? magName == q.magSpecFieldName : magName.find(q.magSpecFieldName) != std::string::npos;
      if (!ok) { err = "cHarmonics: magSpecFieldName '" + std::string(q.magSpecFieldName) + "' does not match the magnitude level's field '" + magName + "'"; return OSM_B200_ERR_INVALID; }
    }
    int col = 0;
    const FieldName *f0 = find_field(d.ops[ho.pitchOp], name_match(q.f0ElementName, q.f0ElementNameIsFull != 0), col);
    if (!f0 || f0->n != 1) {
      err = "cHarmonics: f0ElementName '" + std::string(q.f0ElementName) + "' not found in the pitch level"; return OSM_B200_ERR_INVALID;
    }
    ho.f0Col = d.ops[ho.pitchOp].outCol + col;
    bool fa = q.formantAmplitudes != 0 && q.formantAmplitudesLogRel != 0;
    bool haveFormantDiff = false;
    if (fmt && q.formantFrequencyFieldName[0]) {
      const StaticOp &fop = d.ops[ho.formantOp];
      const FieldName *ff = find_field(fop, name_match(q.formantFrequencyFieldName, q.formantFrequencyFieldNameIsFull != 0), col);
      if (!ff) {
        err = "cHarmonics: formantFrequencyFieldName '" + std::string(q.formantFrequencyFieldName) + "' not found in the formant level"; return OSM_B200_ERR_INVALID;
      }
      ho.fmtCol = fop.outCol + col; ho.nFmt = ff->n;
      const FieldName *bw = q.formantBandwidthFieldName[0] ? find_field(fop, name_match(q.formantBandwidthFieldName, q.formantBandwidthFieldNameIsFull != 0), col) : nullptr;
      if (!bw || bw->n != ho.nFmt) {
        err = "cHarmonics: formantBandwidthFieldName must name the bandwidth field of the formant level (lld/harmonics.cpp:270-296)"; return OSM_B200_ERR_UNSUPPORTED;
      }
      if (ho.nFmt > 8) { err = "cHarmonics: more than 8 formants"; return OSM_B200_ERR_UNSUPPORTED; }
    } else fa = false;
    // harmonicDifferences: "H<i>-H<j>", "H<i>-A<k>", ... (:84-160); A0 = the fundamental
    int maxHarm = 0;
    for (int i = 0; i < q.nHarmonicDifferences && q.harmonicDifferencesLog; i++) {
      const char *t = q.harmonicDifferences[i];
      const char *dash = strchr(t, '-');
      if (!dash || dash == t) { err = std::string("cHarmonics: cannot parse harmonic difference '") + t + "'"; return OSM_B200_ERR_INVALID; }
      int part[2][2];                                            // {formant, idx}
      const char *ps[2] = {t, dash + 1};
      for (int k = 0; k < 2; k++) {
        char *ep = nullptr;
        const long r = strtol(ps[k] + 1, &ep, 10);
        if (ep == ps[k] + 1 || (ps[k][0] != 'H' && ps[k][0] != 'A')) { err = std::string("cHarmonics: cannot parse harmonic difference '") + t + "'"; return OSM_B200_ERR_INVALID; }
        if (ps[k][0] == 'H') { part[k][0] = -1; part[k][1] = (int)r; if (r > maxHarm) maxHarm = (int)r; }
        else if (r == 0) { part[k][0] = -1; part[k][1] = 0; }
        else { part[k][0] = (int)r; part[k][1] = -1; haveFormantDiff = true; }
      }
      ho.diffs.insert(ho.diffs.end(), {part[0][0], part[0][1], part[1][0], part[1][1]});
    }
    if (haveFormantDiff && ho.nFmt == 0) ho.diffs.clear();       // :296-300: disabled without a formant level
    ho.nHarm = q.nHarmonics;
    if (ho.nHarm < q.nHarmonicMagnitudes + q.firstHarmonicMagnitude + 1) ho.nHarm = q.nHarmonicMagnitudes + q.firstHarmonicMagnitude + 1;   // :212-217
    if (ho.nHarm < maxHarm + 1) ho.nHarm = maxHarm + 1;
    if (ho.nHarm < 2 || ho.nHarm > 128) { err = "cHarmonics.nHarmonics must be in 2..128"; return OSM_B200_ERR_UNSUPPORTED; }
    ho.hnr = q.computeAcfHnrLogdB != 0;
    ho.fa = fa;
    if (fa) {                                                    // :341-352
      ho.faStart = q.formantAmplitudesStart < 0 ? 0 : q.formantAmplitudesStart;
      ho.faEnd = q.formantAmplitudesEnd == -1 ? ho.nFmt : std::min(q.formantAmplitudesEnd, ho.nFmt);
      if (ho.faEnd < ho.faStart) ho.fa = false;
      else if (ho.faStart < 1) { err = "cHarmonics.formantAmplitudesStart=0 is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    ho.floorUnvoiced = (float)q.logRelValueFloorUnvoiced;
    ho.nb = fe.nBins;
    ho.binHz = 1.0 / fe.fftFrameSizeSec;                         // dspcore/transformFft.cpp:111-115
    op.kind = SOP_HARMONICS;
    if (ho.hnr) add_field(op, "HarmonicsToNoiseRatioACFLogdB");   // :236-240
    for (size_t i = 0; i < ho.diffs.size() / 4; i++) add_field(op, std::string("HarmonicDifferenceLogRel") + q.harmonicDifferences[i]);
    if (ho.fa) add_field(op, "FormantAmplitudeByMaxHarmonicLogRelF0", ho.faEnd - ho.faStart + 1, ho.faStart);
    ho.nOut = field_elements(op);
    if (ho.nOut < 1) { err = "cHarmonics produces no output"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // [cValbasedSelector <-] cPitchSmootherViterbi <- cPitchShs <- cSpecScale <- cFFTmagphase chain; c = the cPitchShs itself makes the
  // op write the cPitchShs level (no Viterbi stage)
  osm_b200_status build_pitch_chain_op(const osm_b200_component *c, StaticOp &op)
  {
    const osm_b200_component *vit = c, *selSrc = nullptr;
    if (c->type == OSM_B200_C_PITCHSHS) vit = nullptr;
    if (c->type == OSM_B200_C_VALBASEDSELECTOR) {
      const auto &q = c->u.valbasedselector;
      if (c->n_inputs != 2) { err = "cValbasedSelector must read two levels: selector;data"; return OSM_B200_ERR_UNSUPPORTED; }
      if (q.idx != 0 || !q.removeIdx || !q.zeroVec || q.adaptiveThreshold) { err = "cValbasedSelector: only idx=0, removeIdx=1, zeroVec=1, adaptiveThreshold=0 are supported"; return OSM_B200_ERR_UNSUPPORTED; }
      selSrc = R.prod(c->reader_dmLevel[0]);
      vit = R.prod(c->reader_dmLevel[1]);
      if (!selSrc || !vit || vit->type != OSM_B200_C_PITCHSMOOTHERVITERBI) { err = "cValbasedSelector: the data level must come from cPitchSmootherViterbi"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    const osm_b200_component *shs = vit ? single_input(vit) : c;
    if (!shs || shs->type != OSM_B200_C_PITCHSHS) { err = "cPitchSmootherViterbi must read a cPitchShs level"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *scl = single_input(shs);
    if (!scl || scl->type != OSM_B200_C_SPECSCALE) { err = "cPitchShs must read a cSpecScale level"; return OSM_B200_ERR_UNSUPPORTED; }
    ChainInfo ci;
    if (!resolve_mag_chain(single_input(scl), ci)) return OSM_B200_ERR_UNSUPPORTED;
    int selOp = -1;
    if (selSrc) {
      osm_b200_status s3 = get_op(selSrc, selOp);                   // e.g. cEnergy (rms) on the same frames
      if (s3 != OSM_B200_OK) return s3;
      if (d.ops[selOp].nOut != 1) { err = "cValbasedSelector: the selector level must hold exactly one element"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    osm_b200_status s2 = get_stream(ci, true, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    const FrontEnd &fe = d.streams[op.stream].fe;
    if (selOp >= 0 && !same_geometry(d.streams[d.ops[selOp].stream].fe, fe)) { err = "cValbasedSelector: selector and data levels must share the frame geometry"; return OSM_B200_ERR_UNSUPPORTED; }
    op.kind = SOP_PITCH;
    if (!build_pitch_chain(scl->u.specscale, shs->u.pitchshs, vit ? &vit->u.pitchsmootherviterbi : nullptr, fe.nBins, fe.fftFrameSizeSec,
                           op.chain, err))
      return OSM_B200_ERR_UNSUPPORTED;
    PitchChainOp &pc = op.chain;
    if (pc.shsOnly) {                                                 // lldcore/pitchBase.cpp:132-154
      add_field(op, "nCandidates");
      add_field(op, "F0Cand", pc.nCand);
      if (pc.voicing) add_field(op, "candVoicing", pc.nCand);
      if (pc.scores) add_field(op, "candScores", pc.nCand);
      const std::pair<bool, const char *> single[] = {{pc.F0C1, "F0C1"}, {pc.voicingC1, "voicingC1"}, {pc.F0raw, "F0raw"}, {pc.voicingClip, "voicingClip"}};
      for (const auto &o : single) if (o.first) add_field(op, o.second);
      if (field_elements(op) != pc.nShsCols) { err = "internal: cPitchShs name/element mismatch"; return OSM_B200_ERR_INVALID; }
      return OSM_B200_OK;
    }
    if (selOp >= 0) {
      const auto &q = c->u.valbasedselector;
      pc.hasSel = true; pc.selOp = selOp; pc.selThreshold = (float)q.threshold; pc.selOutputVal = (float)q.outputVal;
      pc.selInvert = q.invert != 0; pc.selAllowEqual = q.allowEqual != 0;
    }
    // field names: lld/pitchSmootherViterbi.cpp:297-316; the selector keeps them (valbasedSelector.cpp:105-118)
    const std::pair<bool, const char *> outputs[] = {
      {pc.oF0final, "F0final"}, {pc.oF0finalLog, "F0finalLog"}, {pc.oF0finalEnv, "F0finEnv"}, {pc.oF0finalEnvLog, "F0finEnvLog"},
      {pc.oVClipped, "voicingFinalClipped"}, {pc.oVUnclipped, "voicingFinalUnclipped"}};
    for (const auto &o : outputs)
      if (o.first) add_field(op, c->type == OSM_B200_C_VALBASEDSELECTOR ? name_append_auto(*c, o.second, nullptr) : std::string(o.second));
    if (field_elements(op) != pc.nOut) { err = "internal: cPitchSmootherViterbi name/element mismatch"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  osm_b200_status build_jitter_op(const osm_b200_component *c, StaticOp &op)
  {
    const auto &q = c->u.pitchjitter;
    const osm_b200_component *wv = single_input(c);
    if (!wv || wv->type != OSM_B200_C_WAVESOURCE) { err = "cPitchJitter must read the cWaveSource level"; return OSM_B200_ERR_UNSUPPORTED; }
    const osm_b200_component *f0c = R.prod(q.F0reader_dmLevel);
    if (!f0c) { err = "cPitchJitter: F0reader.dmLevel has no writer"; return OSM_B200_ERR_INVALID; }
    int pOp = -1;
    osm_b200_status s2 = get_op(f0c, pOp);
    if (s2 != OSM_B200_OK) return s2;
    if (d.ops[pOp].kind != SOP_PITCH || d.ops[pOp].chain.shsOnly) { err = "cPitchJitter: the F0 level must come from cPitchSmootherViterbi (optionally through cValbasedSelector)"; return OSM_B200_ERR_UNSUPPORTED; }
    op.kind = SOP_JITTER;
    op.stream = d.ops[pOp].stream;
    JitterOp &jo = op.jitter;
    jo.pitchOp = pOp;
    int col = 0;                                                        // lld/pitchJitter.cpp:271-280: unknown field -> element 0
    jo.f0Col = find_field(d.ops[pOp], name_match(q.F0field, true), col) ? col : 0;
    jo.searchRangeRel = q.searchRangeRel; jo.lgHNRfloor = q.lgHNRfloor;
    jo.minNumPeriods = q.minNumPeriods < 2 ? 2 : q.minNumPeriods;      // :145-149
    jo.minCC = q.minCC;
    jo.jitterLocal = q.jitterLocal != 0; jo.jitterDDP = q.jitterDDP != 0; jo.jitterLocalEnv = q.jitterLocalEnv != 0; jo.jitterDDPEnv = q.jitterDDPEnv != 0;
    jo.shimmerLocal = q.shimmerLocal != 0; jo.shimmerLocalDB = q.shimmerLocalDB != 0; jo.shimmerLocalEnv = q.shimmerLocalEnv != 0;
    jo.shimmerLocalDBEnv = q.shimmerLocalDBEnv != 0; jo.harmonicERMS = q.harmonicERMS != 0; jo.noiseERMS = q.noiseERMS != 0;
    jo.linearHNR = q.linearHNR != 0; jo.logHNR = q.logHNR != 0; jo.shimmerUseRms = q.shimmerUseRmsAmplitude != 0;
    jo.refinedF0 = q.refinedF0 != 0; jo.srcQualRange = q.sourceQualityRange != 0; jo.srcQualMean = q.sourceQualityMean != 0;
    jo.peakToPeak = q.usePeakToPeakPeriodLength != 0; jo.brokenThresh = q.useBrokenJitterThresh != 0;
    if (q.onlyVoiced) { err = "cPitchJitter.onlyVoiced=1 (variable frame count) is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    if (wv->u.wavesource.nChannels > 1 && !wv->u.wavesource.monoMixdown) { err = "cPitchJitter needs mono input"; return OSM_B200_ERR_UNSUPPORTED; }
    const std::pair<bool, const char *> outputs[] = {                   // :283-312
      {jo.jitterLocal, "jitterLocal"}, {jo.jitterDDP, "jitterDDP"}, {jo.jitterLocalEnv, "jitterLocEnv"}, {jo.jitterDDPEnv, "jitterDEnv"},
      {jo.shimmerLocal, "shimmerLocal"}, {jo.shimmerLocalDB, "shimmerLocalDB"}, {jo.shimmerLocalEnv, "shimmerLocEnv"},
      {jo.shimmerLocalDBEnv, "shimmerLocDBEnv"}, {jo.harmonicERMS, "harmonicERMS"}, {jo.noiseERMS, "noiseERMS"}, {jo.linearHNR, "linearHNR"},
      {jo.logHNR, "logHNR"}, {jo.refinedF0, q.F0field[0] ? q.F0field : "F0final"}, {jo.srcQualMean, "sourceQualityMean"},
      {jo.srcQualRange, "sourceQualityRange"}};
    for (const auto &o : outputs) if (o.first) add_field(op, o.second);
    jo.nOut = (int)op.fields.size();
    if (jo.nOut < 1) { err = "cPitchJitter produces no output"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // cTonespec on a plain cFFTmagphase magnitude level, or cChroma on such a cTonespec level (config/chroma/chroma_fft.conf): one
  // band op of the FFT stream.  Both are cVectorProcessors that keep the frame count of the level they read.
  osm_b200_status build_tone_op(const osm_b200_component *c, StaticOp &op)
  {
    const osm_b200_component *ts = c;
    if (c->type == OSM_B200_C_CHROMA) {
      ts = single_input(c);
      if (ts && ts->type == OSM_B200_C_TONEFILT) return build_tonefilt_op(c, op);
      if (!ts || ts->type != OSM_B200_C_TONESPEC) { err = "cChroma must read a cTonespec level (or a cTonefilt level)"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    ChainInfo ci;
    if (!resolve_mag_chain(single_input(ts), ci)) { err = "cTonespec: " + err; return OSM_B200_ERR_UNSUPPORTED; }
    osm_b200_status s2 = get_stream(ci, true, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    const FrontEnd &fe = d.streams[op.stream].fe;
    op.kind = SOP_TONE;
    ToneOp &to = op.tone;
    if (!build_tone(ts->u.tonespec, fe.nBins, fe.fftFrameSizeSec, to, err)) return OSM_B200_ERR_UNSUPPORTED;
    // the field is "tone" with nNotes elements, whatever the input field is called (lld/tonespec.cpp:370-377)
    const std::string toneName = name_append_auto(*ts, "tone", nullptr);
    if (c->type == OSM_B200_C_TONESPEC) {
      add_field(op, toneName, to.nNotes);
      return OSM_B200_OK;
    }
    const auto &q = c->u.chroma;
    // lld/chroma.cpp:94-115: with nNotes not a multiple of octaveSize the reference logs an error and writes rows it never set
    if (q.octaveSize < 1 || to.nNotes % q.octaveSize != 0) {
      err = "cChroma.octaveSize must divide the number of cTonespec notes (12 * nOctaves)"; return OSM_B200_ERR_UNSUPPORTED;
    }
    to.octaveSize = q.octaveSize;
    to.silThresh = (float)q.silThresh;                                                     // :71
    to.nOut = q.octaveSize;
    add_field(op, name_append_auto(*c, toneName, nullptr), q.octaveSize);                 // :78-81
    return OSM_B200_OK;
  }

  // cTonefilt on the wave level, or cChroma on such a cTonefilt level (config/chroma/chroma_filt.conf): a stream of its own whose
  // rows are blocks of P samples (tonefilt.cu)
  osm_b200_status build_tonefilt_op(const osm_b200_component *c, StaticOp &op)
  {
    const osm_b200_component *tfc = c->type == OSM_B200_C_CHROMA ? single_input(c) : c;
    const osm_b200_component *wv = single_input(tfc);
    if (!wv || wv->type != OSM_B200_C_WAVESOURCE) {
      err = "cTonefilt must read the cWaveSource level (on a frame level it would filter every element as a signal of its own)";
      return OSM_B200_ERR_UNSUPPORTED;
    }
    const auto &wp = wv->u.wavesource;
    if (wp.nChannels > 1 && !wp.monoMixdown) { err = "cTonefilt: a multi-element wave level (monoMixdown = 0) is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    if (wp.sampleRate <= 0) { err = "cWaveSource: bad sampleRate/nChannels"; return OSM_B200_ERR_INVALID; }
    op.kind = SOP_TONEFILT;
    TonefiltOp &to = op.tonefilt;
    if (!build_tonefilt(tfc->u.tonefilt, wp.sampleRate, to, err)) return OSM_B200_ERR_UNSUPPORTED;
    osm_b200_status s2 = get_tonefilt_stream(wv, tfc, to, op.stream);
    if (s2 != OSM_B200_OK) return s2;
    // <input field>_<nameAppend> with nNotes elements; copyInputName plays no part (lld/tonefilt.cpp:137-172)
    const std::string na = tfc->nameAppend[0] ? tfc->nameAppend : default_name_append(OSM_B200_C_TONEFILT);
    const std::string tfName = wave_name(ChainInfo{wv}) + "_" + na;
    if (c->type == OSM_B200_C_TONEFILT) {
      add_field(op, tfName, to.nNotes);
      return OSM_B200_OK;
    }
    if (to.nNotes == 1) {                                              // core/vectorProcessor.cpp:196-243
      err = "cChroma on a one-note cTonefilt level: the reference's cChroma (processArrayFields = 1) finds no array field there"; return OSM_B200_ERR_UNSUPPORTED;
    }
    const auto &q = c->u.chroma;
    if (q.octaveSize < 1 || to.nNotes % q.octaveSize != 0) {           // lld/chroma.cpp:94-115
      err = "cChroma.octaveSize must divide the number of cTonefilt notes (nNotes)"; return OSM_B200_ERR_UNSUPPORTED;
    }
    to.octaveSize = q.octaveSize;
    to.silThresh = (float)q.silThresh;                                 // :71
    add_field(op, name_append_auto(*c, tfName, nullptr), q.octaveSize); // :78-81
    return OSM_B200_OK;
  }

  // the stream of a cTonefilt level: the wave format of the source, rows = blocks of P samples with hop P, period outputPeriod
  // (lld/tonefilt.cpp:101-134).  The row rule of desc_num_static_frames gives ceil(L / P) with frameSize 1 and frameStep P.
  osm_b200_status get_tonefilt_stream(const osm_b200_component *wv, const osm_b200_component *tfc, const TonefiltOp &to, int &idx)
  {
    for (size_t s = 0; s < d.streams.size(); s++)
      if (d.streams[s].keyFramer == tfc) { idx = (int)s; return OSM_B200_OK; }
    const auto &wp = wv->u.wavesource;
    if (wp.format < OSM_B200_PCM_S16 || wp.format > OSM_B200_PCM_S32) { err = "cWaveSource: unknown sample format"; return OSM_B200_ERR_INVALID; }
    Stream st;
    FrontEnd &fe = st.fe;
    fe.sampleRate = wp.sampleRate; fe.nChan = wp.nChannels; fe.format = wp.format; fe.mixdown = true;
    fe.frameSize = 1; fe.frameStep = to.P;
    fe.frameSizeSec = to.period; fe.frameStepSec = to.period;
    fe.rowSampleStep = to.P;
    st.keyFramer = tfc;
    d.streams.push_back(st);
    idx = (int)d.streams.size() - 1;
    return OSM_B200_OK;
  }

  // ---- cValbasedSelector gates: the selector value must be one column of the SHS pitch level (directly, or through a cDataSelector
  // that picks it: GeMAPSv01b_core.lld.conf.inc:385-391) ----
  osm_b200_status resolve_gates()
  {
    for (const GateScope &gs : gateScopes) {
      const osm_b200_component *sl = R.prod(gs.c->reader_dmLevel[0]);
      if (!sl) { err = std::string("level '") + gs.c->reader_dmLevel[0] + "' has no writer"; return OSM_B200_ERR_INVALID; }
      const char *want = nullptr;
      if (sl->type == OSM_B200_C_DATASELECTOR) {
        if (sl->u.dataselector.nSelected != 1 || sl->n_inputs != 1 || !sl->u.dataselector.elementMode) { err = "cValbasedSelector: a cDataSelector selector level must pick exactly one element of one level"; return OSM_B200_ERR_UNSUPPORTED; }
        want = sl->u.dataselector.selected[0];
        sl = R.prod(sl->reader_dmLevel[0]);
        if (!sl) { err = "cValbasedSelector: the selector level has no writer"; return OSM_B200_ERR_INVALID; }
      }
      int so = -1;
      osm_b200_status s3 = get_op(sl, so);
      if (s3 != OSM_B200_OK) return s3;
      const StaticOp &po = d.ops[so];
      if (po.kind != SOP_PITCH || po.chain.shsOnly) { err = "cValbasedSelector: the selector level must come from the SHS pitch chain (cPitchSmootherViterbi)"; return OSM_B200_ERR_UNSUPPORTED; }
      int col = 0;
      if (!find_field(po, [&](const FieldName &f) { return f.n == 1 && (want ? f.name == want : po.nOut == 1); }, col)) {
        err = want ? std::string("cValbasedSelector: selector element '") + want + "' not found in the pitch level" : std::string("cValbasedSelector: the selector level must hold exactly one element"); return OSM_B200_ERR_UNSUPPORTED;
      }
      gateInfo.push_back(GateInfo{po.outCol + col, so});
    }
    return OSM_B200_OK;
  }

  osm_b200_status lower_leaves()
  {
    for (size_t l = 0; l < leaves.size(); l++) {
      osm_b200_status s = lower_leaf(l);
      if (s != OSM_B200_OK) return s;
    }
    if (d.ops.empty() || d.groups.empty()) { err = "the output level has no elements (cVectorConcat drops single-element fields unless includeSingleElementFields=1)"; return OSM_B200_ERR_INVALID; }
    return OSM_B200_OK;
  }

  // ---- groups of leaf l: one per run of consecutive fields that survive the concat's field selection ----
  osm_b200_status lower_leaf(size_t l)
  {
    const Leaf &leaf = leaves[l];
    const std::vector<const osm_b200_component *> &stageComps = leaf.stages;
    int opIdx = -1;
    osm_b200_status so = get_op(leaf.c, opIdx);
    if (so != OSM_B200_OK) return so;
    std::vector<Stage> stages;
    std::vector<FieldName> fields = d.ops[opIdx].fields;
    int segId = -1;
    long gateIdx = -1;
    for (size_t q = 0; q < gateScopes.size(); q++) if (l >= gateScopes[q].l0 && l < gateScopes[q].l1) gateIdx = (long)q;
    if (gateIdx >= 0) for (auto &f : fields) f.name = name_append_auto(*gateScopes[gateIdx].c, f.name, nullptr);   // other/valbasedSelector.cpp:84-97
    long selAbove = -1;                                  // stages above the selector this leaf sits below, -1 = none
    for (const SelScope &sc : selScopes) if (l >= sc.l0 && l < sc.l1) selAbove = (long)sc.above;
    leafSelNames.push_back({});
    auto note_selector_names = [&]() {
      leafSelNames.back().clear();
      for (const FieldName &f : fields) append_element_names(f, leafSelNames.back());
    };
    if (selAbove >= 0 && (long)stageComps.size() == selAbove) note_selector_names();
    size_t stageNo = 0;
    for (const osm_b200_component *s : stageComps) {
      Stage st;
      osm_b200_status s2 = make_stage(s, s == stageComps.back(), st, segId);
      if (s2 != OSM_B200_OK) return s2;
      stages.push_back(st);
      for (auto &f : fields) f.name = name_append_auto(*s, f.name, nullptr);
      stageNo++;
      if (selAbove >= 0 && (long)(stageComps.size() - stageNo) == selAbove) note_selector_names();
    }
    if (stages.size() > 3) { err = "more than 3 chained temporal stages"; return OSM_B200_ERR_UNSUPPORTED; }
    const StaticOp &op = d.ops[opIdx];
    // the level period: a cCens level's is its input's times downsampleRatio, and the levels behind it inherit it
    const int ratio = op.kind == SOP_CENS ? op.cens.ratio : 1;
    if (l > 0 && ratio != d.periodScale) {
      err = "levels of different periods (a cCens level with downsampleRatio > 1 next to other levels) in one output level are not supported";
      return OSM_B200_ERR_UNSUPPORTED;
    }
    d.periodScale = ratio;
    const size_t firstGroup = d.groups.size();
    int col = op.outCol;
    bool open = false;
    for (const auto &f : fields) {
      const bool keep = !(leaf.arraysOnly && f.n == 1);
      if (keep) {
        if (!open) {
          OutGroup g;
          g.srcCol = col; g.n = 0; g.stream = op.stream; g.outCol = d.nOut; g.stages = stages;
          if (op.kind == SOP_PITCH && !op.chain.shsOnly) { g.lagKind = 1; g.lagOp = opIdx; }   // the cPitchShs level does not lag
          if (op.kind == SOP_JITTER) { g.lagKind = 2; g.lagOp = op.jitter.pitchOp; }
          if (op.kind == SOP_HARMONICS) { g.lagKind = 1; g.lagOp = op.harmonics.pitchOp; }
          if (gateIdx >= 0) {
            const auto &q = gateScopes[gateIdx].c->u.valbasedselector;
            g.gateCol = gateInfo[gateIdx].col;
            g.gateThreshold = (float)q.threshold; g.gateOutVal = (float)q.outputVal;
            g.gateInvert = q.invert != 0; g.gateAllowEqual = q.allowEqual != 0;
            // the gate reads the pitch level: its output ends where that level ends (truncating reader) and lags with it
            if (g.lagKind == 0) g.lagKind = 1;
            if (g.lagOp >= 0 && g.lagOp != gateInfo[gateIdx].pitchOp) { err = "cValbasedSelector: data behind another pitch chain than the selector's"; return OSM_B200_ERR_UNSUPPORTED; }
            g.lagOp = gateInfo[gateIdx].pitchOp;
          }
          g.segId = segId;
          d.groups.push_back(g);
          open = true;
        }
        d.groups.back().n += f.n;
        d.nOut += f.n;
        append_element_names(f, d.names);
      } else {
        open = false;
      }
      col += f.n;
    }
    leafGroups.push_back({firstGroup, d.groups.size()});
    return OSM_B200_OK;
  }

  // the temporal stage of component s; last = s is the stage nearest the output level
  osm_b200_status make_stage(const osm_b200_component *s, bool last, Stage &st, int &segId)
  {
    if (s->type == OSM_B200_C_DELTAREGRESSION) {
      const auto &p = s->u.deltaregression;
      if (p.deltawin < 1 || p.deltawin > 8) { err = "cDeltaRegression.deltawin must be 1..8"; return OSM_B200_ERR_UNSUPPORTED; }
      // flags: bit 0 onlyInSegments, bit 1 relativeDelta, bit 2 absOutput, bit 3 halfWaveRect (dspcore/deltaRegression.cpp:100-168;
      // halfWaveRect wins over absOutput, :157-165)
      const int variant = (p.relativeDelta ? 2 : 0) | (p.halfWaveRect ? 8 : (p.absOutput ? 4 : 0));
      if (variant && p.onlyInSegments) { err = "cDeltaRegression: relativeDelta / absOutput / halfWaveRect together with onlyInSegments are not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      st = Stage{ST_DELTA, p.deltawin, (p.onlyInSegments ? 1 : 0) | variant};
      if (p.onlyInSegments) {
        segId = -1;
        for (size_t q = 0; q < segComps.size(); q++) if (segComps[q] == s) segId = (int)q;
        if (segId < 0) { segComps.push_back(s); segId = (int)segComps.size() - 1; }
      }
    } else if (s->type == OSM_B200_C_FULLINPUTMEAN) {
      // dspcore/fullinputMean.cpp:484-548 (single EOI loop): all frames are read before EOI, the
      // arithmetic mean is subtracted from every frame at EOI -> same number of frames, and the
      // level is complete only after EOI, so nothing may be chained behind it here
      const auto &p = s->u.fullinputmean;
      if (p.mvn || p.meanNorm != 0 || p.symmSubtract || p.subtractClipToZero || p.specEnorm || p.htkLogEnorm || p.excludeZeros || p.multiLoopMode) {
        err = "cFullinputMean: only plain arithmetic mean subtraction (the defaults) is supported"; return OSM_B200_ERR_UNSUPPORTED;
      }
      if (!last) { err = "a temporal stage reading a cFullinputMean level is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      st = Stage{ST_CMS, 0, 0};
    } else {
      const auto &p = s->u.contoursmoother;
      if (p.smaWin < 1 || (p.smaWin & 1) == 0 || p.smaWin > 9) { err = "cContourSmoother.smaWin must be odd, 1..9"; return OSM_B200_ERR_UNSUPPORTED; }
      st = Stage{ST_SMA, (p.smaWin - 1) / 2, p.noZeroSma};
    }
    return OSM_B200_OK;
  }

  // A concat (or multi-level reader) below temporal stages delivers min over its inputs
  // (core/dataReader.cpp:375-380).  Inputs of different frame geometry are supported when they are
  // static levels (no stage below the concat): every group then carries the other streams as limits.
  osm_b200_status apply_concat_limits()
  {
    for (const ConcatCheck &cc : concatChecks) {
      std::vector<int> streams;
      int w0 = -1;
      bool sameW = true;
      for (size_t l = cc.g0; l < cc.g1; l++)
        for (size_t g = leafGroups[l].first; g < leafGroups[l].second; g++) {
          int w = 0;
          for (const auto &st : d.groups[g].stages) w += st.win;
          if (w0 < 0) w0 = w;
          if (w != w0) sameW = false;
          const FrontEnd &fe = d.streams[d.groups[g].stream].fe;
          bool known = false;
          for (int sidx : streams) known = known || same_geometry(d.streams[sidx].fe, fe);
          if (!known) streams.push_back(d.groups[g].stream);
        }
      if (streams.size() <= 1 && sameW) continue;          // nothing truncates
      bool ok = sameW;
      // the stages every leaf carries must all sit above the concat (i.e. the leaves are statics)
      for (size_t l = cc.g0; l < cc.g1 && ok; l++) ok = leaves[l].stages.size() == cc.above;
      if (!ok) { err = "cVectorConcat of unequally long, already smoothed levels below a temporal stage is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      if (streams.size() > 4) { err = "more than 4 frame geometries below one cVectorConcat"; return OSM_B200_ERR_UNSUPPORTED; }
      for (size_t l = cc.g0; l < cc.g1; l++)
        for (size_t g = leafGroups[l].first; g < leafGroups[l].second; g++)
          for (int sidx : streams) {
            if (same_geometry(d.streams[sidx].fe, d.streams[d.groups[g].stream].fe)) continue;
            if (std::find(d.groups[g].limitStreams.begin(), d.groups[g].limitStreams.end(), sidx) == d.groups[g].limitStreams.end())
              d.groups[g].limitStreams.push_back(sidx);
          }
    }
    return OSM_B200_OK;
  }

  // ---- cDataSelector scopes: replace the groups of the leaves below a selector by the selected elements ----
  osm_b200_status apply_selector_scopes()
  {
    if (selScopes.empty()) return OSM_B200_OK;
    std::vector<OutGroup> ng;
    std::vector<std::string> nn;
    int outCol = 0;
    for (size_t l = 0; l < leaves.size();) {
      const SelScope *sc = nullptr;
      for (const SelScope &x : selScopes) if (x.l0 == l) sc = &x;
      if (!sc) {
        for (size_t g = leafGroups[l].first; g < leafGroups[l].second; g++) {
          OutGroup x = d.groups[g];
          for (int i = 0; i < x.n; i++) nn.push_back(d.names[x.outCol + i]);
          x.outCol = outCol; outCol += x.n;
          ng.push_back(x);
        }
        l++;
        continue;
      }
      struct El { size_t g; int off; const std::string *name; };
      std::vector<El> els;                                // the elements of the selector's input, in reader order
      for (size_t ll = sc->l0; ll < sc->l1; ll++) {
        size_t e = 0;
        for (size_t g = leafGroups[ll].first; g < leafGroups[ll].second; g++)
          for (int i = 0; i < d.groups[g].n; i++, e++) {
            if (e >= leafSelNames[ll].size()) { err = "internal: cDataSelector element bookkeeping"; return OSM_B200_ERR_INVALID; }
            els.push_back(El{g, i, &leafSelNames[ll][e]});
          }
      }
      const auto &q = sc->c->u.dataselector;
      const std::vector<const osm_b200_component *> &lst = leaves[sc->l0].stages;
      // A selector that reads a cPitchJitter level waits for it: during the reference's first end-of-input pass that
      // level does not advance (lld/pitchJitter.cpp:593), so EVERY element of the selector's output lags like the jitter
      // columns do (oracle/formant_oracle.py:gemaps_lld, pinned on the shipped GeMAPS configurations)
      bool scopeLags = false;
      int scopeLagOp = -1;
      for (const El &e : els) if (d.groups[e.g].lagKind == 2) { scopeLags = true; scopeLagOp = d.groups[e.g].lagOp; }
      if (scopeLags)
        for (size_t ll = sc->l0; ll < sc->l1; ll++)
          if (leaves[ll].stages.size() != sc->above) {
            // pinned only for a selector directly on the per-frame levels (the shipped graphs); a selector over levels
            // that were smoothed first sees another tick order
            err = "cDataSelector reading a cPitchJitter level: temporal stages below the selector are not supported"; return OSM_B200_ERR_UNSUPPORTED;
          }
      long prevG = -1;
      for (int k = 0; k < q.nSelected; k++) {
        for (int k2 = 0; k2 < k; k2++)
          if (!strcmp(q.selected[k], q.selected[k2])) { err = std::string("cDataSelector: element selected twice: ") + q.selected[k]; return OSM_B200_ERR_UNSUPPORTED; }
        const El *hit = nullptr;
        for (const El &e : els) if (*e.name == q.selected[k]) { hit = &e; break; }
        if (!hit) {                                       // core/dataSelector.cpp:330-343 aborts as well
          err = std::string("cDataSelector '") + sc->c->name + "': element '" + q.selected[k] + "' not found in its input levels";
          return OSM_B200_ERR_INVALID;
        }
        OutGroup x = d.groups[hit->g];
        x.srcCol += hit->off; x.n = 1; x.outCol = outCol++;
        if (scopeLags) {
          // every input level of a lagging selector must deliver at least the rows of the pitch level: the selector's output
          // then has the pitch level's length and the limits of the truncating reader are redundant.  A per-frame level
          // routed through it (e.g. the formants of the 20 ms frames) lags like the rest.
          if (!group_delivers_rows_of(x, d.streams[d.ops[scopeLagOp].stream].fe)) {
            err = "cDataSelector reading a cPitchJitter level together with a level of another frame step / longer frames is not supported"; return OSM_B200_ERR_UNSUPPORTED;
          }
          x.limitStreams.clear();
          x.lagKind = 2; x.lagOp = scopeLagOp; x.stream = d.ops[scopeLagOp].stream;
        }
        if (prevG == (long)hit->g && !ng.empty() && ng.back().srcCol + ng.back().n == x.srcCol) ng.back().n++;
        else ng.push_back(x);
        prevG = (long)hit->g;
        std::string nm = q.newNames[k][0] ? std::string(q.newNames[k])                                  // :344-356
                         : (sc->c->nameAppend[0] ? std::string(q.selected[k]) + "_" + sc->c->nameAppend : std::string(q.selected[k]));
        for (size_t a = lst.size() - sc->above; a < lst.size(); a++) nm = name_append_auto(*lst[a], nm, nullptr);
        nn.push_back(nm);
      }
      l = sc->l1;
    }
    d.groups.swap(ng);
    d.names.swap(nn);
    d.nOut = outCol;
    return OSM_B200_OK;
  }

  // every stream group g reads (its own and the limits of a truncating reader) delivers at least the rows of ref
  bool group_delivers_rows_of(const OutGroup &g, const FrontEnd &ref) const
  {
    for (int sidx : g.limitStreams) if (!delivers_rows_of(d.streams[sidx].fe, ref)) return false;
    return delivers_rows_of(d.streams[g.stream].fe, ref);
  }

  // ---- gated groups: every data level must deliver at least the rows of the pitch level, the gate's output then has the pitch
  // level's length ----
  osm_b200_status check_gated_groups()
  {
    for (OutGroup &g : d.groups) {
      if (g.gateCol < 0) continue;
      const int ps = d.ops[g.lagOp].stream;
      if (!group_delivers_rows_of(g, d.streams[ps].fe)) { err = "cValbasedSelector: a data level of another frame step / longer frames than the pitch level is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
      g.limitStreams.clear();
      g.stream = ps;
      if (g.stages.empty()) { err = "a cValbasedSelector level as output level (no cContourSmoother behind it) is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    return OSM_B200_OK;
  }

  // ---- groups behind a Viterbi-smoothed pitch level (seq_post_kernel) ----
  // Supported shapes (the ones the shipped feature sets use): [cContourSmoother(3)] and
  // [cContourSmoother(3), cDeltaRegression(onlyInSegments)], no truncating concat in between.
  osm_b200_status check_sequential_groups()
  {
    for (const OutGroup &g : d.groups) {
      const bool seg = g.segId >= 0;
      if (!seg && g.lagKind == 0) continue;
      if (g.lagKind == 0) { err = "cDeltaRegression.onlyInSegments=1 is only supported behind the SHS pitch chain (cPitchSmootherViterbi / cPitchJitter levels)"; return OSM_B200_ERR_UNSUPPORTED; }
      const size_t ns = g.stages.size();
      if (ns == 0 && !seg && g.limitStreams.empty()) continue;   // a static level itself: every frame, nothing lags behind it
      bool ok = ns >= 1 && ns <= 2 && g.stages[0].kind == ST_SMA && g.stages[0].win == 1;
      if (ok && ns == 2) ok = g.stages[1].kind == ST_DELTA && (g.stages[1].flags & 1) && g.stages[1].win >= 1 && g.stages[1].win <= 4;
      if (!ok) { err = "levels behind cPitchSmootherViterbi / cPitchJitter support cContourSmoother(smaWin=3) optionally followed by cDeltaRegression(onlyInSegments=1) only"; return OSM_B200_ERR_UNSUPPORTED; }
      if (!g.limitStreams.empty()) { err = "a truncating concat below the temporal stages of a pitch level is not supported"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    return OSM_B200_OK;
  }

  // ---- execution strategy per stream ----
  // A stream with exactly one band op (MFCC / PLP / tone) and no other spectral consumer evaluates it
  // inside lld_kernel; any other spectral consumer reads the magnitude level from HBM.
  osm_b200_status choose_execution()
  {
    for (size_t s = 0; s < d.streams.size(); s++) {
      int nSpec = 0;
      d.streams[s].bandOps.clear();
      for (size_t o = 0; o < d.ops.size(); o++) {
        if (d.ops[o].stream != (int)s) continue;
        if (d.ops[o].kind == SOP_MFCC || d.ops[o].kind == SOP_PLP || d.ops[o].kind == SOP_TONE) d.streams[s].bandOps.push_back((int)o);
        if (d.ops[o].kind == SOP_SPECTRAL || d.ops[o].kind == SOP_PITCHACF || d.ops[o].kind == SOP_MAG || d.ops[o].kind == SOP_PITCH || d.ops[o].kind == SOP_HARMONICS) nSpec++;
      }
      const int nBand = (int)d.streams[s].bandOps.size();
      d.streams[s].fusedOp = nBand ? d.streams[s].bandOps[0] : -1;
      d.streams[s].dumpMag = nSpec > 0;
      if ((nBand || nSpec) && (d.streams[s].fe.nfft < 64 || d.streams[s].fe.nfft > 4096)) { err = "FFT size out of the supported range"; return OSM_B200_ERR_UNSUPPORTED; }
    }
    return OSM_B200_OK;
  }
};

}  // namespace

osm_b200_status compile_graph(const osm_b200_component *comps, int n, const char *outputLevel,
                              PlanDesc &d, std::string &err)
{
  GraphCompiler g(comps, n, d, err);
  osm_b200_status s = g.index_writers(outputLevel);
  if (s != OSM_B200_OK) return s;
  d = PlanDesc();
  d.padRows = g.R.prod(outputLevel)->type == OSM_B200_C_VECTORCONCAT && strcmp(g.R.prod(outputLevel)->name, "_unionconcat") == 0;
  s = g.expand(outputLevel, {}, 0, false);
  // gate resolution creates the selectors' pitch ops before the leaves are lowered: op indices follow this order
  if (s == OSM_B200_OK) s = g.resolve_gates();
  if (s == OSM_B200_OK) s = g.lower_leaves();
  if (s == OSM_B200_OK) s = g.apply_concat_limits();
  if (s == OSM_B200_OK) s = g.apply_selector_scopes();
  if (s == OSM_B200_OK) s = g.check_gated_groups();
  if (s == OSM_B200_OK) s = g.check_sequential_groups();
  if (s == OSM_B200_OK) s = g.choose_execution();
  return s;
}

}  // namespace osm

// front.cpp -- host front end: openSMILE .conf parsing -> osm_b200_component[] -> plan, WAV in,
// HTK / CSV out (include/osm_b200_host.h).  Pure host C++; all numerics happen in the CUDA plan.
// Citations relative to /root/reference/src.
#include <algorithm>
#include <cmath>
#include <charconv>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <atomic>
#include <map>
#include <mutex>
#include <thread>
#include <set>
#include <sstream>
#include <string>
#include <vector>
#include <memory>

#include "../../include/osm_b200_host.h"
#include "../../include/osm_b200_functionals.h"
#include <cuda_runtime_api.h>
#include "../csrc/cuda_owned.hpp"

namespace {

thread_local std::string g_herr;
osm_b200_status hfail(osm_b200_status s, const std::string &m) { g_herr = m; return s; }

// ------------------------------------------------------------------------------------------
// ini-style config reader (core/configManager.cpp:1632-1645 format, :2180-2300 line rules)
// ------------------------------------------------------------------------------------------
struct Section {
  std::string name, type;
  std::vector<std::pair<std::string, std::string>> kv;   // field -> value, in file order
  const std::string *get(const std::string &k) const
  {
    const std::string *r = nullptr;
    for (const auto &p : kv) if (p.first == k) r = &p.second;    // last assignment wins
    return r;
  }
};

struct Conf {
  std::vector<Section> sections;
  std::vector<std::pair<std::string, std::string>> instances;   // instance name -> type, in order
  std::map<std::string, std::string> cmOpts;                    // declared \cm options -> value
};

std::string trim(const std::string &s)
{
  size_t a = 0, b = s.size();
  while (a < b && (s[a] == ' ' || s[a] == '\t' || s[a] == '\r' || s[a] == '\n')) a++;
  while (b > a && (s[b - 1] == ' ' || s[b - 1] == '\t' || s[b - 1] == '\r' || s[b - 1] == '\n')) b--;
  return s.substr(a, b - a);
}

// an `a;b;c` list (level lists, functionalsEnabled, array fields given in one line): items trimmed, empty items dropped
std::vector<std::string> split_list(const std::string &v)
{
  std::vector<std::string> out;
  std::stringstream ss(v);
  std::string one;
  while (std::getline(ss, one, ';')) { one = trim(one); if (!one.empty()) out.push_back(one); }
  return out;
}

std::string dir_of(const std::string &p)
{
  const size_t i = p.find_last_of('/');
  return i == std::string::npos ? std::string(".") : p.substr(0, i);
}

// \cm[long(short){default}:description] -> value (configManager.cpp:2012-2070).  The first
// occurrence declares the option and its default; later \cm[long] references reuse it.
bool substitute_cm(std::string &value, Conf &cf, const std::map<std::string, std::string> &given, std::string &err)
{
  for (;;) {
    const size_t a = value.find("\\cm[");
    if (a == std::string::npos) return true;
    const size_t b = value.find(']', a);
    if (b == std::string::npos) { err = "unterminated \\cm[...] in '" + value + "'"; return false; }
    std::string body = value.substr(a + 4, b - a - 4);
    const size_t colon = body.find(':');
    if (colon != std::string::npos) body = body.substr(0, colon);
    std::string name = body, dflt;
    bool hasDflt = false;
    const size_t br = body.find('{');
    if (br != std::string::npos) {
      const size_t be = body.find('}', br);
      dflt = body.substr(br + 1, (be == std::string::npos ? body.size() : be) - br - 1);
      hasDflt = true;
      name = body.substr(0, br);
    }
    const size_t par = name.find('(');
    std::string shortName;
    if (par != std::string::npos) {
      const size_t pe = name.find(')', par);
      shortName = name.substr(par + 1, (pe == std::string::npos ? name.size() : pe) - par - 1);
      name = name.substr(0, par);
    }
    name = trim(name);
    std::string v;
    auto g = given.find(name);
    if (g == given.end() && !shortName.empty()) g = given.find(shortName);
    if (g != given.end()) v = g->second;
    else if (cf.cmOpts.count(name)) v = cf.cmOpts[name];
    else if (hasDflt) v = dflt;
    else { err = "command line option '" + name + "' referenced by the config has no value"; return false; }
    cf.cmOpts[name] = v;
    value = value.substr(0, a) + v + value.substr(b + 1);
  }
}

bool parse_file(const std::string &path, Conf &cf, const std::map<std::string, std::string> &given,
                std::string &err, int &cur, int depth = 0)
{
  if (depth > 16) { err = "config includes nested too deeply"; return false; }
  std::ifstream in(path);
  if (!in) { err = "cannot open config file '" + path + "'"; return false; }
  std::stringstream ss;
  ss << in.rdbuf();
  std::string text = ss.str();
  // block comments /* ... */
  for (;;) {
    const size_t a = text.find("/*");
    if (a == std::string::npos) break;
    const size_t b = text.find("*/", a + 2);
    text.erase(a, (b == std::string::npos ? text.size() : b + 2) - a);
  }
  std::istringstream ls(text);
  std::string line;
  int lineNr = 0;
  while (std::getline(ls, line)) {
    lineNr++;
    line = trim(line);
    if (line.empty()) continue;
    if (line[0] == '%' || line[0] == '#' || line[0] == ';' || (line.size() > 1 && line[0] == '/' && line[1] == '/')) continue;
    const size_t cc = line.find("//");                         // EOL comments (configManager.cpp:2226-2232)
    if (cc != std::string::npos) line = trim(line.substr(0, cc));
    if (line.empty()) continue;
    if (line.compare(0, 2, "\\{") == 0) {                       // include (configManager.cpp:1757-1791)
      const size_t e = line.rfind('}');
      std::string inc = trim(line.substr(2, (e == std::string::npos || e < 2 ? line.size() : e) - 2));
      if (!substitute_cm(inc, cf, given, err)) return false;
      std::string full = inc;
      if (!inc.empty() && inc[0] != '/') full = dir_of(path) + "/" + inc;
      // an include inside a section continues that section (e.g. arff_targets.conf.inc)
      if (!parse_file(full, cf, given, err, cur, depth + 1)) {
        std::string err2;
        if (!(inc[0] != '/' && parse_file(inc, cf, given, err2, cur, depth + 1))) return false;   // also relative to cwd
        err.clear();
      }
      continue;
    }
    if (line[0] == '[') {
      const size_t e = line.find(']');
      const std::string head = line.substr(1, (e == std::string::npos ? line.size() : e) - 1);
      const size_t c = head.find(':');
      if (c == std::string::npos) { err = path + ":" + std::to_string(lineNr) + ": section header without ':type'"; return false; }
      cf.sections.push_back(Section{trim(head.substr(0, c)), trim(head.substr(c + 1)), {}});
      cur = (int)cf.sections.size() - 1;
      continue;
    }
    if (cur < 0) { err = path + ":" + std::to_string(lineNr) + ": assignment outside of a section"; return false; }
    const size_t eq = line.find('=');
    if (eq == std::string::npos) { err = path + ":" + std::to_string(lineNr) + ": missing '='"; return false; }
    std::string field = trim(line.substr(0, eq)), value = trim(line.substr(eq + 1));
    Section &sec = cf.sections[cur];
    if (field.compare(0, sec.name.size() + 1, sec.name + ".") == 0) field = field.substr(sec.name.size() + 1);
    if (!substitute_cm(value, cf, given, err)) return false;
    if (sec.type == "cComponentManager") {
      // instance[NAME].type = TYPE (core/componentManager.cpp:840-957)
      if (field.compare(0, 9, "instance[") == 0) {
        const size_t e = field.find(']');
        const std::string nm = field.substr(9, e - 9);
        if (field.find(".type", e) != std::string::npos) cf.instances.push_back({nm, value});
      }
      continue;   // nThreads, printLevelStats, ... : runtime options of the reference's tick loop
    }
    sec.kv.push_back({field, value});
  }
  return true;
}

// ------------------------------------------------------------------------------------------
// component registry: accepted fields per type (the reference's ConfigType schemas, SURVEY.md
// Appendix A).  Unknown fields are an error, like CONF_PARSER_ERR (configManager.cpp:2599).
// ------------------------------------------------------------------------------------------
const char *kCommonFields[] = {"reader.dmLevel", "writer.dmLevel", "reader.dmInstance", "writer.dmInstance",
  "reader.forceAsyncMerge", "reader.errorOnFullInputIncomplete", "nameAppend", "copyInputName", "EOIlevel",
  "processArrayFields", "includeSingleElementFields", "preserveFieldNames", "buffersize", "buffersize_sec",
  "blocksize", "blocksizeR", "blocksizeW", "blocksize_sec", "blocksizeR_sec", "blocksizeW_sec",
  "writer.levelconf.isRb", "writer.levelconf.nT", "writer.levelconf.T", "writer.levelconf.lenSec",
  "writer.levelconf.frameSizeSec", "writer.levelconf.growDyn", "writer.levelconf.noHang", "writer.levelconf.type"};

bool is_common(const std::string &f)
{
  for (const char *c : kCommonFields) if (f == c) return true;
  return false;
}

double num(const std::string &v) { return atof(v.c_str()); }
int inum(const std::string &v) { return (int)lround(atof(v.c_str())); }

int win_func(const std::string &s)
{
  // cWindower::winFuncToInt (dspcore/windower.cpp:60-80): prefix match, case-insensitive
  std::string l;
  for (char c : s) l.push_back((char)tolower(c));
  if (l.compare(0, 3, "han") == 0) return OSM_B200_WIN_HANNING;
  if (l.compare(0, 3, "ham") == 0) return OSM_B200_WIN_HAMMING;
  if (l.compare(0, 3, "rec") == 0) return OSM_B200_WIN_RECTANGLE;
  if (l.compare(0, 3, "gau") == 0) return OSM_B200_WIN_GAUSS;
  if (l.compare(0, 3, "sin") == 0 || l.compare(0, 3, "cos") == 0) return OSM_B200_WIN_SINE;
  if (l.compare(0, 3, "tri") == 0) return OSM_B200_WIN_TRIANGLE;
  if (l.compare(0, 3, "bah") == 0 || l.compare(0, 10, "bartlett-h") == 0) return OSM_B200_WIN_BARTHANN;
  if (l.compare(0, 3, "bar") == 0) return OSM_B200_WIN_BARTLETT;
  if (l.compare(0, 3, "blh") == 0 || l.compare(0, 10, "blackman-h") == 0) return OSM_B200_WIN_BLACKHARR;
  if (l.compare(0, 3, "bla") == 0) return OSM_B200_WIN_BLACKMAN;
  if (l.compare(0, 3, "lac") == 0 || l.compare(0, 3, "lan") == 0) return OSM_B200_WIN_LANCZOS;
  return -1;
}

bool parse_range(const std::string &v, double &lo, double &hi)   // "250-650" (lldcore/spectral.cpp:142-200)
{
  const size_t d = v.find('-', 1);
  if (d == std::string::npos) return false;
  lo = (double)strtol(v.substr(0, d).c_str(), nullptr, 10);
  hi = (double)strtol(v.substr(d + 1).c_str(), nullptr, 10);
  return true;
}

struct TypeInfo { const char *name; int type; };
const TypeInfo kTypes[] = {
  {"cWaveSource", OSM_B200_C_WAVESOURCE}, {"cExternalAudioSource", OSM_B200_C_WAVESOURCE}, {"cFramer", OSM_B200_C_FRAMER},
  {"cVectorPreemphasis", OSM_B200_C_VECTORPREEMPHASIS}, {"cWindower", OSM_B200_C_WINDOWER},
  {"cTransformFFT", OSM_B200_C_TRANSFORMFFT}, {"cFFTmagphase", OSM_B200_C_FFTMAGPHASE}, {"cMelspec", OSM_B200_C_MELSPEC},
  {"cMfcc", OSM_B200_C_MFCC}, {"cPlp", OSM_B200_C_PLP}, {"cSpectral", OSM_B200_C_SPECTRAL}, {"cEnergy", OSM_B200_C_ENERGY},
  {"cMZcr", OSM_B200_C_MZCR}, {"cAcf", OSM_B200_C_ACF}, {"cPitchACF", OSM_B200_C_PITCHACF},
  {"cDeltaRegression", OSM_B200_C_DELTAREGRESSION}, {"cContourSmoother", OSM_B200_C_CONTOURSMOOTHER},
  {"cVectorConcat", OSM_B200_C_VECTORCONCAT}, {"cVectorOperation", OSM_B200_C_VECTOROPERATION},
  {"cFullinputMean", OSM_B200_C_FULLINPUTMEAN}, {"cIntensity", OSM_B200_C_INTENSITY},
  {"cSpecScale", OSM_B200_C_SPECSCALE}, {"cPitchShs", OSM_B200_C_PITCHSHS},
  {"cPitchSmootherViterbi", OSM_B200_C_PITCHSMOOTHERVITERBI}, {"cValbasedSelector", OSM_B200_C_VALBASEDSELECTOR},
  {"cPitchJitter", OSM_B200_C_PITCHJITTER}, {"cSpecResample", OSM_B200_C_SPECRESAMPLE}, {"cLpc", OSM_B200_C_LPC},
  {"cFormantLpc", OSM_B200_C_FORMANTLPC}, {"cDataSelector", OSM_B200_C_DATASELECTOR},
  {"cHarmonics", OSM_B200_C_HARMONICS}, {"cLsp", OSM_B200_C_LSP}, {"cTonespec", OSM_B200_C_TONESPEC}, {"cChroma", OSM_B200_C_CHROMA},
  {"cTonefilt", OSM_B200_C_TONEFILT}, {"cCens", OSM_B200_C_CENS}};

// cTonespec.filterType spellings (lld/tonespec.cpp:107-111); any other value leaves the constructor's Gaussian (:83)
int tone_filter(const std::string &f)
{
  for (const char *s : {"tri", "Tri", "triangular", "Triangular"}) if (f == s) return OSM_B200_TONE_TRI;
  for (const char *s : {"trp", "TrP", "Trp", "triangular-powered", "Triangular-Powered"}) if (f == s) return OSM_B200_TONE_TRP;
  for (const char *s : {"rec", "Rec", "rectangular", "Rectangular"}) if (f == s) return OSM_B200_TONE_REC;
  return OSM_B200_TONE_GAU;
}

int type_of(const std::string &t)
{
  for (const auto &ti : kTypes) if (t == ti.name) return ti.type;
  return -1;
}

#define SETI(field, member) if (f == field) { member = inum(v); continue; }
#define SETD(field, member) if (f == field) { member = num(v); continue; }

// one [name:cType] section -> osm_b200_component
bool to_component(const Section &s, osm_b200_component &c, std::string &err)
{
  const int t = type_of(s.type);
  if (t < 0) { err = "component type '" + s.type + "' (instance '" + s.name + "') is not on the supported LLD path"; return false; }
  if (osm_b200_component_defaults(t, &c) != OSM_B200_OK) { err = osm_b200_last_error(); return false; }
  snprintf(c.name, sizeof c.name, "%s", s.name.c_str());
  bool usePowerSet = false;
  double melFirstNote = 27.5, melLogBase = 2.0;                  // cMelspec defaults (lldcore/melspec.cpp:48-49)
  if (t == OSM_B200_C_VECTOROPERATION) c.u.vectoroperation.operation = -1;   // the reference's default is "norm"
  for (const auto &kv : s.kv) {
    const std::string &f = kv.first, &v = kv.second;
    if (f == "reader.dmLevel") {
      const std::vector<std::string> levels = split_list(v);
      if (levels.size() > OSM_B200_MAX_INPUTS) { err = "too many input levels for '" + s.name + "'"; return false; }
      c.n_inputs = 0;
      for (const std::string &l : levels) snprintf(c.reader_dmLevel[c.n_inputs++], OSM_B200_NAME_LEN, "%s", l.c_str());
      continue;
    }
    if (f == "writer.dmLevel") { snprintf(c.writer_dmLevel, sizeof c.writer_dmLevel, "%s", v.c_str()); continue; }
    if (f == "nameAppend") { snprintf(c.nameAppend, sizeof c.nameAppend, "%s", v.c_str()); continue; }
    if (f == "copyInputName") { c.copyInputName = inum(v); continue; }
    if (t == OSM_B200_C_VECTORCONCAT) {
      SETI("processArrayFields", c.u.vectorconcat.processArrayFields)
      SETI("includeSingleElementFields", c.u.vectorconcat.includeSingleElementFields)
      if (f == "preserveFieldNames") { if (!inum(v)) { err = "cVectorConcat.preserveFieldNames=0 is not supported"; return false; } continue; }
    }
    if (t == OSM_B200_C_LSP && f == "processArrayFields") { c.u.lsp.processArrayFields = inum(v); continue; }
    if (is_common(f)) continue;
    switch (t) {
      case OSM_B200_C_WAVESOURCE:
        SETI("monoMixdown", c.u.wavesource.monoMixdown)
        if (f == "outFieldName") { snprintf(c.u.wavesource.outFieldName, OSM_B200_NAME_LEN, "%s", v.c_str()); continue; }
        // reading a part of the file (iocore/waveSource.cpp:48-58) or header-less PCM changes the samples the graph sees: refused
        // unless left at the defaults (start 0, end -1 = to the end, endrel 0, noHeader 0), never silently ignored
        if (f == "start" || f == "startSamples" || f == "endrel" || f == "endrelSamples") {
          if (num(v) != 0.0) { err = "cWaveSource." + f + " != 0 is not supported (whole files are read)"; return false; }
          continue;
        }
        if (f == "end" || f == "endSamples") {
          if (num(v) >= 0.0) { err = "cWaveSource." + f + " is not supported (whole files are read)"; return false; }
          continue;
        }
        if (f == "noHeader") { if (inum(v)) { err = "cWaveSource.noHeader=1 (raw PCM files) is not supported"; return false; } continue; }
        if (f == "filename" || f == "properTimestamps" || f == "period" || f == "sampleRate" ||
            f == "channels" || f == "nBits" || f == "nBPS" || f == "fieldName") continue;
        break;
      case OSM_B200_C_FRAMER:
        SETD("frameSize", c.u.framer.frameSize) SETD("frameStep", c.u.framer.frameStep)
        SETI("noPostEOIprocessing", c.u.framer.noPostEOIprocessing)
        SETD("frameCenter", c.u.framer.frameCenter)
        if (f == "frameCenterFrames") { c.u.framer.frameCenterFrames = inum(v); c.u.framer.frameCenterFramesSet = 1; continue; }
        if (f == "frameCenterSpecial") {   // core/winToVecProcessor.cpp:461-475: strncasecmp on the first two letters
          std::string k = v.substr(0, 2);
          for (char &ch : k) ch = (char)tolower((unsigned char)ch);
          c.u.framer.frameCenterSpecial = (k == "mi" || k == "ce") ? OSM_B200_CENTER_MID : (k == "ri") ? OSM_B200_CENTER_RIGHT : OSM_B200_CENTER_LEFT;
          continue;
        }
        if (f == "frameMode") { if (v != "fixed") { err = "cFramer.frameMode=" + v + " is not supported"; return false; } continue; }
        if (f == "allowLastFrameIncomplete") { if (inum(v)) { err = "cFramer.allowLastFrameIncomplete=1 is not supported"; return false; } continue; }
        break;
      case OSM_B200_C_VECTORPREEMPHASIS:
        SETD("k", c.u.vectorpreemphasis.k) SETI("de", c.u.vectorpreemphasis.de)
        break;
      case OSM_B200_C_WINDOWER:
        SETD("gain", c.u.windower.gain) SETD("offset", c.u.windower.offset) SETD("sigma", c.u.windower.sigma)
        if (f == "winFunc") { c.u.windower.winFunc = win_func(v); if (c.u.windower.winFunc < 0) { err = "cWindower.winFunc=" + v + " is not supported"; return false; } continue; }
        SETD("fade", c.u.windower.fade) SETI("squareRoot", c.u.windower.squareRoot)
        if (f == "alpha" || f == "alpha0" || f == "alpha1" || f == "alpha2" || f == "alpha3") continue;   // resolved below (they depend on winFunc)
        if (f == "xscale" || f == "xshift") {
          const double d = num(v);
          if (!((f == "xscale" && d == 1.0) || (f == "xshift" && d == 0.0))) { err = "cWindower." + f + " is not supported"; return false; }
          continue;
        }
        break;
      case OSM_B200_C_TRANSFORMFFT:
        SETI("inverse", c.u.transformfft.inverse) SETI("zeroPadSymmetric", c.u.transformfft.zeroPadSymmetric)
        break;
      case OSM_B200_C_FFTMAGPHASE:
        SETI("magnitude", c.u.fftmagphase.magnitude) SETI("phase", c.u.fftmagphase.phase) SETI("normalise", c.u.fftmagphase.normalise)
        SETI("power", c.u.fftmagphase.power) SETI("dBpsd", c.u.fftmagphase.dBpsd)
        if (f == "inverse" || f == "joinMagphase") { if (inum(v)) { err = "cFFTmagphase." + f + " is not supported"; return false; } continue; }
        SETD("dBpnorm", c.u.fftmagphase.dBpnorm) SETD("mindBp", c.u.fftmagphase.mindBp)
        break;
      case OSM_B200_C_MELSPEC:
        SETI("nBands", c.u.melspec.nBands) SETD("lofreq", c.u.melspec.lofreq) SETD("hifreq", c.u.melspec.hifreq)
        SETI("usePower", c.u.melspec.usePower) SETI("htkcompatible", c.u.melspec.htkcompatible)
        if (f == "specScale") {                              // lldcore/melspec.cpp:100-126 (case-insensitive; semi / lin / log by prefix)
          std::string lv = v;
          for (char &ch : lv) ch = (char)tolower((unsigned char)ch);
          if (lv == "mel") c.u.melspec.specScale = OSM_B200_SCALE_MEL;
          else if (lv == "bark") c.u.melspec.specScale = OSM_B200_SCALE_BARK;
          else if (lv == "bark_speex") c.u.melspec.specScale = OSM_B200_SCALE_BARK_SPEEX;
          else if (lv == "bark_schroed") c.u.melspec.specScale = OSM_B200_SCALE_BARK_SCHROED;
          else if (lv.compare(0, 4, "semi") == 0) c.u.melspec.specScale = OSM_B200_SCALE_SEMITONE;
          else if (lv.compare(0, 3, "lin") == 0) c.u.melspec.specScale = OSM_B200_SCALE_LINEAR;
          else if (lv.compare(0, 3, "log") == 0) c.u.melspec.specScale = OSM_B200_SCALE_LOG;
          else c.u.melspec.specScale = OSM_B200_SCALE_MEL;   // unknown: the reference logs an error and assumes mel (:123-125)
          continue;
        }
        if (f == "firstNote") { melFirstNote = num(v); continue; }
        if (f == "logScaleBase") { melLogBase = num(v); continue; }
        if (f == "bwMethod") { if (v.compare(0, 2, "lr") != 0) { err = "cMelspec.bwMethod=" + v + " is not supported"; return false; } continue; }
        if (f == "inverse") { if (inum(v)) { err = "cMelspec.inverse is not supported"; return false; } continue; }
        if (f == "showFbank" || f == "halfBwTarg") continue;
        break;
      case OSM_B200_C_MFCC:
        SETI("firstMfcc", c.u.mfcc.firstMfcc) SETI("lastMfcc", c.u.mfcc.lastMfcc) SETD("melfloor", c.u.mfcc.melfloor)
        SETI("doLog", c.u.mfcc.doLog) SETD("cepLifter", c.u.mfcc.cepLifter) SETI("htkcompatible", c.u.mfcc.htkcompatible)
        if (f == "nMfcc") { if (!s.get("lastMfcc")) c.u.mfcc.lastMfcc = -1000 - inum(v); continue; }   // resolved below
        if (f == "inverse") { if (inum(v)) { err = "cMfcc.inverse is not supported"; return false; } continue; }
        if (f == "nBands" || f == "printDctBaseFunctions") continue;
        break;
      case OSM_B200_C_PLP:
        SETI("lpOrder", c.u.plp.lpOrder) SETI("nCeps", c.u.plp.nCeps) SETI("firstCC", c.u.plp.firstCC) SETI("lastCC", c.u.plp.lastCC)
        SETI("doLog", c.u.plp.doLog) SETI("doAud", c.u.plp.doAud) SETI("RASTA", c.u.plp.RASTA) SETI("newRASTA", c.u.plp.newRASTA)
        SETI("doInvLog", c.u.plp.doInvLog) SETI("doIDFT", c.u.plp.doIDFT) SETI("doLP", c.u.plp.doLP) SETI("doLpToCeps", c.u.plp.doLpToCeps)
        SETD("rastaUpperCutoff", c.u.plp.rastaUpperCutoff) SETD("rastaLowerCutoff", c.u.plp.rastaLowerCutoff)
        SETD("cepLifter", c.u.plp.cepLifter) SETD("compression", c.u.plp.compression) SETD("melfloor", c.u.plp.melfloor)
        SETI("htkcompatible", c.u.plp.htkcompatible)
        break;
      case OSM_B200_C_SPECTRAL: {
        auto &sp = c.u.spectral;
        SETI("squareInput", sp.squareInput) SETI("flux", sp.flux) SETI("centroid", sp.centroid) SETI("maxPos", sp.maxPos)
        SETI("minPos", sp.minPos) SETI("entropy", sp.entropy) SETI("standardDeviation", sp.standardDeviation)
        SETI("variance", sp.variance) SETI("skewness", sp.skewness) SETI("kurtosis", sp.kurtosis) SETI("slope", sp.slope)
        SETI("alphaRatio", sp.alphaRatio) SETI("hammarbergIndex", sp.hammarbergIndex) SETI("sharpness", sp.sharpness)
        SETI("harmonicity", sp.harmonicity) SETI("flatness", sp.flatness) SETI("logFlatness", sp.logFlatness)
        SETI("normBandEnergies", sp.normBandEnergies) SETI("buggyRollOff", sp.buggyRollOff) SETI("oldSlopeScale", sp.oldSlopeScale)
        SETI("useLogSpectrum", sp.useLogSpectrum) SETD("specFloor", sp.specFloor)
        if (f == "freqRange") { if (!parse_range(v, sp.freqRangeLo, sp.freqRangeHi)) { err = "cSpectral.freqRange: bad value '" + v + "'"; return false; } continue; }
        auto arr = [&](const char *base, int &n, double *lo, double *hi) -> int {
          const std::string b = std::string(base) + "[";
          if (f.compare(0, b.size(), b) != 0) return 0;
          const int idx = atoi(f.c_str() + b.size());
          if (idx < 0 || idx >= OSM_B200_MAX_LIST) return -1;
          if (hi) { if (!parse_range(v, lo[idx], hi[idx])) return -1; } else lo[idx] = num(v);
          n = std::max(n, idx + 1);
          return 1;
        };
        int r = arr("bands", sp.nBands, sp.bandLo, sp.bandHi);
        if (!r) r = arr("slopes", sp.nSlopes, sp.slopeLo, sp.slopeHi);
        if (!r) r = arr("rollOff", sp.nRollOff, sp.rollOff, nullptr);
        if (r < 0) { err = "cSpectral: bad array entry '" + f + " = " + v + "'"; return false; }
        if (r > 0) continue;
        if (f == "specDiff" || f == "specPosDiff" || f == "fluxCentroid" || f == "fluxAtFluxCentroid" || f == "tonality") {
          if (inum(v)) { err = "cSpectral." + f + " is not supported"; return false; }
          continue;
        }
        break;
      }
      case OSM_B200_C_ENERGY:
        SETI("htkcompatible", c.u.energy.htkcompatible) SETI("rms", c.u.energy.rms) SETI("energy2", c.u.energy.energy2)
        SETI("log", c.u.energy.log) SETD("escaleLog", c.u.energy.escaleLog) SETD("escaleRms", c.u.energy.escaleRms)
        SETD("escaleSquare", c.u.energy.escaleSquare) SETD("ebiasLog", c.u.energy.ebiasLog) SETD("ebiasRms", c.u.energy.ebiasRms)
        SETD("ebiasSquare", c.u.energy.ebiasSquare)
        break;
      case OSM_B200_C_MZCR:
        SETI("zcr", c.u.mzcr.zcr) SETI("mcr", c.u.mzcr.mcr) SETI("amax", c.u.mzcr.amax) SETI("maxmin", c.u.mzcr.maxmin) SETI("dc", c.u.mzcr.dc)
        break;
      case OSM_B200_C_ACF:
        if (f == "usePower") { c.u.acf.usePower = inum(v); usePowerSet = true; continue; }
        SETI("cepstrum", c.u.acf.cepstrum) SETI("inverse", c.u.acf.inverse) SETI("cosLifterCepstrum", c.u.acf.cosLifterCepstrum)
        SETI("expBeforeAbs", c.u.acf.expBeforeAbs) SETI("symmetricData", c.u.acf.symmetricData)
        SETI("acfCepsNormOutput", c.u.acf.acfCepsNormOutput) SETI("oldCompatCepstrum", c.u.acf.oldCompatCepstrum)
        SETI("absCepstrum", c.u.acf.absCepstrum)
        break;
      case OSM_B200_C_PITCHACF:
        SETD("maxPitch", c.u.pitchacf.maxPitch) SETI("voiceProb", c.u.pitchacf.voiceProb) SETI("voiceQual", c.u.pitchacf.voiceQual)
        SETI("HNR", c.u.pitchacf.HNR) SETI("HNRdB", c.u.pitchacf.HNRdB) SETI("linHNR", c.u.pitchacf.linHNR) SETI("F0", c.u.pitchacf.F0)
        SETI("F0raw", c.u.pitchacf.F0raw) SETI("F0env", c.u.pitchacf.F0env) SETD("voicingCutoff", c.u.pitchacf.voicingCutoff)
        break;
      case OSM_B200_C_DELTAREGRESSION:
        SETI("deltawin", c.u.deltaregression.deltawin) SETI("absOutput", c.u.deltaregression.absOutput)
        SETI("halfWaveRect", c.u.deltaregression.halfWaveRect) SETI("onlyInSegments", c.u.deltaregression.onlyInSegments)
        SETI("zeroSegBound", c.u.deltaregression.zeroSegBound) SETI("relativeDelta", c.u.deltaregression.relativeDelta)
        if (f == "noPostEOIprocessing") { if (inum(v)) { err = "cDeltaRegression.noPostEOIprocessing=1 is not supported"; return false; } continue; }
        break;
      case OSM_B200_C_CONTOURSMOOTHER:
        SETI("smaWin", c.u.contoursmoother.smaWin) SETI("noZeroSma", c.u.contoursmoother.noZeroSma)
        if (f == "noPostEOIprocessing") { if (inum(v)) { err = "cContourSmoother.noPostEOIprocessing=1 is not supported"; return false; } continue; }
        break;
      case OSM_B200_C_VECTORCONCAT:
        break;
      case OSM_B200_C_INTENSITY:
        SETI("intensity", c.u.intensity.intensity) SETI("loudness", c.u.intensity.loudness)
        break;
      case OSM_B200_C_FULLINPUTMEAN:
        SETI("mvn", c.u.fullinputmean.mvn) SETI("symmSubtract", c.u.fullinputmean.symmSubtract)
        SETI("subtractClipToZero", c.u.fullinputmean.subtractClipToZero) SETI("specEnorm", c.u.fullinputmean.specEnorm)
        SETI("htkLogEnorm", c.u.fullinputmean.htkLogEnorm) SETI("excludeZeros", c.u.fullinputmean.excludeZeros)
        SETI("multiLoopMode", c.u.fullinputmean.multiLoopMode)
        if (f == "meanNorm") { c.u.fullinputmean.meanNorm = (v.compare(0, 3, "ame") == 0) ? 0 : 1; continue; }
        if (f == "printMeans" || f == "printStddevs") continue;
        break;
      case OSM_B200_C_VECTOROPERATION:
        if (f == "operation") {
          if (v.compare(0, 3, "ll1") != 0) { err = "cVectorOperation.operation=" + v + " is not supported (ll1 only)"; return false; }
          c.u.vectoroperation.operation = 0;
          continue;
        }
        if (f == "nameBase") { snprintf(c.u.vectoroperation.nameBase, OSM_B200_NAME_LEN, "%s", v.c_str()); continue; }
        if (f == "param1" || f == "param2" || f == "logfloor" || f == "powOnlyPos") continue;
        break;
      case OSM_B200_C_SPECSCALE: {          // dsp/specScale.cpp:38-62,104-176
        auto &q = c.u.specscale;
        SETD("minF", q.minF) SETD("maxF", q.maxF) SETI("nPointsTarget", q.nPointsTarget) SETI("specSmooth", q.specSmooth)
        SETI("specEnhance", q.specEnhance) SETI("auditoryWeighting", q.auditoryWeighting)
        if (f == "scale") {
          std::string l = v; for (auto &ch : l) ch = (char)tolower(ch);
          q.scaleOctave = (l.compare(0, 3, "oct") == 0) ? 1 : ((l.compare(0, 3, "log") == 0) ? 2 : 0);   // 2: needs logScaleBase == 2
          continue;
        }
        if (f == "logScaleBase") { if (num(v) != 2.0) q.scaleOctave = 0; continue; }
        if (f == "sourceScale") { std::string l = v; for (auto &ch : l) ch = (char)tolower(ch); q.sourceLin = l.compare(0, 3, "lin") == 0; continue; }
        if (f == "interpMethod") { q.splineInterp = v == "spline"; continue; }
        if (f == "logSourceScaleBase" || f == "firstNote") continue;
        break;
      }
      case OSM_B200_C_PITCHSHS: {           // lldcore/pitchBase.cpp:41-62, lld/pitchShs.cpp:56-64
        auto &q = c.u.pitchshs;
        SETD("maxPitch", q.maxPitch) SETD("minPitch", q.minPitch) SETI("nCandidates", q.nCandidates) SETI("scores", q.scores)
        SETI("voicing", q.voicing) SETI("F0C1", q.F0C1) SETI("voicingC1", q.voicingC1) SETI("F0raw", q.F0raw)
        SETI("voicingClip", q.voicingClip) SETD("voicingCutoff", q.voicingCutoff) SETI("octaveCorrection", q.octaveCorrection)
        SETI("nHarmonics", q.nHarmonics) SETD("compressionFactor", q.compressionFactor) SETI("greedyPeakAlgo", q.greedyPeakAlgo)
        SETD("lfCut", q.lfCut)
        if (f == "shsSpectrumOutput") { if (inum(v)) { err = "cPitchShs.shsSpectrumOutput=1 is not supported"; return false; } continue; }
        if (f == "inputFieldSearch" || f.compare(0, 10, "shsWriter.") == 0) continue;
        break;
      }
      case OSM_B200_C_PITCHSMOOTHERVITERBI: {   // lld/pitchSmootherViterbi.cpp:45-68
        auto &q = c.u.pitchsmootherviterbi;
        SETI("bufferLength", q.bufferLength) SETI("F0final", q.F0final) SETI("F0finalLog", q.F0finalLog) SETI("F0finalEnv", q.F0finalEnv)
        SETI("F0finalEnvLog", q.F0finalEnvLog) SETI("voicingFinalClipped", q.voicingFinalClipped)
        SETI("voicingFinalUnclipped", q.voicingFinalUnclipped) SETI("F0raw", q.F0raw) SETI("voicingC1", q.voicingC1)
        SETI("voicingClip", q.voicingClip) SETD("wLocal", q.wLocal) SETD("wTvv", q.wTvv) SETD("wTvvd", q.wTvvd) SETD("wTvuv", q.wTvuv)
        SETD("wThr", q.wThr) SETD("wRange", q.wRange) SETD("wTuu", q.wTuu)
        if (f == "no0f0") continue;
        if (f == "reader2.dmLevel") {        // the second reader only fetches time stamps; it must name the same level
          const std::string *r1 = s.get("reader.dmLevel");
          if (!r1 || *r1 != v) { err = "cPitchSmootherViterbi: reader2.dmLevel must equal reader.dmLevel"; return false; }
          continue;
        }
        if (f.compare(0, 8, "reader2.") == 0) continue;
        break;
      }
      case OSM_B200_C_VALBASEDSELECTOR: {   // other/valbasedSelector.cpp:35-49
        auto &q = c.u.valbasedselector;
        SETD("threshold", q.threshold) SETI("idx", q.idx) SETI("invert", q.invert) SETI("allowEqual", q.allowEqual)
        SETI("removeIdx", q.removeIdx) SETI("zeroVec", q.zeroVec) SETD("outputVal", q.outputVal)
        SETI("adaptiveThreshold", q.adaptiveThreshold)
        if (f == "adaptationLengthSec" || f == "adaptationLength" || f == "debugAdaptiveThreshold") continue;
        break;
      }
      case OSM_B200_C_PITCHJITTER: {        // lld/pitchJitter.cpp:45-78
        auto &q = c.u.pitchjitter;
        if (f == "F0reader.dmLevel") { snprintf(q.F0reader_dmLevel, OSM_B200_NAME_LEN, "%s", v.c_str()); continue; }
        if (f == "F0field") { snprintf(q.F0field, OSM_B200_NAME_LEN, "%s", v.c_str()); continue; }
        SETD("searchRangeRel", q.searchRangeRel) SETI("jitterLocal", q.jitterLocal) SETI("jitterDDP", q.jitterDDP)
        SETI("jitterLocalEnv", q.jitterLocalEnv) SETI("jitterDDPEnv", q.jitterDDPEnv) SETI("shimmerLocal", q.shimmerLocal)
        SETI("shimmerLocalDB", q.shimmerLocalDB) SETI("shimmerLocalEnv", q.shimmerLocalEnv) SETI("shimmerLocalDBEnv", q.shimmerLocalDBEnv)
        SETI("harmonicERMS", q.harmonicERMS) SETI("noiseERMS", q.noiseERMS) SETI("linearHNR", q.linearHNR) SETI("logHNR", q.logHNR)
        SETD("lgHNRfloor", q.lgHNRfloor) SETI("shimmerUseRmsAmplitude", q.shimmerUseRmsAmplitude) SETI("minNumPeriods", q.minNumPeriods)
        SETD("minCC", q.minCC) SETI("refinedF0", q.refinedF0) SETI("sourceQualityRange", q.sourceQualityRange)
        SETI("sourceQualityMean", q.sourceQualityMean) SETI("usePeakToPeakPeriodLength", q.usePeakToPeakPeriodLength)
        SETI("useBrokenJitterThresh", q.useBrokenJitterThresh) SETI("onlyVoiced", q.onlyVoiced)
        if (f == "periodOutputFile") { if (!v.empty()) { err = "cPitchJitter.periodOutputFile is not supported"; return false; } continue; }
        if (f == "inputMaxDelaySec" || f.compare(0, 9, "F0reader.") == 0) continue;
        break;
      }
      case OSM_B200_C_SPECRESAMPLE: {       // dsp/specResample.cpp:36-46
        auto &q = c.u.specresample;
        SETD("targetFs", q.targetFs) SETD("resampleRatio", q.resampleRatio)
        if (f == "inputFieldPartial") { if (!v.empty()) { err = "cSpecResample.inputFieldPartial is not supported"; return false; } continue; }
        break;
      }
      case OSM_B200_C_LPC: {                // lld/lpc.cpp:33-45
        auto &q = c.u.lpc;
        if (f == "method") { q.method = (v == "acf") ? 0 : 1; continue; }
        SETI("p", q.p) SETI("saveLPCoeff", q.saveLPCoeff) SETI("lpGain", q.lpGain) SETI("saveRefCoeff", q.saveRefCoeff)
        SETI("residual", q.residual) SETI("residualGainScale", q.residualGainScale) SETI("forwardFilter", q.forwardFilter)
        SETI("lpSpectrum", q.lpSpectrum)
        if (f == "forwardLPspec" || f == "forwardLPspecFloor" || f == "lpSpecDeltaF" || f == "lpSpecBins") continue;   // only read with lpSpectrum=1
        break;
      }
      case OSM_B200_C_DATASELECTOR: {       // core/dataSelector.cpp:35-41
        auto &q = c.u.dataselector;
        if (f == "selected" || f == "newNames") {          // array fields: a;b;c (configManager array syntax)
          int k = 0;
          size_t a = 0;
          while (a <= v.size()) {
            size_t b = v.find(';', a);
            if (b == std::string::npos) b = v.size();
            std::string item = v.substr(a, b - a);
            while (!item.empty() && (item.back() == ' ' || item.back() == '\t')) item.pop_back();
            while (!item.empty() && (item.front() == ' ' || item.front() == '\t')) item.erase(item.begin());
            if (b == v.size() && item.empty()) break;       // trailing ';'
            if (k >= OSM_B200_MAX_SELECTED) { err = "cDataSelector: more than 32 selected elements"; return false; }
            if (item.size() >= OSM_B200_NAME_LEN) { err = "cDataSelector: element name too long: " + item; return false; }
            snprintf(f == "selected" ? q.selected[k] : q.newNames[k], OSM_B200_NAME_LEN, "%s", item.c_str());
            k++;
            a = b + 1;
          }
          if (f == "selected") q.nSelected = k;
          continue;
        }
        {                                                   // indexed form: selected[2] = name
          const bool isSel = f.compare(0, 9, "selected[") == 0, isNew = f.compare(0, 9, "newNames[") == 0;
          if (isSel || isNew) {
            const int idx = atoi(f.c_str() + 9);
            if (idx < 0 || idx >= OSM_B200_MAX_SELECTED || v.size() >= OSM_B200_NAME_LEN) { err = "cDataSelector: bad array index / name too long in '" + f + "'"; return false; }
            snprintf(isSel ? q.selected[idx] : q.newNames[idx], OSM_B200_NAME_LEN, "%s", v.c_str());
            if (isSel) q.nSelected = std::max(q.nSelected, idx + 1);
            continue;
          }
        }
        SETI("elementMode", q.elementMode)
        if (f == "selFile" || f == "selectedRange" || f == "outputSingleField") { if (!v.empty()) { err = "cDataSelector." + f + " is not supported"; return false; } continue; }
        if (f == "dummyMode") { if (inum(v)) { err = "cDataSelector.dummyMode is not supported"; return false; } continue; }
        break;
      }
      case OSM_B200_C_HARMONICS: {          // lld/harmonics.cpp:28-56
        auto &q = c.u.harmonics;
#define SETS(field, member) if (f == field) { if (v.size() >= sizeof(member)) { err = "cHarmonics." + f + ": name too long"; return false; } snprintf(member, sizeof(member), "%s", v.c_str()); continue; }
        SETS("f0ElementName", q.f0ElementName) SETS("magSpecFieldName", q.magSpecFieldName)
        SETS("formantFrequencyFieldName", q.formantFrequencyFieldName) SETS("formantBandwidthFieldName", q.formantBandwidthFieldName)
#undef SETS
        SETI("f0ElementNameIsFull", q.f0ElementNameIsFull) SETI("magSpecFieldNameIsFull", q.magSpecFieldNameIsFull)
        SETI("formantFrequencyFieldNameIsFull", q.formantFrequencyFieldNameIsFull) SETI("formantBandwidthFieldNameIsFull", q.formantBandwidthFieldNameIsFull)
        SETI("nHarmonics", q.nHarmonics) SETI("firstHarmonicMagnitude", q.firstHarmonicMagnitude) SETI("nHarmonicMagnitudes", q.nHarmonicMagnitudes)
        SETI("outputLogRelMagnitudes", q.outputLogRelMagnitudes) SETI("outputLinearMagnitudes", q.outputLinearMagnitudes)
        SETI("harmonicDifferencesLog", q.harmonicDifferencesLog) SETI("harmonicDifferencesRatioLinear", q.harmonicDifferencesRatioLinear)
        SETI("formantAmplitudes", q.formantAmplitudes) SETI("formantAmplitudesLinear", q.formantAmplitudesLinear)
        SETI("formantAmplitudesLogRel", q.formantAmplitudesLogRel) SETI("formantAmplitudesStart", q.formantAmplitudesStart)
        SETI("formantAmplitudesEnd", q.formantAmplitudesEnd) SETI("computeAcfHnrLogdB", q.computeAcfHnrLogdB)
        SETI("computeAcfHnrLinear", q.computeAcfHnrLinear) SETD("logRelValueFloorUnvoiced", q.logRelValueFloorUnvoiced)
        if (f.compare(0, 20, "harmonicDifferences[") == 0) {   // indexed form
          const int idx = atoi(f.c_str() + 20);
          if (idx < 0 || idx >= 4 || v.size() >= 16) { err = "cHarmonics.harmonicDifferences: at most 4 entries of < 16 characters"; return false; }
          snprintf(q.harmonicDifferences[idx], 16, "%s", v.c_str());
          q.nHarmonicDifferences = std::max(q.nHarmonicDifferences, idx + 1);
          continue;
        }
        if (f == "harmonicDifferences") {                   // array field: H1-H2;H1-A3
          int k = 0;
          size_t a = 0;
          while (a <= v.size()) {
            size_t b = v.find(';', a);
            if (b == std::string::npos) b = v.size();
            std::string item = v.substr(a, b - a);
            while (!item.empty() && item.back() == ' ') item.pop_back();
            while (!item.empty() && item.front() == ' ') item.erase(item.begin());
            if (b == v.size() && item.empty()) break;
            if (k >= 4 || item.size() >= 16) { err = "cHarmonics.harmonicDifferences: at most 4 entries of < 16 characters"; return false; }
            snprintf(q.harmonicDifferences[k++], 16, "%s", item.c_str());
            a = b + 1;
          }
          q.nHarmonicDifferences = k;
          continue;
        }
        break;
      }
      case OSM_B200_C_FORMANTLPC: {         // lld/formantLpc.cpp:40-52
        auto &q = c.u.formantlpc;
        SETI("nFormants", q.nFormants) SETI("saveFormants", q.saveFormants) SETI("saveIntensity", q.saveIntensity)
        SETI("saveNumberOfValidFormants", q.saveNumberOfValidFormants) SETI("saveBandwidths", q.saveBandwidths)
        SETD("minF", q.minF) SETD("maxF", q.maxF) SETI("useLpSpec", q.useLpSpec) SETI("medianFilter", q.medianFilter)
        SETI("octaveCorrection", q.octaveCorrection)
        break;
      }
      case OSM_B200_C_TONESPEC: {           // lld/tonespec.cpp:46-56: printBinMap / printFilterMap exist in DEBUG builds only
        auto &q = c.u.tonespec;
        SETI("nOctaves", q.nOctaves) SETD("firstNote", q.firstNote) SETI("usePower", q.usePower) SETI("dbA", q.dbA)
        if (f == "filterType") { q.filterType = tone_filter(v); continue; }
        break;
      }
      case OSM_B200_C_CHROMA:               // lld/chroma.cpp:46-49
        SETI("octaveSize", c.u.chroma.octaveSize) SETD("silThresh", c.u.chroma.silThresh)
        break;
      case OSM_B200_C_TONEFILT: {           // lld/tonefilt.cpp:35-41 (outputBuffersize is commented out there: unknown)
        auto &q = c.u.tonefilt;
        SETI("nNotes", q.nNotes) SETD("firstNote", q.firstNote) SETD("decayF0", q.decayF0) SETD("decayFN", q.decayFN)
        SETD("outputPeriod", q.outputPeriod)
        break;
      }
      case OSM_B200_C_CENS: {               // lld/cens.cpp:40-48, 64-105
        auto &q = c.u.cens;
        // strncmp on the first three characters, case-sensitive; any other string is Hanning (with an error message there)
        if (f == "window") {
          q.window = v.compare(0, 3, "ham") == 0 ? OSM_B200_WIN_HAMMING : (v.compare(0, 3, "bar") == 0 ? OSM_B200_WIN_BARTLETT : OSM_B200_WIN_HANNING);
          continue;
        }
        SETI("winlength", q.winlength) SETI("l2norm", q.l2norm) SETI("downsampleRatio", q.downsampleRatio)
        if (f == "winlength_sec") { q.winlength_sec = num(v); q.winlength_secSet = 1; continue; }
        break;
      }
      default: break;
    }
    // same behaviour as the reference: an unknown field aborts configuration (configManager.cpp:2599)
    err = "unknown field '" + f + "' in section [" + s.name + ":" + s.type + "]";
    return false;
  }
  if (t == OSM_B200_C_MFCC && c.u.mfcc.lastMfcc <= -1000)          // lastMfcc = firstMfcc + nMfcc - 1 (lldcore/mfcc.cpp:77-82)
    c.u.mfcc.lastMfcc = c.u.mfcc.firstMfcc + (-1000 - c.u.mfcc.lastMfcc) - 1;
  if (t == OSM_B200_C_ACF && c.u.acf.cepstrum && !usePowerSet) c.u.acf.usePower = 0;   // dspcore/acf.cpp:91-99
  if (t == OSM_B200_C_MELSPEC)
    c.u.melspec.scaleParam = c.u.melspec.specScale == OSM_B200_SCALE_SEMITONE ? melFirstNote : (c.u.melspec.specScale == OSM_B200_SCALE_LOG ? melLogBase : 0.0);
  if (t == OSM_B200_C_WINDOWER) {                                  // window coefficients, dspcore/windower.cpp:83-113
    auto &w = c.u.windower;
    const std::string *a = s.get("alpha"), *a0 = s.get("alpha0"), *a1 = s.get("alpha1"), *a2 = s.get("alpha2"), *a3 = s.get("alpha3");
    if (w.winFunc == OSM_B200_WIN_BLACKMAN) {
      if (a0 && a1 && a2) { w.alpha0 = num(*a0); w.alpha1 = num(*a1); w.alpha2 = num(*a2); }
      else { const double al = a ? num(*a) : 0.16; w.alpha0 = (1.0 - al) * 0.5; w.alpha1 = 0.5; w.alpha2 = al * 0.5; }
    } else if (w.winFunc == OSM_B200_WIN_BLACKHARR) {
      w.alpha0 = a0 ? num(*a0) : 0.35875; w.alpha1 = a1 ? num(*a1) : 0.48829; w.alpha2 = a2 ? num(*a2) : 0.14128; w.alpha3 = a3 ? num(*a3) : 0.01168;
    } else if (w.winFunc == OSM_B200_WIN_BARTHANN) {
      w.alpha0 = a0 ? num(*a0) : 0.62; w.alpha1 = a1 ? num(*a1) : 0.48; w.alpha2 = a2 ? num(*a2) : 0.38;
    }
  }
  if (t == OSM_B200_C_VECTOROPERATION && c.u.vectoroperation.operation < 0) { err = "cVectorOperation.operation=norm (the default) is not supported (ll1 only)"; return false; }
  return true;
}

// ------------------------------------------------------------------------------------------
// [x:cFunctionals] -> osm_b200_functionals_spec (src/functionals/functionals.cpp:33-100, the sub-components' registerComponent
// blocks for the field names).  Only full-input mode (frameMode = full, shared/FrameModeFunctionals.conf.inc) is executed.
// ------------------------------------------------------------------------------------------
int time_norm(const std::string &v)          // functionalComponent.cpp:51-64: prefix match
{
  if (v.compare(0, 3, "tur") == 0 || v.compare(0, 3, "seg") == 0) return OSM_B200_TIMENORM_SEGMENT;
  if (v.compare(0, 3, "sec") == 0) return OSM_B200_TIMENORM_SECOND;
  if (v.compare(0, 3, "fra") == 0) return OSM_B200_TIMENORM_FRAME;
  return OSM_B200_TIMENORM_UNSET;
}

osm_b200_status to_functionals(const Section &s, osm_b200_functionals_spec &fs, std::string &err)
{
  auto fail = [&err](osm_b200_status st, const std::string &m) { err = m; return st; };
  osm_b200_functionals_defaults(&fs);
  std::map<int, std::string> enabledIdx;         // functionalsEnabled[i] entries
  std::string enabledList;
  std::map<int, double> pct;
  std::map<int, std::string> pctRange;
  bool quartilesSet = false, iqrSet = false;
  int quartiles = 0, iqr = 0;
  auto &E = fs.extremes; auto &M = fs.means; auto &Q = fs.moments; auto &P = fs.percentiles; auto &R = fs.regression;
  auto &TI = fs.times; auto &LP = fs.lpc; auto &SG = fs.segments; auto &PK = fs.peaks2;
  std::map<int, double> segThresh;
  std::string segThreshList, segAlgo = "delta";
  bool unsupportedTimes = false, unsupportedSeg = false, unsupportedPeaks = false, peaksNoOverlap = false;
  std::map<int, double> samplePos;
  int dctLast = 6, dctN = -1;
  bool frameModeFull = false, subWindow = false;
  double onsetThr = 0.0, onsetThrOn = 0.0, onsetThrOff = 0.0;
  bool onsetThrOnSet = false, onsetThrOffSet = false;
  auto &ON = fs.onset; auto &PO = fs.peaks; auto &CR = fs.crossings;
  static const char *peaksNames[OSM_B200_F_PEAKS2_VALUES] = {"numPeaks", "meanPeakDist", "meanPeakDistDelta", "peakDistStddev", "peakRangeAbs",
      "peakRangeRel", "peakMeanAbs", "peakMeanMeanDist", "peakMeanRel", "ptpAmpMeanAbs", "ptpAmpMeanRel", "ptpAmpStddevAbs", "ptpAmpStddevRel",
      "minRangeAbs", "minRangeRel", "minMeanAbs", "minMeanMeanDist", "minMeanRel", "mtmAmpMeanAbs", "mtmAmpMeanRel", "mtmAmpStddevAbs",
      "mtmAmpStddevRel", "meanRisingSlope", "maxRisingSlope", "minRisingSlope", "stddevRisingSlope", "meanFallingSlope", "maxFallingSlope",
      "minFallingSlope", "stddevFallingSlope", "covFallingSlope", "covRisingSlope"};   // configuration field = value name (functionalPeaks2.cpp:84-118)
  struct IntField { const char *name; int32_t *dst; };
  const IntField fields[] = {
    {"Extremes.max", &E.max}, {"Extremes.min", &E.min}, {"Extremes.range", &E.range}, {"Extremes.maxpos", &E.maxpos}, {"Extremes.minpos", &E.minpos},
    {"Extremes.amean", &E.amean}, {"Extremes.maxameandist", &E.maxameandist}, {"Extremes.minameandist", &E.minameandist},
    {"Means.amean", &M.amean}, {"Means.absmean", &M.absmean}, {"Means.qmean", &M.qmean}, {"Means.nzamean", &M.nzamean}, {"Means.nzabsmean", &M.nzabsmean},
    {"Means.nzqmean", &M.nzqmean}, {"Means.nzgmean", &M.nzgmean}, {"Means.nnz", &M.nnz}, {"Means.flatness", &M.flatness}, {"Means.posamean", &M.posamean},
    {"Means.negamean", &M.negamean}, {"Means.posqmean", &M.posqmean}, {"Means.posrqmean", &M.posrqmean}, {"Means.negqmean", &M.negqmean},
    {"Means.negrqmean", &M.negrqmean}, {"Means.rqmean", &M.rqmean}, {"Means.nzrqmean", &M.nzrqmean},
    {"Moments.variance", &Q.variance}, {"Moments.stddev", &Q.stddev}, {"Moments.skewness", &Q.skewness}, {"Moments.kurtosis", &Q.kurtosis},
    {"Moments.amean", &Q.amean}, {"Moments.stddevNorm", &Q.stddevNorm}, {"Moments.doRatioLimit", &Q.doRatioLimit},
    {"Percentiles.quartile1", &P.quartile1}, {"Percentiles.quartile2", &P.quartile2}, {"Percentiles.quartile3", &P.quartile3},
    {"Percentiles.iqr12", &P.iqr12}, {"Percentiles.iqr23", &P.iqr23}, {"Percentiles.iqr13", &P.iqr13}, {"Percentiles.interp", &P.interp},
    {"Regression.linregc1", &R.linregc1}, {"Regression.linregc2", &R.linregc2}, {"Regression.linregerrA", &R.linregerrA}, {"Regression.linregerrQ", &R.linregerrQ},
    {"Regression.qregc1", &R.qregc1}, {"Regression.qregc2", &R.qregc2}, {"Regression.qregc3", &R.qregc3}, {"Regression.qregerrA", &R.qregerrA},
    {"Regression.qregerrQ", &R.qregerrQ}, {"Regression.centroid", &R.centroid}, {"Regression.centroidUseAbsValues", &R.centroidUseAbsValues},
    {"Regression.centroidRatioLimit", &R.centroidRatioLimit}, {"Regression.normRegCoeff", &R.normRegCoeff}, {"Regression.normInputs", &R.normInputs},
    {"Regression.oldBuggyQerr", &R.oldBuggyQerr}, {"Regression.doRatioLimit", &R.doRatioLimit},
    {"Times.upleveltime25", &TI.upleveltime25}, {"Times.downleveltime25", &TI.downleveltime25}, {"Times.upleveltime50", &TI.upleveltime50},
    {"Times.downleveltime50", &TI.downleveltime50}, {"Times.upleveltime75", &TI.upleveltime75}, {"Times.downleveltime75", &TI.downleveltime75},
    {"Times.upleveltime90", &TI.upleveltime90}, {"Times.downleveltime90", &TI.downleveltime90}, {"Times.risetime", &TI.risetime},
    {"Times.falltime", &TI.falltime}, {"Times.leftctime", &TI.leftctime}, {"Times.rightctime", &TI.rightctime}, {"Times.duration", &TI.duration},
    {"Times.buggySecNorm", &TI.buggySecNorm},
    {"Lpc.lpGain", &LP.lpGain}, {"Lpc.lpc", &LP.lpc}, {"Lpc.firstCoeff", &LP.firstCoeff}, {"Lpc.order", &LP.order},
    {"Segments.numSegments", &SG.numSegments}, {"Segments.meanSegLen", &SG.meanSegLen}, {"Segments.maxSegLen", &SG.maxSegLen},
    {"Segments.minSegLen", &SG.minSegLen}, {"Segments.segLenStddev", &SG.segLenStddev}, {"Segments.maxNumSeg", &SG.maxNumSeg},
    {"Segments.XisRel", &SG.XisRel}, {"Segments.pauseMinLng", &SG.pauseMinLng},
    {"Peaks2.dynRelThresh", &PK.dynRelThresh}, {"Peaks2.doRatioLimit", &PK.doRatioLimit},
    {"Onset.onsetPos", &ON.onsetPos}, {"Onset.offsetPos", &ON.offsetPos}, {"Onset.numOnsets", &ON.numOnsets}, {"Onset.numOffsets", &ON.numOffsets},
    {"Onset.onsetRate", &ON.onsetRate}, {"Onset.useAbsVal", &ON.useAbsVal},
    {"Peaks.numPeaks", &PO.numPeaks}, {"Peaks.meanPeakDist", &PO.meanPeakDist}, {"Peaks.peakMean", &PO.peakMean},
    {"Peaks.peakMeanMeanDist", &PO.peakMeanMeanDist}, {"Peaks.peakDistStddev", &PO.peakDistStddev},
    {"Crossings.zcr", &CR.zcr}, {"Crossings.mcr", &CR.mcr}, {"Crossings.amean", &CR.amean}};
  for (const auto &kv : s.kv) {
    const std::string &f = kv.first, &v = kv.second;
    // EOIlevel > 0 makes the summary wait for later end-of-input passes (more rows of the window processors behind it); a frame list
    // cuts the input into several summaries: both change what the rows mean and are refused rather than ignored
    if (f == "EOIlevel" && inum(v) != 0) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionals.EOIlevel != 0 is not supported (the summary is taken at the first end-of-input tick)");
    if ((f == "frameListFile" || f == "frameList") && !trim(v).empty()) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionals." + f + " is not supported");
    if (is_common(f) || f == "noPostEOIprocessing" || f == "allowLastFrameIncomplete" || f == "frameListFile" || f == "frameList") continue;
    if (f == "frameMode") { frameModeFull = true; if (v.compare(0, 3, "ful") != 0) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionals.frameMode=" + v + " is not supported (only full-input summaries)"); continue; }
    if (f == "frameSize" || f == "frameStep" || f == "frameSizeFrames" || f == "frameStepFrames") { if (num(v) != 0.0) subWindow = true; continue; }
    if (f == "frameCenterSpecial" || f == "frameCenter" || f == "frameCenterFrames") continue;
    if (f == "functionalsEnabled") { enabledList = v; continue; }
    if (f.compare(0, 19, "functionalsEnabled[") == 0) { enabledIdx[atoi(f.c_str() + 19)] = v; continue; }
    if (f == "nonZeroFuncts") { fs.nonZeroFuncts = inum(v); continue; }
    if (f == "functNameAppend") { snprintf(fs.functNameAppend, sizeof fs.functNameAppend, "%s", v.c_str()); continue; }
    if (f == "masterTimeNorm") { fs.masterTimeNorm = time_norm(v); continue; }
    if (f == "preserveFields") continue;             // checked by the session against the input level (single-element fields only)
    if (f == "Extremes.norm") { E.norm = time_norm(v); E.normIsSet = 1; continue; }
    if (f == "Means.norm") { M.norm = time_norm(v); M.normIsSet = 1; continue; }
    if (f == "Regression.centroidNorm") { R.centroidNorm = time_norm(v); continue; }
    if (f == "Times.norm") { TI.norm = time_norm(v); TI.normIsSet = 1; continue; }
    if (f == "Segments.norm") { SG.norm = time_norm(v); SG.normIsSet = 1; continue; }
    if (f == "Peaks2.norm") { PK.norm = time_norm(v); PK.normIsSet = 1; continue; }
    if (f.compare(0, 17, "Times.upleveltime") == 0 || f.compare(0, 19, "Times.downleveltime") == 0) {
      bool fixedName = false;
      for (const char *sfx : {"25", "50", "75", "90"}) fixedName = fixedName || f == std::string("Times.upleveltime") + sfx || f == std::string("Times.downleveltime") + sfx;
      if (!fixedName) { unsupportedTimes = true; continue; }         // the upleveltime[] / downleveltime[] arrays
    }
    if (f == "Times.useRobustPercentileRange") { if (inum(v)) unsupportedTimes = true; continue; }
    if (f == "Times.pctlRangeMargin") continue;
    if (f == "Segments.segmentationAlgorithm") { segAlgo = v; continue; }
    if (f == "Segments.thresholds") { segThreshList = v; continue; }
    if (f.compare(0, 20, "Segments.thresholds[") == 0) { segThresh[atoi(f.c_str() + 20)] = num(v); continue; }
    if (f == "Segments.X") { SG.X = (float)num(v); continue; }
    if (f == "Segments.segMinLng") { SG.segMinLng = inum(v); SG.segMinLngIsSet = 1; continue; }
    if (f == "Segments.ravgLng" || f == "Segments.rangeRelThreshold" || f == "Segments.dbgPrint") continue;   // not read by relTh / nonX / eqX
    if (f == "Segments.useOldBuggyChX" || f == "Segments.growDynSegBuffer") { if (inum(v)) unsupportedSeg = true; continue; }
    if (f == "Peaks2.relThresh") { PK.relThresh = (float)num(v); continue; }
    if (f == "Peaks2.absThresh") { PK.absThresh = (float)num(v); PK.useAbsThresh = 1; continue; }
    if (f == "Peaks2.noClearPeakList") { if (inum(v)) unsupportedPeaks = true; continue; }
    if (f == "Peaks2.posDbgOutp" || f == "Peaks2.posDbgAppend" || f == "Peaks2.consoleDbg") continue;
    if (f.compare(0, 7, "Peaks2.") == 0) {
      bool hitP = false;
      for (int k = 0; k < OSM_B200_F_PEAKS2_VALUES; k++) if (f.compare(7, std::string::npos, peaksNames[k]) == 0) { PK.value[k] = inum(v); hitP = true; break; }
      if (hitP) continue;
    }
    if (f.compare(0, 18, "Samples.samplepos[") == 0) { samplePos[atoi(f.c_str() + 18)] = num(v); continue; }
    if (f == "Samples.samplepos") {
      const std::vector<std::string> items = split_list(v);
      for (size_t k = 0; k < items.size(); k++) samplePos[(int)k] = num(items[k]);
      continue;
    }
    if (f == "DCT.firstCoeff") { fs.dct.firstCoeff = std::max(0, inum(v)); continue; }          // functionalDCT.cpp:58-62
    if (f == "DCT.lastCoeff") { dctLast = inum(v); continue; }
    if (f == "DCT.nCoeffs") { dctN = inum(v); continue; }
    if (f == "Onset.threshold") { onsetThr = num(v); continue; }
    if (f == "Onset.thresholdOnset") { onsetThrOn = num(v); onsetThrOnSet = true; continue; }
    if (f == "Onset.thresholdOffset") { onsetThrOff = num(v); onsetThrOffSet = true; continue; }
    if (f == "Onset.norm") { fs.onset.norm = time_norm(v); fs.onset.normIsSet = 1; continue; }
    if (f == "Peaks.norm") { fs.peaks.norm = time_norm(v); fs.peaks.normIsSet = 1; continue; }
    if (f == "Peaks.overlapFlag") { peaksNoOverlap = inum(v) == 0; continue; }
    if (f == "Percentiles.quartiles") { quartilesSet = true; quartiles = inum(v); continue; }
    if (f == "Percentiles.iqr") { iqrSet = true; iqr = inum(v); continue; }
    if (f.compare(0, 23, "Percentiles.percentile[") == 0) { pct[atoi(f.c_str() + 23)] = num(v); continue; }
    if (f.compare(0, 22, "Percentiles.pctlrange[") == 0) { pctRange[atoi(f.c_str() + 22)] = v; continue; }
    // array fields given as one `a;b;c` list (core/configManager.cpp:2229-2262: the elements are assigned in order from index 0)
    if (f == "Percentiles.percentile" || f == "Percentiles.pctlrange") {
      const std::vector<std::string> items = split_list(v);
      for (size_t k = 0; k < items.size(); k++) { if (f == "Percentiles.percentile") pct[(int)k] = num(items[k]); else pctRange[(int)k] = items[k]; }
      continue;
    }
    if (f.compare(0, 24, "Percentiles.pctlquotient") == 0 || f.compare(0, 15, "Percentiles.iqq") == 0) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionalPercentiles: quotients are not supported");
    if (f.compare(0, 15, "Regression.qreg") == 0 && (f == "Regression.qregls" || f == "Regression.qregrs" || f == "Regression.qregx0" || f == "Regression.qregy0" ||
        f == "Regression.qregyr" || f == "Regression.qregy0nn" || f == "Regression.qregc3nn" || f == "Regression.qregyrnn")) {
      if (inum(v)) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionalRegression." + f.substr(11) + " is not supported");
      continue;
    }
    bool hit = false;
    for (const IntField &fd : fields) if (f == fd.name) { *fd.dst = inum(v); hit = true; break; }
    if (hit) continue;
    // a sub-configuration of a functional that is not implemented is only an error if that functional is enabled (below)
    const size_t dot = f.find('.');
    if (dot != std::string::npos) {
      const std::string sub = f.substr(0, dot);
      static const char *known[] = {"Crossings", "DCT", "Modulation", "Onset", "Peaks", "Samples"};
      bool other = false;
      for (const char *k : known) other = other || sub == k;
      if (other) continue;
    }
    return fail(OSM_B200_ERR_INVALID, "unknown field '" + f + "' in section [" + s.name + ":cFunctionals]");
  }
  fs.dct.lastCoeff = dctN >= 0 ? fs.dct.firstCoeff + dctN - 1 : dctLast;            // functionalDCT.cpp:63-68
  if (!samplePos.empty()) {                                                         // functionalSamples.cpp:50-66 (clipped to [0, 1])
    if (samplePos.size() > OSM_B200_F_MAX_SAMPLES) return fail(OSM_B200_ERR_INVALID, "cFunctionalSamples: more than 16 sample positions");
    fs.samples.n_samplepos = 0;
    for (const auto &kv : samplePos) fs.samples.samplepos[fs.samples.n_samplepos++] = std::min(1.0, std::max(0.0, kv.second));
  }
  ON.thresholdOnset = (float)(onsetThrOnSet ? onsetThrOn : onsetThr);               // functionalOnset.cpp:77-81
  ON.thresholdOffset = (float)(onsetThrOffSet ? onsetThrOff : onsetThr);
  if (quartilesSet) P.quartile1 = P.quartile2 = P.quartile3 = quartiles;          // functionalPercentiles.cpp:112-116
  if (iqrSet) P.iqr12 = P.iqr23 = P.iqr13 = iqr;
  std::vector<std::string> names;
  if (!enabledIdx.empty()) for (const auto &kv : enabledIdx) names.push_back(trim(kv.second));
  else names = split_list(enabledList);
  if (names.empty()) return fail(OSM_B200_ERR_INVALID, "cFunctionals '" + s.name + "': functionalsEnabled is empty");
  // the reference's default frameMode is "fixed" (core/winToVecProcessor.cpp:66): a section that does not say frameMode = full
  // summarises sub-windows of frameSize seconds (MediaEval_Audio_IS12based_subwin2.conf: 2 s) -- not the full-input summary built here
  if (!frameModeFull) return fail(OSM_B200_ERR_UNSUPPORTED, std::string("cFunctionals '") + s.name + "': frameMode = fixed (the default" + (subWindow ? ", with a frameSize" : "") + ") is not supported (only full-input summaries: frameMode = full)");

  if (names.size() > OSM_B200_F_MAX_ENABLED) return fail(OSM_B200_ERR_INVALID, "cFunctionals: too many enabled functionals");
  fs.n_enabled = 0;
  for (const std::string &n : names) {
    int t = -1;
    if (n == "Extremes") t = OSM_B200_F_EXTREMES;
    else if (n == "Means") t = OSM_B200_F_MEANS;
    else if (n == "Moments") t = OSM_B200_F_MOMENTS;
    else if (n == "Percentiles") t = OSM_B200_F_PERCENTILES;
    else if (n == "Regression") t = OSM_B200_F_REGRESSION;
    else if (n == "Times") t = OSM_B200_F_TIMES;
    else if (n == "Lpc") t = OSM_B200_F_LPC;
    else if (n == "Segments") t = OSM_B200_F_SEGMENTS;
    else if (n == "Peaks2") t = OSM_B200_F_PEAKS2;
    else if (n == "Onset") t = OSM_B200_F_ONSET;
    else if (n == "Peaks") t = OSM_B200_F_PEAKS;
    else if (n == "Crossings") t = OSM_B200_F_CROSSINGS;
    else if (n == "Samples") t = OSM_B200_F_SAMPLES;
    else if (n == "DCT") t = OSM_B200_F_DCT;
    else return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctional" + n + " (instance '" + s.name + "') is not supported on the GPU path (Extremes, Means, Moments, Percentiles, Regression, Times, Lpc, Segments, Peaks2, Onset, Peaks, Crossings, Samples, DCT are)");
    if (t == OSM_B200_F_PEAKS && peaksNoOverlap) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionalPeaks.overlapFlag = 0 (peak history carried from one contour to the next) is not supported");
    fs.enabled[fs.n_enabled++] = t;
    if (t == OSM_B200_F_TIMES && unsupportedTimes) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionalTimes: upleveltime[] / downleveltime[] arrays and useRobustPercentileRange are not supported");
    if (t == OSM_B200_F_PEAKS2 && unsupportedPeaks) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionalPeaks2.noClearPeakList = 1 is not supported");
    if (t == OSM_B200_F_SEGMENTS) {
      if (unsupportedSeg) return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionalSegments: useOldBuggyChX / growDynSegBuffer are not supported");
      // functionalSegments.cpp:124-158: prefix match in this order
      if (segAlgo.compare(0, 5, "relTh") == 0) SG.algorithm = OSM_B200_SEG_RELTH;
      else if (segAlgo.compare(0, 4, "nonX") == 0) SG.algorithm = OSM_B200_SEG_NONX;
      else if (segAlgo.compare(0, 3, "eqX") == 0) SG.algorithm = OSM_B200_SEG_EQX;
      else if (segAlgo.compare(0, 7, "NArelTh") == 0) SG.algorithm = OSM_B200_SEG_NARELTH;
      else return fail(OSM_B200_ERR_UNSUPPORTED, "cFunctionalSegments.segmentationAlgorithm = " + segAlgo + " is not supported (relTh, NArelTh, nonX, eqX are)");
      std::vector<double> th;
      if (!segThresh.empty()) for (const auto &kv : segThresh) th.push_back(kv.second);
      else for (const std::string &one : split_list(segThreshList)) th.push_back(num(one));
      if (SG.algorithm == OSM_B200_SEG_RELTH && th.empty()) th.push_back(0.0);       // the field's default value
      if (th.size() > OSM_B200_F_MAX_THRESH) return fail(OSM_B200_ERR_INVALID, "cFunctionalSegments: more than 8 thresholds");
      SG.n_thresholds = (int)th.size();
      for (size_t k = 0; k < th.size(); k++) SG.thresholds[k] = (float)std::min(1.0, std::max(0.0, th[k]));   // :198-207
    }
  }
  P.n_percentile = 0;
  for (const auto &kv : pct) {
    if (P.n_percentile >= OSM_B200_F_MAX_PCTL) return fail(OSM_B200_ERR_INVALID, "cFunctionalPercentiles: more than 8 percentiles");
    P.percentile[P.n_percentile++] = std::min(1.0, std::max(0.0, kv.second));
  }
  P.n_pctlrange = 0;
  if (P.n_percentile > 0)
    for (const auto &kv : pctRange) {
      double a, b;
      if (P.n_pctlrange >= OSM_B200_F_MAX_PCTL || !parse_range(kv.second, a, b)) return fail(OSM_B200_ERR_INVALID, "cFunctionalPercentiles.pctlrange: expected X-Y");
      P.pctlrange[P.n_pctlrange][0] = (int)a; P.pctlrange[P.n_pctlrange][1] = (int)b; P.n_pctlrange++;
    }
  return OSM_B200_OK;
}

// ------------------------------------------------------------------------------------------
// WAV in, HTK / CSV out
// ------------------------------------------------------------------------------------------
// data chunk as it is in the file (interleaved sample frames of `format`, an osm_b200_pcm_format); the device converts
struct Wav { int sampleRate = 0, nChan = 0, format = OSM_B200_PCM_S16, frameBytes = 2; std::vector<unsigned char> pcm;
             size_t frames() const { return pcm.size() / (size_t)frameBytes; } };

// RIFF/WAVE as smilePcm_readWaveHeader accepts it (smileUtil.c:2381-2481): AudioFormat 1 (integer PCM: 8 / 16 / 24 bit, 32-bit
// containers with 24 or 32 valid bits) or 3 (IEEE float, 32 bit); bytes per sample = BlockAlign / NumChannels (:2473)
bool read_wav(const char *path, Wav &w, std::string &err)
{
  FILE *f = fopen(path, "rb");
  if (!f) { err = std::string("cannot open '") + path + "'"; return false; }
  // chunk sizes come from the file: every one is clamped to what the file still holds before anything is allocated
  long fileSize = 0;
  if (fseek(f, 0, SEEK_END) == 0) fileSize = ftell(f);
  if (fileSize < 12 || fseek(f, 0, SEEK_SET) != 0) { fclose(f); err = std::string(path) + ": not a RIFF/WAVE file"; return false; }
  unsigned char h[12];
  if (fread(h, 1, 12, f) != 12 || memcmp(h, "RIFF", 4) || memcmp(h + 8, "WAVE", 4)) { fclose(f); err = std::string(path) + ": not a RIFF/WAVE file"; return false; }
  bool fmtOk = false;
  int bits = 0, fmtTag = 0, blockAlign = 0;
  for (;;) {
    unsigned char ch[8];
    if (fread(ch, 1, 8, f) != 8) break;
    uint32_t sz = ch[4] | (ch[5] << 8) | (ch[6] << 16) | ((uint32_t)ch[7] << 24);
    const long here = ftell(f);
    if (here < 0) break;
    const uint32_t left = (uint32_t)std::min<long>(fileSize - here, 0x7fffffffL);
    if (!memcmp(ch, "fmt ", 4)) {
      if (sz < 16 || sz > left || sz > 4096) break;
      std::vector<unsigned char> b(sz);
      if (fread(b.data(), 1, sz, f) != sz) break;
      fmtTag = b[0] | (b[1] << 8); w.nChan = b[2] | (b[3] << 8);
      w.sampleRate = b[4] | (b[5] << 8) | (b[6] << 16) | (b[7] << 24);
      blockAlign = b[12] | (b[13] << 8);
      bits = b[14] | (b[15] << 8);
      if (w.nChan <= 0 || w.sampleRate <= 0) { fclose(f); err = std::string(path) + ": invalid WAV header (channels / sample rate)"; return false; }
      fmtOk = true;
      if ((sz & 1) && fseek(f, 1, SEEK_CUR) != 0) break;
    } else if (!memcmp(ch, "data", 4)) {
      if (!fmtOk) break;
      if (blockAlign <= 0 || blockAlign % w.nChan != 0) { fclose(f); err = std::string(path) + ": invalid WAV header (block alignment)"; return false; }
      const int bps = blockAlign / w.nChan;
      w.format = -1;
      if (fmtTag == 1 || (fmtTag == 0xFFFE && bits == 16 && bps == 2)) {     // (the extensible tag was accepted for 16-bit files before)
        if (bps == 1) w.format = OSM_B200_PCM_S8;
        else if (bps == 2) w.format = OSM_B200_PCM_S16;
        else if (bps == 3) w.format = OSM_B200_PCM_S24;
        else if (bps == 4 && bits == 24) w.format = OSM_B200_PCM_S24_32;
        else if (bps == 4 && bits == 32) w.format = OSM_B200_PCM_S32;
      } else if (fmtTag == 3 && bps == 4 && bits == 32) w.format = OSM_B200_PCM_F32;
      if (w.format < 0) {
        char b[160];
        snprintf(b, sizeof b, ": unsupported sample format (format tag %d, %d bits, %d bytes per sample); integer PCM 8/16/24/32 bit and 32-bit float are supported", fmtTag, bits, bps);
        fclose(f); err = std::string(path) + b; return false;
      }
      w.frameBytes = blockAlign;
      if (sz == 0 || sz == 0xFFFFFFFFu || sz > left) sz = left;        // streamed files: the data chunk runs to the end of the file
      try { w.pcm.resize(sz); } catch (const std::exception &) { fclose(f); err = std::string(path) + ": out of memory"; return false; }
      const size_t got = fread(w.pcm.data(), 1, sz, f);
      w.pcm.resize(got - got % (size_t)blockAlign);
      fclose(f);
      return true;
    } else {
      if (sz > left || fseek(f, (long)sz + (long)(sz & 1), SEEK_CUR) != 0) break;
    }
  }
  fclose(f);
  err = std::string(path) + ": malformed WAV file";
  return false;
}

// HTK parameter file (iocore/htkSink.cpp:90-106 header, :183-206 rows): big-endian
// `packed` (optional): the payload already in file byte order (sinks.cu: htk_pack_kernel), n * K 32-bit words
bool write_htk(const char *path, const float *rows, int64_t n, int K, double period, int parmKind, std::string &err,
               const uint32_t *packed = nullptr)
{
  FILE *f = fopen(path, "wb");
  if (!f) { err = std::string("cannot write '") + path + "'"; return false; }
  auto be32 = [&](uint32_t v) { unsigned char b[4] = {(unsigned char)(v >> 24), (unsigned char)(v >> 16), (unsigned char)(v >> 8), (unsigned char)v}; fwrite(b, 1, 4, f); };
  auto be16 = [&](uint16_t v) { unsigned char b[2] = {(unsigned char)(v >> 8), (unsigned char)v}; fwrite(b, 1, 2, f); };
  be32((uint32_t)n);
  be32(period <= 0.0 ? 100000u : (uint32_t)round(period * 10000000.0));
  be16((uint16_t)(sizeof(float) * K));
  be16((uint16_t)parmKind);
  if (packed) {
    const bool okw = fwrite(packed, 4, (size_t)n * K, f) == (size_t)n * K;
    if (fclose(f) != 0 || !okw) { err = std::string("write error on '") + path + "'"; return false; }
    return true;
  }
  std::vector<unsigned char> buf((size_t)K * 4);
  for (int64_t r = 0; r < n; r++) {
    for (int k = 0; k < K; k++) {
      uint32_t u;
      memcpy(&u, &rows[r * K + k], 4);
      buf[4 * k] = (unsigned char)(u >> 24); buf[4 * k + 1] = (unsigned char)(u >> 16);
      buf[4 * k + 2] = (unsigned char)(u >> 8); buf[4 * k + 3] = (unsigned char)u;
    }
    fwrite(buf.data(), 1, buf.size(), f);
  }
  const bool bad = ferror(f) != 0;
  if (fclose(f) != 0 || bad) { err = std::string("write error on '") + path + "'"; return false; }
  return true;
}

// ---- number formatting of the text sinks -------------------------------------------------------------------
// The reference prints every value with fprintf("%e") (iocore/csvSink.cpp:216-233, arffSink.cpp:400-420).  At GPU
// rates the sink is the bottleneck, so rows are formatted into a buffer with std::to_chars: for finite values the
// scientific / fixed conversions with an explicit precision produce the correctly rounded decimal expansion of the
// same real number printf sees (float -> double is exact), i.e. the same bytes (tests/test_host_cpu.py checks
// millions of values against printf).  Non-finite values take the printf path.
struct TextBuf {
  FILE *f;
  std::vector<char> b;
  size_t n = 0;
  explicit TextBuf(FILE *fp) : f(fp), b(1 << 20) {}
  void room(size_t need) { if (n + need > b.size()) flush(); if (need > b.size()) b.resize(need * 2); }
  void flush() { if (n && fwrite(b.data(), 1, n, f) != n) failed = true; n = 0; }
  bool failed = false;
  void ch(char c) { room(1); b[n++] = c; }
  void str(const char *s, size_t len) { room(len); memcpy(b.data() + n, s, len); n += len; }
  void str(const std::string &s) { str(s.data(), s.size()); }
  void fmt_e(float v)                       // == fprintf("%e", v)
  {
    room(64);
    if (std::isfinite(v)) {
      auto r = std::to_chars(b.data() + n, b.data() + n + 48, v, std::chars_format::scientific, 6);
      n = (size_t)(r.ptr - b.data());
    } else n += (size_t)snprintf(b.data() + n, 48, "%e", (double)v);
  }
  void fmt_f0(float v)                      // == fprintf("%.0f", v)
  {
    room(64);
    if (std::isfinite(v) && fabsf(v) < 1e15f) {
      auto r = std::to_chars(b.data() + n, b.data() + n + 48, v, std::chars_format::fixed, 0);
      n = (size_t)(r.ptr - b.data());
    } else { char t[400]; const int l = snprintf(t, sizeof t, "%.0f", (double)v); str(t, (size_t)l); }
  }
  void fmt_f6(double v)                     // == fprintf("%f", v)
  {
    char t[400];
    const int l = snprintf(t, sizeof t, "%f", v);
    str(t, (size_t)l);
  }
  void fmt_ld(long v) { room(32); auto r = std::to_chars(b.data() + n, b.data() + n + 24, v); n = (size_t)(r.ptr - b.data()); }
};

// cCsvSink options with the component's defaults (iocore/csvSink.cpp:40-54,78-110)
struct CsvOpts { bool printHeader = true, timestamp = true, number = true; int prname = 0; char delim = ';'; std::string instName; };

// iocore/csvSink.cpp:150-235
// value text of the rows formatted on the device (sinks.cu: csv_format_kernel): row r at text + r * slot, len[r] bytes ending in the
// newline; host[r] != 0: the row holds a value the device left to the host formatter
struct DevText { const char *text; int64_t slot; const int32_t *len; const uint8_t *host; };

// rows [n][K] in HBM formatted on the device (sinks.cu) and brought back: the value text of every row in a slot of its own, its
// length and its host-format flag.  Values separated by `delim`; alwaysE: every value "%e" (cArffSink), otherwise as cCsvSink.
struct HostText {
  std::vector<char> text; std::vector<int32_t> len; std::vector<uint8_t> hostFlag; int64_t slot = 0;
  DevText view() const { return DevText{text.data(), slot, len.data(), hostFlag.data()}; }
};

bool device_text(const float *dRows, int64_t n, int K, char delim, bool alwaysE, HostText &t)
{
  t.slot = osm_b200_device_csv_slot_bytes(K);
  t.text.resize((size_t)n * t.slot + 1); t.len.resize((size_t)n + 1); t.hostFlag.resize((size_t)n + 1);
  if (n == 0) return true;
  osm::DevBuf<char> dText; osm::DevBuf<int32_t> dLen; osm::DevBuf<uint8_t> dHost;
  return dText.reserve_exact((size_t)n * t.slot) == cudaSuccess && dLen.reserve_exact((size_t)n) == cudaSuccess &&
         dHost.reserve_exact((size_t)n) == cudaSuccess &&
         osm_b200_device_format_rows(dRows, n, K, delim, alwaysE, dText.p, t.slot, dLen.p, dHost.p, nullptr) == 0 &&
         cudaMemcpy(t.text.data(), dText.p, (size_t)n * t.slot, cudaMemcpyDeviceToHost) == cudaSuccess &&
         cudaMemcpy(t.len.data(), dLen.p, (size_t)n * 4, cudaMemcpyDeviceToHost) == cudaSuccess &&
         cudaMemcpy(t.hostFlag.data(), dHost.p, (size_t)n, cudaMemcpyDeviceToHost) == cudaSuccess;
}

// rows [n][K] in HBM packed into the HTK payload on the device and brought back into `packed`
bool device_htk(const float *dRows, int64_t n, int K, std::vector<uint32_t> &packed)
{
  packed.resize((size_t)n * K + 1);
  if (n == 0) return true;
  osm::DevBuf<uint32_t> dPack;
  return dPack.reserve_exact((size_t)n * K) == cudaSuccess && osm_b200_device_pack_htk(dRows, n * K, dPack.p, nullptr) == 0 &&
         cudaMemcpy(packed.data(), dPack.p, (size_t)n * K * 4, cudaMemcpyDeviceToHost) == cudaSuccess;
}

// time stamp of row r: min(r, nTimeFrames - 1) rows into the level, whose rows are `period` apart unless the plan says otherwise
// (osm_b200_plan_row_time: cTonefilt rows carry the time of their first sample)
static double row_time(int64_t r, int64_t nTimeFrames, double period, const osm_b200_plan *timePlan)
{
  const int64_t t = (nTimeFrames > 0 && r > nTimeFrames - 1) ? nTimeFrames - 1 : r;
  return timePlan ? osm_b200_plan_row_time(timePlan, t) : (double)t * period;
}

bool write_csv(const char *path, const float *rows, int64_t n, int K, const std::vector<std::string> &names, double period,
               const CsvOpts &o, std::string &err, int64_t nTimeFrames = 0, const DevText *dt = nullptr,
               const osm_b200_plan *timePlan = nullptr)
{
  FILE *f = fopen(path, "w");
  if (!f) { err = std::string("cannot write '") + path + "'"; return false; }
  if (o.printHeader) {
    if (o.prname) fprintf(f, "name%c", o.delim);
    if (o.number) fprintf(f, "frameIndex%c", o.delim);
    if (o.timestamp) fprintf(f, "frameTime%c", o.delim);
    for (int k = 0; k < K - 1; k++) fprintf(f, "%s%c", names[k].c_str(), o.delim);
    fprintf(f, "%s\n", names[K - 1].c_str());
  }
  TextBuf tb(f);
  for (int64_t r = 0; r < n; r++) {
    if (o.prname) {
      tb.ch('\''); tb.str(o.instName);
      if (o.prname == 2) { tb.ch('_'); tb.fmt_ld((long)r); }
      tb.ch('\''); tb.ch(o.delim);
    }
    if (o.number) { tb.fmt_ld((long)r); tb.ch(o.delim); }
    // rows appended by a window processor at the end of input carry a copy of the last frame's time stamp
    if (o.timestamp) { tb.fmt_f6(row_time(r, nTimeFrames, period, timePlan)); tb.ch(o.delim); }
    if (dt && !dt->host[r]) { tb.str(dt->text + r * dt->slot, (size_t)dt->len[r]); continue; }
    for (int k = 0; k < K; k++) {
      const float v = rows[r * K + k];
      if (v == floorf(v)) tb.fmt_f0(v); else tb.fmt_e(v);
      tb.ch(k == K - 1 ? '\n' : o.delim);
    }
  }
  tb.flush();
  const bool bad = tb.failed || ferror(f) != 0;
  if (fclose(f) != 0 || bad) { err = std::string("write error on '") + path + "'"; return false; }
  return true;
}

// cArffSink options (iocore/arffSink.cpp:40-100) and writer (:225-330 header, :337-440 rows)
struct ArffOpts {
  std::string relation = "smile", instName;
  int prname = 0;                      // 1 instanceName, 2 instanceBase_<index>
  bool number = true, timestamp = true, append = false, dummyClass = true;
  double frameTimeAdd = 0.0;
  std::vector<std::pair<std::string, std::string>> classes;   // (name, type); type "" = numeric
  std::vector<std::string> targetAll;                         // per class, already escaped; "" -> NULL
};

std::string arff_escape(const std::string &str)               // iocore/arffSink.cpp:189-232
{
  if (str.empty()) return "''";
  bool quote = false;
  std::string e;
  for (char c : str) {
    switch (c) {
      case '"': case '\'': case '%': case '\\': e += '\\'; e += c; quote = true; break;
      case '\r': e += "\\r"; quote = true; break;
      case '\n': e += "\\n"; quote = true; break;
      case '\t': e += "\\t"; quote = true; break;
      case ' ': case ',': case '{': case '}': e += c; quote = true; break;
      default: e += c;
    }
  }
  return quote ? "'" + e + "'" : e;
}

bool write_arff(const char *path, const float *rows, int64_t n, int K, const std::vector<std::string> &names, double period,
                const ArffOpts &o, std::string &err, int64_t nTimeFrames = 0, const DevText *dt = nullptr,
                const osm_b200_plan *timePlan = nullptr)
{
  bool header = true;
  if (o.append) {                                             // :244-256: append to an existing file without a header
    FILE *t = fopen(path, "r");
    if (t) { fclose(t); header = false; }
  }
  FILE *f = fopen(path, header ? "w" : "a");
  if (!f) { err = std::string("cannot write '") + path + "'"; return false; }
  if (header) {
    fprintf(f, "@relation %s\n\n", arff_escape(o.relation).c_str());
    if (o.prname) fprintf(f, "@attribute name string\n");
    if (o.number) fprintf(f, "@attribute frameIndex numeric\n");
    if (o.timestamp) fprintf(f, "@attribute frameTime numeric\n");
    for (int k = 0; k < K; k++) fprintf(f, "@attribute %s numeric\n", arff_escape(names[k]).c_str());
    if (!o.classes.empty()) {
      for (const auto &c : o.classes) fprintf(f, "@attribute %s %s\n", c.first.c_str(), c.second.empty() ? "numeric" : c.second.c_str());
    } else if (o.dummyClass) {
      fprintf(f, "@attribute class {0,1,2,3}\n");
    }
    fprintf(f, "\n@data\n\n");
  }
  TextBuf tb(f);
  for (int64_t r = 0; r < n; r++) {
    if (o.prname == 1) fprintf(f, "%s,", arff_escape(o.instName).c_str());
    else if (o.prname == 2) { char b[512]; snprintf(b, sizeof b, "%s_%ld", o.instName.c_str(), (long)r); fprintf(f, "%s,", arff_escape(b).c_str()); }
    if (o.number) fprintf(f, "%ld,", (long)r);
    if (o.timestamp) fprintf(f, "%f,", row_time(r, nTimeFrames, period, timePlan) + o.frameTimeAdd);
    if (dt && !dt->host[r]) tb.str(dt->text + r * dt->slot, (size_t)dt->len[r] - 1);   // the device's row text without its newline
    else {
      tb.fmt_e(rows[r * K]);
      for (int k = 1; k < K; k++) { tb.ch(','); tb.fmt_e(rows[r * K + k]); }
    }
    tb.flush();                          // keeps the order with the fprintf calls around it (both end in the FILE buffer)
    if (!o.classes.empty()) {
      for (size_t c = 0; c < o.classes.size(); c++) {
        if (c < o.targetAll.size() && !o.targetAll[c].empty()) fprintf(f, ",%s", o.targetAll[c].c_str());
        else fprintf(f, ",NULL");
      }
    } else if (o.dummyClass) {
      fprintf(f, ",0");
    }
    fputc('\n', f);
  }
  const bool bad = tb.failed || ferror(f) != 0;
  if (fclose(f) != 0 || bad) { err = std::string("write error on '") + path + "'"; return false; }
  return true;
}

}  // namespace

// ------------------------------------------------------------------------------------------
template <auto Destroy> struct Deleter { template <typename T> void operator()(T *p) const { Destroy(p); } };
using PlanPtr = std::unique_ptr<osm_b200_plan, Deleter<osm_b200_plan_destroy>>;
using FuncPtr = std::unique_ptr<osm_b200_functionals, Deleter<osm_b200_functionals_destroy>>;

struct osm_b200_session {
  Conf conf;
  std::vector<osm_b200_component> comps;     // everything except the wave source parameters
  int waveIdx = -1;
  std::string outputLevel;
  int device = 0;
  int parmKind = 9;
  CsvOpts csv;
  ArffOpts arff;
  // plan cache keyed by (sample rate, channels)
  std::map<std::pair<long, int>, PlanPtr> plans;
  osm_b200_plan *cur = nullptr;
  std::vector<osm_b200_component> curComps;
  // a cFunctionals summary between the LLD level and the sink (full-input mode): the plan then produces the functionals'
  // input level, which stays in HBM, and one functionals object per input format summarises it (osm_b200_functionals.h)
  // One instance (the shipped IS09 graph) or several behind a cVectorConcat / multi-level sink reader (ComParE_2016: six instances on
  // column subsets of the LLD rows): the plan's output level is the union of the instances' reader levels.
  bool hasFunc = false;
  // a reader level of an instance: a level of the plan, or the view a cDataSelector (`selected` names + nameAppend) gives of one
  struct FuncReader { std::string level; std::vector<std::string> sel; std::string nameAppend;
                      bool operator==(const FuncReader &o) const { return level == o.level && sel == o.sel && nameAppend == o.nameAppend; } };
  struct FuncInst { osm_b200_functionals_spec spec; std::vector<FuncReader> readers; bool preserveFields = false; };
  std::vector<FuncInst> finsts;              // in the order of their first appearance in the summary row
  // what sits between the cFunctionals levels and the sink (the shipped GeMAPS / eGeMAPS summary graphs): cVectorConcat (any depth),
  // cDataSelector (picks and renames summary values, core/dataSelector.cpp:296-366), cVectorOperation dBp / dBv
  // (other/vectorOperation.cpp:508-527).  All of it works value by value on the summary row, so the instances write their values
  // side by side into a scratch row and one gather pass (osm_b200_summary_assemble_device) produces the sink's row.
  struct SummNode {
    int kind = 0;                            // 0 cFunctionals instance, 1 concat, 2 cDataSelector, 3 cVectorOperation
    int inst = -1;
    std::vector<int> kids;
    std::vector<std::string> sel, newNames;  // cDataSelector
    std::string nameAppend;                  // cDataSelector / cVectorOperation (the operation name when appendOperationToName = 1)
    std::string nameBase;                    // cVectorOperation
    bool copyInputName = true;
    int op = 0; float logfloor = 1e-12f;     // OSM_B200_VOP_*
  };
  std::vector<SummNode> snodes;
  int sroot = -1;
  std::vector<std::string> unionLevels;      // levels of the plan's output level, in order
  struct FuncRt {                            // per input format
    std::vector<FuncPtr> f;
    std::vector<std::vector<int32_t>> cols;  // columns of every instance's input elements inside the plan's rows
    std::vector<std::vector<std::string>> inNames;
    std::vector<PlanPtr> desc;               // description-only plan over the instance's reader levels (its frame-count rule); null = the main plan
    std::vector<int> off;                    // first value of every instance inside the scratch row
    int scratch = 0;                         // values per scratch row (all instances side by side)
    std::vector<std::string> names;          // the sink's row
    int total = 0;
    bool identity = true;                    // the sink's row is the scratch row
    std::vector<int32_t> gSrc, gOp; std::vector<float> gFloor;
    PlanPtr sum;                             // with an LLD part: the summary's own plan description (frame counts, period); null = the main plan
    PlanPtr lld;                             // the LLD part's plan description (its row counts, names, period, time stamps); null = none
    std::vector<int64_t> lldCols;            // its columns inside the plan's rows
    std::vector<std::string> lldNames;
  };
  std::map<std::pair<long, int>, FuncRt> funcs;
  FuncRt *curFunc = nullptr;
  osm::DevBuf<float> dFuncOut, dFuncScratch;
  // osm_b200_session_extract_device: the LLD rows a summary configuration's plan leaves for its cFunctionals instances, and the
  // end of the last call's work on its stream (the next call, on whatever stream, starts behind it: the buffers are reused)
  osm::DevBuf<float> dLldRows;
  osm::CudaEvent evDevice;
  // sinks that read a summary level and an LLD level (choose_output_level): the LLD sink's level and its parts, which the plan's union
  // level holds next to the summary's inputs, the options of the sinks reading it, and its rows gathered out of the union rows
  std::string lldLevel;
  std::vector<std::string> lldLevels;
  std::vector<std::string> lldSources;       // the levels its rows are taken from: a cVectorConcat level as the levels it joins when
                                             // the summary's inputs hold them all, otherwise the level itself
  CsvOpts lldCsv;
  ArffOpts lldArff;
  int lldParmKind = 9;
  std::vector<int64_t> lldMeta;              // {columns, union row offsets, LLD row offsets} of the last gather, uploaded to dLldMeta
  osm::DevBuf<int64_t> dLldMeta;
  osm::DevBuf<float> dLldOut;                // extract_files: the gathered LLD rows

  // plans and functionals select their own device, the buffers above need it; a session without plans has made no CUDA call
  ~osm_b200_session() { if (device >= 0 && !plans.empty()) cudaSetDevice(device); }
};

static osm_b200_status get_plan(osm_b200_session *s, double sampleRate, int nChan, osm_b200_plan **out, int format = OSM_B200_PCM_S16)
{
  const auto key = std::make_pair((long)lround(sampleRate * 1000.0), nChan + 4096 * format);
  auto it = s->plans.find(key);
  if (it == s->plans.end()) {
    std::vector<osm_b200_component> cs = s->comps;
    cs[s->waveIdx].u.wavesource.sampleRate = sampleRate;
    cs[s->waveIdx].u.wavesource.nChannels = nChan;
    cs[s->waveIdx].u.wavesource.format = format;
    osm_b200_plan *p = nullptr;
    osm_b200_status st = osm_b200_plan_create(cs.data(), (int)cs.size(), s->outputLevel.c_str(), s->device, &p);
    if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    it = s->plans.emplace(key, PlanPtr(p)).first;
    s->curComps = cs;
  }
  s->cur = it->second.get();
  *out = it->second.get();
  return OSM_B200_OK;
}

// description-only plan (names, counts, frame rules) of the session's graph with `levels` as output level, several levels read
// through a concat named `concat` (_unionconcat: every level keeps its own length)
static osm_b200_status desc_plan(osm_b200_session *s, double sampleRate, int nChan, const std::vector<std::string> &levels, PlanPtr &out,
                                 const char *concat = "_fconcat")
{
  std::vector<osm_b200_component> cs;
  for (const osm_b200_component &c : s->comps) if (strcmp(c.name, "_sinkconcat") != 0 && strcmp(c.name, "_unionconcat") != 0) cs.push_back(c);
  int wave = -1;
  for (size_t i = 0; i < cs.size(); i++) if (cs[i].type == OSM_B200_C_WAVESOURCE) wave = (int)i;
  cs[wave].u.wavesource.sampleRate = sampleRate;
  cs[wave].u.wavesource.nChannels = nChan;
  std::string lvl = levels[0];
  if (levels.size() > 1) {
    if (levels.size() > OSM_B200_MAX_INPUTS) return hfail(OSM_B200_ERR_UNSUPPORTED, "more than 8 levels in one reader");
    osm_b200_component c;
    osm_b200_component_defaults(OSM_B200_C_VECTORCONCAT, &c);
    snprintf(c.name, sizeof c.name, "%s", concat);
    for (const std::string &l : levels) snprintf(c.reader_dmLevel[c.n_inputs++], OSM_B200_NAME_LEN, "%s", l.c_str());
    snprintf(c.writer_dmLevel, sizeof c.writer_dmLevel, "%s", concat);
    c.u.vectorconcat.processArrayFields = 0;
    cs.push_back(c);
    lvl = concat;
  }
  osm_b200_plan *p = nullptr;
  const osm_b200_status st = osm_b200_plan_create(cs.data(), (int)cs.size(), lvl.c_str(), -1, &p);
  out.reset(p);
  return st == OSM_B200_OK ? OSM_B200_OK : hfail(st, osm_b200_last_error());
}

// one value of the sink's summary row: where it is in the scratch row, the operation applied to it, and its name
struct SummEl { int src; int op; float fl; std::string name; };

// the values summary node ni appends to `out`, over the instances' values in rt.f (their scratch row offsets rt.off)
static bool eval_summary(const osm_b200_session *s, const osm_b200_session::FuncRt &rt, int ni, std::vector<SummEl> &out, std::string &err)
{
  const osm_b200_session::SummNode &nd = s->snodes[(size_t)ni];
  if (nd.kind == 0) {
    const int n = osm_b200_functionals_num_elements(rt.f[(size_t)nd.inst].get());
    for (int j = 0; j < n; j++) out.push_back(SummEl{rt.off[(size_t)nd.inst] + j, OSM_B200_VOP_COPY, 0.f, osm_b200_functionals_element_name(rt.f[(size_t)nd.inst].get(), j)});
    return true;
  }
  std::vector<SummEl> in;
  for (int k : nd.kids) if (!eval_summary(s, rt, k, in, err)) return false;
  if (nd.kind == 1) { out.insert(out.end(), in.begin(), in.end()); return true; }
  if (nd.kind == 2) {                                               // core/dataSelector.cpp:296-366 (elementMode)
    for (size_t k = 0; k < nd.sel.size(); k++) {
      const SummEl *hit = nullptr;
      for (const SummEl &e : in) if (e.name == nd.sel[k]) { hit = &e; break; }
      if (!hit) { err = "cDataSelector: element '" + nd.sel[k] + "' not found in the summary levels it reads"; return false; }
      SummEl e = *hit;
      if (k < nd.newNames.size() && !nd.newNames[k].empty()) e.name = nd.newNames[k];
      else if (!nd.nameAppend.empty()) e.name += "_" + nd.nameAppend;
      out.push_back(e);
    }
    return true;
  }
  for (SummEl e : in) {                                             // other/vectorOperation.cpp:226-249 + core/dataProcessor.cpp:250-269
    if (e.op != OSM_B200_VOP_COPY) { err = "chained cVectorOperation instances behind cFunctionals are not supported"; return false; }
    const std::string base = !nd.nameBase.empty() ? nd.nameBase : e.name;
    if (!nd.nameAppend.empty()) e.name = (nd.copyInputName && !base.empty()) ? base + "_" + nd.nameAppend : nd.nameAppend;
    else e.name = (nd.copyInputName && !base.empty()) ? base : std::string("noname");
    e.op = nd.op; e.fl = nd.logfloor;
    out.push_back(e);
  }
  return true;
}

// the levels of the plan's output level: the summary's inputs, then the parts of the LLD sink's level not among them
static std::vector<std::string> plan_levels(const osm_b200_session *s)
{
  std::vector<std::string> v = s->unionLevels;
  for (const std::string &l : s->lldSources) if (std::find(v.begin(), v.end(), l) == v.end()) v.push_back(l);
  return v;
}

// the functionals objects of the session for one input format; device < 0: names / counts only
static osm_b200_status build_func_rt(osm_b200_session *s, double sampleRate, int nChan, osm_b200_plan *p, int device, osm_b200_session::FuncRt &rt)
{
  const int K = osm_b200_plan_num_elements(p);
  // columns of every level of the plan's output level
  std::map<std::string, std::pair<int, int>> range;
  const std::vector<std::string> levels = plan_levels(s);
  if (levels.size() == 1) range[levels[0]] = {0, K};
  else {
    int o = 0;
    for (const std::string &l : levels) {
      PlanPtr d;
      osm_b200_status st = desc_plan(s, sampleRate, nChan, {l}, d);
      if (st != OSM_B200_OK) return st;
      const int n = osm_b200_plan_num_elements(d.get());
      range[l] = {o, n};
      o += n;
    }
    if (o != K) return hfail(OSM_B200_ERR_INVALID, "cFunctionals: the levels of the summary's inputs do not add up to the plan's row");
  }
  rt.total = 0; rt.scratch = 0;
  if (!s->lldLevels.empty()) {
    // the LLD sink reads its levels' columns, with the row count of its own reader (the min over its levels); the summary keeps the
    // frame counts and period of the plan it would have on its own
    osm_b200_status st = desc_plan(s, sampleRate, nChan, s->unionLevels, rt.sum, "_unionconcat");
    if (st == OSM_B200_OK) st = desc_plan(s, sampleRate, nChan, s->lldLevels, rt.lld);
    if (st != OSM_B200_OK) return st;
    for (const std::string &l : s->lldSources)
      for (int c = 0; c < range[l].second; c++) rt.lldCols.push_back(range[l].first + c);
    if ((int)rt.lldCols.size() != osm_b200_plan_num_elements(rt.lld.get()))
      return hfail(OSM_B200_ERR_INVALID, "the LLD sink's levels do not add up to its row");
    for (int k = 0; k < (int)rt.lldCols.size(); k++) {
      rt.lldNames.push_back(osm_b200_plan_element_name(rt.lld.get(), k));
      if (rt.lldNames.back() != osm_b200_plan_element_name(p, (int)rt.lldCols[(size_t)k]))
        return hfail(OSM_B200_ERR_INVALID, "the LLD sink's row is not the concatenation of the levels it is taken from");
    }
  }
  const osm_b200_plan *sp = rt.sum ? rt.sum.get() : p;
  for (const osm_b200_session::FuncInst &fi : s->finsts) {
    std::vector<int32_t> cols;
    std::vector<std::string> inNames;
    std::vector<std::string> plain;                                    // the levels behind the readers (frame-count rule)
    for (const osm_b200_session::FuncReader &rd : fi.readers) {
      const auto r = range[rd.level];
      plain.push_back(rd.level);
      if (rd.sel.empty()) {
        for (int c = 0; c < r.second; c++) { cols.push_back(r.first + c); inNames.push_back(osm_b200_plan_element_name(p, r.first + c)); }
      } else {
        // cDataSelector (core/dataSelector.cpp:296-366, elementMode): the selected elements in the order of `selected`
        for (const std::string &want : rd.sel) {
          int hit = -1;
          for (int c = 0; c < r.second && hit < 0; c++) if (want == osm_b200_plan_element_name(p, r.first + c)) hit = r.first + c;
          if (hit < 0) return hfail(OSM_B200_ERR_INVALID, "cDataSelector: element '" + want + "' not found in level '" + rd.level + "'");
          cols.push_back(hit);
          inNames.push_back(rd.nameAppend.empty() ? want : want + "_" + rd.nameAppend);
        }
      }
    }
    std::vector<const char *> names(cols.size());
    for (size_t i = 0; i < cols.size(); i++) names[i] = inNames[i].c_str();
    osm_b200_functionals *fp = nullptr;
    osm_b200_status st = osm_b200_functionals_create(&fi.spec, (int)cols.size(), names.data(), osm_b200_plan_frame_period(sp), device, &fp);
    FuncPtr f(fp);
    if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    PlanPtr d;
    if (plain != s->unionLevels || rt.sum) {
      st = desc_plan(s, sampleRate, nChan, plain, d, plain == s->unionLevels ? "_unionconcat" : "_fconcat");
      if (st != OSM_B200_OK) return st;
    }
    // preserveFields = 1 keeps the field structure of the input (functionals.cpp:133-137); for single-element fields that is the
    // same row, which is all the shipped graphs ask for (eGeMAPSv02_core.func.conf.inc:14-19)
    if (fi.preserveFields && cols.size() != 1)
      return hfail(OSM_B200_ERR_UNSUPPORTED, "cFunctionals.preserveFields=1 on more than one input element is not supported");
    rt.off.push_back(rt.scratch);
    rt.scratch += osm_b200_functionals_num_elements(f.get());
    rt.f.push_back(std::move(f)); rt.cols.push_back(cols); rt.desc.push_back(std::move(d));
  }
  // the sink's row: walk the summary graph over the instances' values
  std::vector<SummEl> els;
  std::string err;
  if (!eval_summary(s, rt, s->sroot, els, err)) return hfail(OSM_B200_ERR_INVALID, err);
  if (els.empty()) return hfail(OSM_B200_ERR_INVALID, "the summary level has no elements");
  rt.total = (int)els.size();
  rt.identity = rt.total == rt.scratch;
  for (size_t k = 0; k < els.size(); k++) {
    rt.names.push_back(els[k].name); rt.gSrc.push_back(els[k].src); rt.gOp.push_back(els[k].op); rt.gFloor.push_back(els[k].fl);
    if (els[k].src != (int)k || els[k].op != OSM_B200_VOP_COPY) rt.identity = false;
  }
  if (!rt.identity && rt.total > OSM_B200_SUMMARY_MAX_OUT) return hfail(OSM_B200_ERR_UNSUPPORTED, "a re-ordered / transformed summary row of more than OSM_B200_SUMMARY_MAX_OUT values is not supported");
  return OSM_B200_OK;
}

static osm_b200_status get_func(osm_b200_session *s, double sampleRate, int nChan, osm_b200_plan *p, osm_b200_session::FuncRt **out)
{
  const auto key = std::make_pair((long)lround(sampleRate * 1000.0), nChan);      // names / counts do not depend on the sample format
  auto it = s->funcs.find(key);
  if (it == s->funcs.end()) {
    osm_b200_session::FuncRt rt;
    osm_b200_status st = build_func_rt(s, sampleRate, nChan, p, s->device, rt);
    if (st != OSM_B200_OK) return st;
    it = s->funcs.emplace(key, std::move(rt)).first;
  }
  s->curFunc = &it->second;
  *out = &it->second;
  return OSM_B200_OK;
}

// ------------------------------------------------------------------------------------------
// osm_b200_session_open, pass by pass; the first error wins
// ------------------------------------------------------------------------------------------
// cCsvSink options (iocore/csvSink.cpp:40-54,78-110)
static osm_b200_status read_csv_opts(const Section &sec, CsvOpts &o)
{
  o = CsvOpts();
  if (const std::string *x = sec.get("printHeader")) o.printHeader = inum(*x) != 0;
  if (const std::string *x = sec.get("timestamp")) o.timestamp = inum(*x) == 1;
  if (const std::string *x = sec.get("frameTime")) o.timestamp = inum(*x) == 1;
  if (const std::string *x = sec.get("number")) o.number = inum(*x) == 1;
  if (const std::string *x = sec.get("frameIndex")) o.number = inum(*x) == 1;
  if (const std::string *x = sec.get("instanceBase")) { o.instName = *x; o.prname = 2; }
  if (const std::string *x = sec.get("instanceName")) { o.instName = *x; o.prname = 1; }
  if (const std::string *x = sec.get("frameLength")) if (inum(*x) == 1) return hfail(OSM_B200_ERR_UNSUPPORTED, "cCsvSink.frameLength=1 is not supported");
  if (const std::string *x = sec.get("delimChar")) if (!x->empty()) o.delim = *x == "<space>" ? ' ' : (*x == "<tab>" ? '\t' : (*x)[0]);
  return OSM_B200_OK;
}

// cArffSink options (iocore/arffSink.cpp:40-170)
static osm_b200_status read_arff_opts(const Section &sec, ArffOpts &a)
{
  a = ArffOpts();
  if (const std::string *x = sec.get("relation")) a.relation = *x;
  if (const std::string *x = sec.get("append")) a.append = inum(*x) != 0;
  if (const std::string *x = sec.get("number")) a.number = inum(*x) == 1;
  if (const std::string *x = sec.get("frameIndex")) a.number = inum(*x) == 1;
  if (const std::string *x = sec.get("timestamp")) a.timestamp = inum(*x) == 1;
  if (const std::string *x = sec.get("frameTime")) a.timestamp = inum(*x) == 1;
  if (const std::string *x = sec.get("frameTimeAdd")) a.frameTimeAdd = num(*x);
  if (const std::string *x = sec.get("printDefaultClassDummyAttribute")) a.dummyClass = inum(*x) != 0;
  if (const std::string *x = sec.get("frameLength")) if (inum(*x) == 1) return hfail(OSM_B200_ERR_UNSUPPORTED, "cArffSink.frameLength=1 is not supported");
  if (const std::string *x = sec.get("instanceBase")) if (!x->empty() && *x != "-") { a.instName = *x; a.prname = 2; }
  if (const std::string *x = sec.get("instanceName")) if (!x->empty() && *x != "-") { a.instName = *x; a.prname = 1; }
  for (int c = 0; c < 64; c++) {                       // class[c].name / class[c].type, target[c].all (:112-170)
    char key[64];
    snprintf(key, sizeof key, "class[%d].name", c);
    const std::string *nm = sec.get(key);
    snprintf(key, sizeof key, "class[%d].type", c);
    const std::string *ty = sec.get(key);
    if (!nm && !ty) break;
    a.classes.push_back({nm ? *nm : std::string("class"), ty ? *ty : std::string("numeric")});
    snprintf(key, sizeof key, "target[%d].all", c);
    const std::string *tg = sec.get(key);
    a.targetAll.push_back(tg ? (*tg == "?" ? *tg : arff_escape(*tg)) : std::string());
    snprintf(key, sizeof key, "target[%d].instance[0]", c);
    if (sec.get(key)) return hfail(OSM_B200_ERR_UNSUPPORTED, "cArffSink.target[].instance[] is not supported");
  }
  return OSM_B200_OK;
}

// pass 2: the instances listed in [componentInstances:cComponentManager] (core/componentManager.cpp:840-957) -> the compute
// sections in order, the levels the active sinks read, and the sinks' options
static osm_b200_status read_instances(osm_b200_session *s, std::vector<const Section *> &compute, std::vector<std::string> &sinkLevels)
{
  std::map<std::string, const Section *> secOf;
  for (const auto &sec : s->conf.sections) if (sec.type != "cComponentManager") secOf[sec.name] = &sec;
  bool csvLocked = false, arffLocked = false;
  static const std::set<std::string> hostTypes = {"cDataMemory", "cHtkSink", "cCsvSink", "cArffSink", "cExternalSink", "cNullSink", "cDatadumpSink"};
  for (const auto &inst : s->conf.instances) {
    const std::string &name = inst.first, &type = inst.second;
    const Section *sec = secOf.count(name) ? secOf[name] : nullptr;
    if (sec && sec->type != type) return hfail(OSM_B200_ERR_INVALID, "instance '" + name + "' is declared as " + type + " but configured as " + sec->type);
    if (hostTypes.count(type)) {
      if (!sec || (type != "cHtkSink" && type != "cCsvSink" && type != "cArffSink" && type != "cExternalSink")) continue;
      const std::string *fn = sec->get("filename");
      const bool active = type == "cExternalSink" || (fn && *fn != "?" && !fn->empty());
      const std::string *lv = sec->get("reader.dmLevel");
      if (active && lv) sinkLevels.push_back(*lv);
      if (type == "cArffSink" && active && !arffLocked) {
        arffLocked = true;
        if (osm_b200_status st = read_arff_opts(*sec, s->arff); st != OSM_B200_OK) return st;
      }
      if (type == "cHtkSink") { if (const std::string *pk = sec->get("parmKind")) s->parmKind = inum(*pk); }
      // CSV formatting options: those of the active CSV sink; without one (explicit csv paths over the API),
      // those of the last cCsvSink section
      if (type == "cCsvSink" && !csvLocked) {
        csvLocked = active;
        if (osm_b200_status st = read_csv_opts(*sec, s->csv); st != OSM_B200_OK) return st;
      }
      continue;
    }
    if (!sec) return hfail(OSM_B200_ERR_INVALID, "instance '" + name + "' (" + type + ") has no configuration section");
    compute.push_back(sec);
  }
  return OSM_B200_OK;
}

static bool is_summary_level(osm_b200_session *s, const std::map<std::string, const Section *> &writerOf, const std::string &level);

// pass 3: the output level: explicit, or the level the active sinks read; a multi-level sink reader is an
// implicit concat (core/dataReader.cpp:360-444)
static osm_b200_status choose_output_level(osm_b200_session *s, const char *output_level, const std::vector<std::string> &sinkLevels,
                                           const std::map<std::string, const Section *> &writerOf)
{
  std::string &lvl = s->outputLevel;
  lvl = output_level ? output_level : "";
  if (!lvl.empty()) return OSM_B200_OK;
  if (sinkLevels.empty()) return hfail(OSM_B200_ERR_INVALID, "no active sink: pass output_level or enable a sink (-O / -csvoutput)");
  lvl = sinkLevels[0];
  // every active sink gets the rows of ONE plan run.  Sinks of two levels are served together when one is a summary level and the
  // other is not: the plan's union level then holds the LLD sink's level next to the summary's inputs
  std::set<std::string> distinct(sinkLevels.begin(), sinkLevels.end());
  for (const std::string &l : sinkLevels) {
    if (l == lvl) continue;
    const bool sumFirst = is_summary_level(s, writerOf, lvl), sumOther = is_summary_level(s, writerOf, l);
    if (distinct.size() != 2 || sumFirst == sumOther)
      return hfail(OSM_B200_ERR_UNSUPPORTED, "the active sinks read different levels ('" + lvl + "' and '" + l + "'): enable the sinks of one level per session");
    s->lldLevel = sumFirst ? l : lvl;
    lvl = sumFirst ? lvl : l;
    break;
  }
  return OSM_B200_OK;
}

// the options of the sinks that read `level`, by the rules of read_instances: CSV / ARFF those of the first active sink of the
// type (CSV: of the last cCsvSink section without one), HTK the parmKind of the last cHtkSink section
static osm_b200_status read_level_sink_opts(const osm_b200_session *s, const std::string &level, CsvOpts &csv, ArffOpts &arff, int &parmKind)
{
  std::map<std::string, const Section *> secOf;
  for (const auto &sec : s->conf.sections) if (sec.type != "cComponentManager") secOf[sec.name] = &sec;
  bool csvLocked = false, arffLocked = false;
  for (const auto &inst : s->conf.instances) {
    const Section *sec = secOf.count(inst.first) ? secOf[inst.first] : nullptr;
    const std::string *lv = sec ? sec->get("reader.dmLevel") : nullptr;
    if (!lv || *lv != level) continue;
    const std::string *fn = sec->get("filename");
    const bool active = fn && *fn != "?" && !fn->empty();
    if (inst.second == "cArffSink" && active && !arffLocked) {
      arffLocked = true;
      if (osm_b200_status st = read_arff_opts(*sec, arff); st != OSM_B200_OK) return st;
    }
    if (inst.second == "cHtkSink") { if (const std::string *pk = sec->get("parmKind")) parmKind = inum(*pk); }
    if (inst.second == "cCsvSink" && !csvLocked) {
      csvLocked = active;
      if (osm_b200_status st = read_csv_opts(*sec, csv); st != OSM_B200_OK) return st;
    }
  }
  return OSM_B200_OK;
}

// a cDataSelector section (core/dataSelector.cpp:296-366, elementMode): the element names it selects, the new names it gives
// them, the text it appends to their names, and the first field the summary path does not model ("" if there is none)
struct Selector { std::vector<std::string> sel, newNames; std::string nameAppend, unsupported; bool renames = false; };

static Selector read_selector(const Section &ds)
{
  Selector r;
  std::map<int, std::string> selIdx, newIdx;
  std::string selList, newList;
  for (const auto &kv : ds.kv) {
    const std::string &f = kv.first;
    if (f == "nameAppend") { r.nameAppend = kv.second; continue; }
    if (is_common(f) || f == "reader.dmLevel" || f == "writer.dmLevel") continue;
    if (f == "selected") selList = kv.second;
    else if (f.compare(0, 9, "selected[") == 0) selIdx[atoi(f.c_str() + 9)] = kv.second;
    else if (f == "newNames") { newList = kv.second; r.renames = true; }
    else if (f.compare(0, 9, "newNames[") == 0) { newIdx[atoi(f.c_str() + 9)] = kv.second; r.renames = true; }
    else if (r.unsupported.empty() && (f != "elementMode" || inum(kv.second) != 1)) r.unsupported = f;
  }
  if (!selIdx.empty()) for (const auto &kv : selIdx) r.sel.push_back(trim(kv.second));
  else r.sel = split_list(selList);
  if (!newIdx.empty()) {
    r.newNames.assign(r.sel.size(), "");
    for (const auto &kv : newIdx) if (kv.first >= 0 && (size_t)kv.first < r.newNames.size()) r.newNames[(size_t)kv.first] = trim(kv.second);
  } else r.newNames = split_list(newList);
  return r;
}

static bool summary_glue(const std::string &type) { return type == "cVectorConcat" || type == "cDataSelector" || type == "cVectorOperation"; }

// pass 4: the summary graph behind the output level -- cFunctionals levels below cVectorConcat (any depth), cDataSelector and
// cVectorOperation nodes.  Fills the session's finsts, snodes, sroot and unionLevels (the instances' reader levels, which the
// plan computes; the summaries then run on the resident rows, functionals.cu, each instance on its columns).
struct SummaryBuilder {
  osm_b200_session &s;
  const std::map<std::string, const Section *> &writerOf;      // level -> the compute section that writes it
  std::map<const Section *, int> instOf;                       // cFunctionals section -> its index in s.finsts
  osm_b200_status status = OSM_B200_OK;
  std::string msg;

  int fail(osm_b200_status st, const std::string &m) { status = st; msg = m; return -1; }

  bool has_functionals(const std::string &level, int depth) const
  {
    auto it = writerOf.find(level);
    if (it == writerOf.end() || depth > 16) return false;
    const Section &w = *it->second;
    if (w.type == "cFunctionals") return true;
    const std::string *r = w.get("reader.dmLevel");
    if (!summary_glue(w.type) || !r) return false;
    for (const std::string &l : split_list(*r)) if (has_functionals(l, depth + 1)) return true;
    return false;
  }

  // the instance of cFunctionals section w, added on first use; -1 on error
  int add_instance(const Section &w)
  {
    auto it = instOf.find(&w);
    if (it != instOf.end()) return it->second;
    osm_b200_session::FuncInst fi;
    std::string err;
    if (osm_b200_status st = to_functionals(w, fi.spec, err); st != OSM_B200_OK) return fail(st, err);
    if (const std::string *x = w.get("preserveFields")) fi.preserveFields = inum(*x) != 0;
    const std::string *r = w.get("reader.dmLevel");
    if (!r) return fail(OSM_B200_ERR_INVALID, "cFunctionals '" + w.name + "' has no reader.dmLevel");
    for (const std::string &l : split_list(*r)) {
      osm_b200_session::FuncReader rd;
      rd.level = l;
      // a cDataSelector that only picks named elements (and appends to their names) is a view of its input level
      auto itw = writerOf.find(l);
      if (itw != writerOf.end() && itw->second->type == "cDataSelector") {
        Selector sel = read_selector(*itw->second);
        const std::string *base = itw->second->get("reader.dmLevel");
        if (sel.unsupported.empty() && !sel.renames && base && base->find(';') == std::string::npos && !sel.sel.empty()) {
          rd.level = trim(*base);
          rd.sel = std::move(sel.sel);
          rd.nameAppend = sel.nameAppend;
        }
      }
      fi.readers.push_back(rd);
      if (std::find(s.unionLevels.begin(), s.unionLevels.end(), rd.level) == s.unionLevels.end()) s.unionLevels.push_back(rd.level);
    }
    s.finsts.push_back(fi);
    return instOf[&w] = (int)s.finsts.size() - 1;
  }

  // the node of s.snodes that produces `level`; -1 on error
  int build_node(const std::string &level, int depth)
  {
    auto it = writerOf.find(level);
    if (it == writerOf.end() || depth > 16) return fail(OSM_B200_ERR_INVALID, "level '" + level + "' has no writer");
    const Section &w = *it->second;
    osm_b200_session::SummNode nd;
    if (w.type == "cFunctionals") {
      nd.kind = 0;
      nd.inst = add_instance(w);
      if (nd.inst < 0) return -1;
      s.snodes.push_back(nd);
      return (int)s.snodes.size() - 1;
    }
    const std::string *r = w.get("reader.dmLevel");
    if (!r || !summary_glue(w.type))
      return fail(OSM_B200_ERR_UNSUPPORTED, "a level that mixes cFunctionals summaries with other levels is not supported (level '" + level + "')");
    const std::vector<std::string> rl = split_list(*r);
    for (const std::string &l : rl) { const int k = build_node(l, depth + 1); if (k < 0) return -1; nd.kids.push_back(k); }
    if (w.type == "cVectorConcat") {
      // summary levels hold single-element fields: a cVectorConcat that keeps only array fields (its default) would be empty
      nd.kind = 1;
      int paf = 1, incl = 0;
      if (const std::string *x = w.get("processArrayFields")) paf = inum(*x);
      if (const std::string *x = w.get("includeSingleElementFields")) incl = inum(*x);
      if (paf == 1 && !incl && rl.size() > 1)
        return fail(OSM_B200_ERR_UNSUPPORTED, "cVectorConcat '" + w.name + "' behind cFunctionals drops single-element fields (includeSingleElementFields = 0)");
    } else if (w.type == "cDataSelector") {
      nd.kind = 2;
      Selector sel = read_selector(w);
      if (sel.unsupported == "elementMode") return fail(OSM_B200_ERR_UNSUPPORTED, "cDataSelector.elementMode=0 is not supported");
      if (!sel.unsupported.empty()) return fail(OSM_B200_ERR_UNSUPPORTED, "cDataSelector '" + w.name + "': field '" + sel.unsupported + "' is not supported");
      if (sel.sel.empty()) return fail(OSM_B200_ERR_INVALID, "cDataSelector '" + w.name + "': no elements selected");
      nd.sel = std::move(sel.sel);
      nd.newNames = std::move(sel.newNames);
      nd.nameAppend = sel.nameAppend;
    } else {
      nd.kind = 3;                                                  // other/vectorOperation.cpp:42-48,136-139,210-222
      std::string opn = "norm";
      int appendOp = 0;
      double lf = 1e-12;                                            // default of `logfloor`
      for (const auto &kv : w.kv) {
        const std::string &f = kv.first;
        if (f == "nameAppend") { nd.nameAppend = kv.second; continue; }
        if (f == "copyInputName") { nd.copyInputName = inum(kv.second) != 0; continue; }
        if (is_common(f) || f == "reader.dmLevel" || f == "writer.dmLevel") continue;
        if (f == "operation") opn = kv.second;
        else if (f == "nameBase") nd.nameBase = kv.second;
        else if (f == "appendOperationToName") appendOp = inum(kv.second);
        else if (f == "logfloor") lf = atof(kv.second.c_str());
        else if (f == "processArrayFields" || f == "includeSingleElementFields" || f == "param1" || f == "param2" || f == "powOnlyPos") continue;
        else return fail(OSM_B200_ERR_UNSUPPORTED, "cVectorOperation '" + w.name + "': field '" + f + "' is not supported");
      }
      if (opn.compare(0, 3, "dBp") == 0) nd.op = OSM_B200_VOP_DBP;
      else if (opn.compare(0, 3, "dBv") == 0) nd.op = OSM_B200_VOP_DBV;
      else return fail(OSM_B200_ERR_UNSUPPORTED, "cVectorOperation behind cFunctionals: only operation = dBp / dBv is supported (got '" + opn + "')");
      if (appendOp) nd.nameAppend = opn;                             // overrides nameAppend (:210-216, :240-243)
      if (lf <= 0) lf = 0.000000000001;                              // :219-223
      nd.logfloor = (float)lf;
      if (rl.size() != 1) return fail(OSM_B200_ERR_UNSUPPORTED, "cVectorOperation must read exactly one level");
    }
    s.snodes.push_back(nd);
    return (int)s.snodes.size() - 1;
  }
};

// a level (or a multi-level reader's `a;b`) with cFunctionals behind it
static bool is_summary_level(osm_b200_session *s, const std::map<std::string, const Section *> &writerOf, const std::string &level)
{
  const SummaryBuilder b{*s, writerOf};
  for (const std::string &pl : split_list(level)) if (b.has_functionals(pl, 0)) return true;
  return false;
}

// pass 4 on the output level: with cFunctionals behind it, the output level becomes the union of the instances' reader levels, and
// of the LLD sink's levels when sinks read both
static osm_b200_status build_summary(osm_b200_session *s, const std::map<std::string, const Section *> &writerOf)
{
  SummaryBuilder b{*s, writerOf};
  const std::vector<std::string> parts = split_list(s->outputLevel);
  if (!is_summary_level(s, writerOf, s->outputLevel)) return OSM_B200_OK;
  osm_b200_session::SummNode root;
  root.kind = 1;
  for (const std::string &pl : parts) {
    const int k = b.build_node(pl, 0);
    if (k < 0) return hfail(b.status, b.msg);
    root.kids.push_back(k);
  }
  if (parts.size() == 1) s->sroot = root.kids[0];
  else { s->snodes.push_back(root); s->sroot = (int)s->snodes.size() - 1; }
  if (s->unionLevels.size() > OSM_B200_MAX_INPUTS) return hfail(OSM_B200_ERR_UNSUPPORTED, "cFunctionals: more than 8 input levels in total");
  s->hasFunc = true;
  if (!s->lldLevel.empty()) {
    s->lldLevels = split_list(s->lldLevel);
    for (const std::string &l : s->lldLevels) {
      auto it = writerOf.find(l);
      const std::string *r = (it != writerOf.end() && it->second->type == "cVectorConcat") ? it->second->get("reader.dmLevel") : nullptr;
      std::vector<std::string> src = r ? split_list(*r) : std::vector<std::string>();
      bool held = !src.empty();
      for (const std::string &x : src) held = held && std::find(s->unionLevels.begin(), s->unionLevels.end(), x) != s->unionLevels.end();
      if (held) s->lldSources.insert(s->lldSources.end(), src.begin(), src.end());
      else s->lldSources.push_back(l);
    }
    osm_b200_status st = read_level_sink_opts(s, s->outputLevel, s->csv, s->arff, s->parmKind);
    if (st == OSM_B200_OK) st = read_level_sink_opts(s, s->lldLevel, s->lldCsv, s->lldArff, s->lldParmKind);
    if (st != OSM_B200_OK) return st;
  }
  s->outputLevel.clear();
  for (const std::string &l : plan_levels(s)) s->outputLevel += (s->outputLevel.empty() ? "" : ";") + l;
  return OSM_B200_OK;
}

// pass 5: only the components the output level depends on are part of the plan: the shipped feature-set
// configurations carry sinks and summaries (cFunctionals ...) that stay idle when their output file is
// not requested (filename = ?), exactly like the reference leaves those sinks unwritten.
static osm_b200_status lower_sections(osm_b200_session *s, const std::vector<const Section *> &compute,
                                      const std::map<std::string, const Section *> &writerOf)
{
  std::set<const Section *> need;
  std::vector<std::string> todo = split_list(s->outputLevel);
  todo.insert(todo.end(), s->lldLevels.begin(), s->lldLevels.end());     // the LLD part's own plan description reads them
  while (!todo.empty()) {
    const std::string l = todo.back();
    todo.pop_back();
    auto it = writerOf.find(l);
    if (it == writerOf.end() || need.count(it->second)) continue;
    need.insert(it->second);
    for (const char *key : {"reader.dmLevel", "reader2.dmLevel", "F0reader.dmLevel"})
      if (const std::string *r = it->second->get(key))
        for (const std::string &more : split_list(*r)) todo.push_back(more);
  }
  for (const Section *sec : compute) {
    const bool isWave = sec->type == "cWaveSource" || sec->type == "cExternalAudioSource";
    if (!isWave && !need.count(sec)) continue;
    osm_b200_component c;
    std::string err;
    if (!to_component(*sec, c, err)) return hfail(type_of(sec->type) < 0 ? OSM_B200_ERR_UNSUPPORTED : OSM_B200_ERR_INVALID, err);
    if (c.type == OSM_B200_C_WAVESOURCE) s->waveIdx = (int)s->comps.size();
    s->comps.push_back(c);
  }
  if (s->waveIdx < 0) return hfail(OSM_B200_ERR_INVALID, "the configuration has no cWaveSource / cExternalAudioSource");
  return OSM_B200_OK;
}

// pass 6: an output level of several levels is read through one concat component
static osm_b200_status add_reader_concat(osm_b200_session *s)
{
  if (s->outputLevel.find(';') == std::string::npos) return OSM_B200_OK;
  const std::vector<std::string> levels = split_list(s->outputLevel);
  if (levels.size() > OSM_B200_MAX_INPUTS) return hfail(OSM_B200_ERR_UNSUPPORTED, "more than 8 levels in one reader");
  osm_b200_component c;
  osm_b200_component_defaults(OSM_B200_C_VECTORCONCAT, &c);
  // the union of the input levels of several cFunctionals instances keeps every level's own length (graph.cpp: padRows)
  const char *cname = (s->hasFunc && levels.size() > 1) ? "_unionconcat" : "_sinkconcat";
  snprintf(c.name, sizeof c.name, "%s", cname);
  for (const std::string &l : levels) snprintf(c.reader_dmLevel[c.n_inputs++], OSM_B200_NAME_LEN, "%s", l.c_str());
  snprintf(c.writer_dmLevel, sizeof c.writer_dmLevel, "%s", cname);
  c.u.vectorconcat.processArrayFields = 0;     // a reader's level concatenation keeps every field
  s->comps.push_back(c);
  s->outputLevel = cname;
  return OSM_B200_OK;
}

// pass 7: validate the graph now (description-only plan at a nominal format) so that errors surface at open
static osm_b200_status validate(osm_b200_session *s)
{
  std::vector<osm_b200_component> cs = s->comps;
  cs[s->waveIdx].u.wavesource.sampleRate = 16000;
  cs[s->waveIdx].u.wavesource.nChannels = 1;
  osm_b200_plan *p = nullptr;
  osm_b200_status st = osm_b200_plan_create(cs.data(), (int)cs.size(), s->outputLevel.c_str(), -1, &p);
  const PlanPtr plan(p);
  if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
  if (!s->hasFunc) return OSM_B200_OK;
  // the summary is taken at the first end-of-input tick; how many cTonefilt rows exist then (its last, padded block is
  // written only after end of input) is not modelled
  for (const osm_b200_component &c : cs)
    if (c.type == OSM_B200_C_TONEFILT)
      return hfail(OSM_B200_ERR_UNSUPPORTED, std::string("cFunctionals reading a level behind cTonefilt '") + c.name + "' is not supported");
  osm_b200_session::FuncRt rt;
  return build_func_rt(s, 16000, 1, p, -1, rt);
}

extern "C" {

// no exception crosses the C boundary (host allocation failures while the configuration is read and lowered)
osm_b200_status osm_b200_session_open(const char *conf_path, int32_t n_opts, const char *const *opt_names,
                                      const char *const *opt_values, const char *output_level, int32_t device,
                                      osm_b200_session **session)
try {
  if (!conf_path || !session) return hfail(OSM_B200_ERR_INVALID, "null argument");
  *session = nullptr;
  std::map<std::string, std::string> given;
  for (int i = 0; i < n_opts; i++) if (opt_names && opt_names[i]) given[opt_names[i]] = (opt_values && opt_values[i]) ? opt_values[i] : "";
  auto s = std::make_unique<osm_b200_session>();
  s->device = device;
  std::string err;
  int curSec = -1;
  g_herr.clear();
  if (!parse_file(conf_path, s->conf, given, err, curSec)) return hfail(OSM_B200_ERR_INVALID, err);
  std::vector<const Section *> compute;
  std::vector<std::string> sinkLevels;
  osm_b200_status st = read_instances(s.get(), compute, sinkLevels);
  std::map<std::string, const Section *> writerOf;
  for (const Section *sec : compute) if (const std::string *w = sec->get("writer.dmLevel")) writerOf[*w] = sec;
  if (st == OSM_B200_OK) st = choose_output_level(s.get(), output_level, sinkLevels, writerOf);
  if (st == OSM_B200_OK) st = build_summary(s.get(), writerOf);
  if (st == OSM_B200_OK) st = lower_sections(s.get(), compute, writerOf);
  if (st == OSM_B200_OK) st = add_reader_concat(s.get());
  if (st == OSM_B200_OK) st = validate(s.get());
  if (st != OSM_B200_OK) return st;
  *session = s.release();
  return OSM_B200_OK;
} catch (const std::bad_alloc &) { return hfail(OSM_B200_ERR_NOMEM, "out of host memory"); }
catch (const std::exception &e) { return hfail(OSM_B200_ERR_INVALID, e.what()); }

void osm_b200_session_close(osm_b200_session *s)
{
  if (!s) return;
  delete s;
}

int32_t osm_b200_session_num_elements(osm_b200_session *s, double sampleRate, int32_t nChan)
{
  if (!s) return 0;
  osm_b200_plan *p;
  if (get_plan(s, sampleRate, nChan, &p) != OSM_B200_OK) return 0;
  if (s->hasFunc) {
    osm_b200_session::FuncRt *f;
    if (get_func(s, sampleRate, nChan, p, &f) != OSM_B200_OK) return 0;
    return f->total;
  }
  return osm_b200_plan_num_elements(p);
}

const char *osm_b200_session_element_name(osm_b200_session *s, int32_t idx)
{
  if (s && s->hasFunc) return (s->curFunc && idx >= 0 && idx < s->curFunc->total) ? s->curFunc->names[idx].c_str() : nullptr;
  return (s && s->cur) ? osm_b200_plan_element_name(s->cur, idx) : nullptr;
}

int32_t osm_b200_session_components(osm_b200_session *s, double sampleRate, int32_t nChan, const osm_b200_component **comps,
                                    const char **outputLevel)
{
  if (!s) return 0;
  s->curComps = s->comps;
  s->curComps[s->waveIdx].u.wavesource.sampleRate = sampleRate;
  s->curComps[s->waveIdx].u.wavesource.nChannels = nChan;
  if (comps) *comps = s->curComps.data();
  if (outputLevel) *outputLevel = s->outputLevel.c_str();
  return (int32_t)s->curComps.size();
}

osm_b200_status osm_b200_session_plan(osm_b200_session *s, double sampleRate, int32_t nChan, osm_b200_plan **plan)
{
  if (!s || !plan) return hfail(OSM_B200_ERR_INVALID, "null argument");
  return get_plan(s, sampleRate, nChan, plan);
}

// a padded device batch (osm_b200_session_extract_device): its samples, stride and lengths, and the stream its work goes to
struct DeviceBatch { const void *pcm; int64_t stride; const int64_t *lengths; cudaStream_t stream; };
// the LLD part of a call on a session whose sinks read a summary and an LLD level: its frame offsets (n_utt + 1 entries, filled) and
// a device buffer of at least maxRows rows for its rows (NULL: the offsets only)
struct LldOut { int64_t *frameOff; float *dOut; int64_t maxRows; };

// the LLD sink's rows out of the union rows the plan left in HBM (rows [lldOff[u], ...) of utterance u, K values each): its columns,
// the first lo.frameOff[u + 1] - lo.frameOff[u] rows of every utterance, on `stream`
static osm_b200_status gather_lld(osm_b200_session *s, const osm_b200_session::FuncRt &f, const float *dRows, int K, const int64_t *lldOff,
                                  int32_t nUtt, const LldOut &lo, cudaStream_t stream)
{
  const size_t nc = f.lldCols.size();
  s->lldMeta.assign(f.lldCols.begin(), f.lldCols.end());
  s->lldMeta.insert(s->lldMeta.end(), lldOff, lldOff + nUtt);
  s->lldMeta.insert(s->lldMeta.end(), lo.frameOff, lo.frameOff + nUtt + 1);
  // a copy from pageable memory is staged before cudaMemcpyAsync returns; lldMeta is not touched again before the next call
  if (s->dLldMeta.reserve(s->lldMeta.size()) != cudaSuccess ||
      cudaMemcpyAsync(s->dLldMeta.p, s->lldMeta.data(), s->lldMeta.size() * sizeof(int64_t), cudaMemcpyHostToDevice, stream) != cudaSuccess ||
      osm_b200_device_gather_rows(dRows, K, s->dLldMeta.p, (int32_t)nc, nUtt, lo.frameOff[nUtt], lo.dOut, stream) != 0)
    return hfail(OSM_B200_ERR_CUDA, std::string("gather of the LLD rows: ") + cudaGetErrorString(cudaGetLastError()));
  return OSM_B200_OK;
}

// Both extract entry points: packed PCM in host memory with `out` in host memory (dev == NULL: the plan's pipelined host run, the
// summary on the null stream, then a copy to `out`), or a padded device batch with `out` in device memory (every launch on
// dev->stream; the host waits on that stream only where it needs device data or hands it host data: the Viterbi lags, the
// cPitchJitter flag, the cFunctionals instances' row offsets and counts).
static osm_b200_status osm_b200_session_extract_pcm_impl(osm_b200_session *s, const void *pcm, const int64_t *uttOff, int32_t nUtt,
                                             double sampleRate, int32_t nChan, int64_t *frameOff, float *out, int64_t maxRows,
                                             int format = OSM_B200_PCM_S16, const DeviceBatch *dev = nullptr, const LldOut *lld = nullptr)
{
  if (!s || !uttOff || !frameOff) return hfail(OSM_B200_ERR_INVALID, "null argument");
  const cudaStream_t stream = dev ? dev->stream : nullptr;
  osm_b200_plan *p;
  osm_b200_status st = get_plan(s, sampleRate, nChan, &p, format);
  if (st != OSM_B200_OK) return st;
  if (s->hasFunc) {
    // one summary row per utterance that has frames; the rows a plan run leaves in HBM are summarised in place.  The
    // contour of utterance u = its first osm_b200_plan_num_frames_first_eoi() rows (what the reference's functionals see).
    osm_b200_session::FuncRt *f;
    st = get_func(s, sampleRate, nChan, p, &f);
    if (st != OSM_B200_OK) return st;
    const size_t nI = f->f.size();
    std::vector<int64_t> lldOff((size_t)nUtt + 1), rowOff((size_t)nUtt);
    std::vector<std::vector<int64_t>> nRows(nI, std::vector<int64_t>((size_t)nUtt));
    st = osm_b200_plan_frame_offsets(p, uttOff, nUtt, lldOff.data());
    if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    // the rows the summary's own plan would hold (with an LLD part the union holds more levels)
    std::vector<int64_t> sumOff;
    if (f->sum) {
      sumOff.resize((size_t)nUtt + 1);
      st = osm_b200_plan_frame_offsets(f->sum.get(), uttOff, nUtt, sumOff.data());
      if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    }
    const std::vector<int64_t> &capOff = f->sum ? sumOff : lldOff;
    if (lld) {
      if (!f->lld) return hfail(OSM_B200_ERR_INVALID, "the session's active sinks read one level: it has no LLD part");
      st = osm_b200_plan_frame_offsets(f->lld.get(), uttOff, nUtt, lld->frameOff);
      if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    }
    std::vector<int> live;
    frameOff[0] = 0;
    for (int u = 0; u < nUtt; u++) {
      // every instance sees the rows its own reader holds when end of input is first signalled; a summary row exists when
      // every instance has at least one frame
      bool all = true;
      for (size_t i = 0; i < nI; i++) {
        const int64_t n = std::min<int64_t>(osm_b200_plan_num_frames_first_eoi(f->desc[i] ? f->desc[i].get() : p, uttOff[u + 1] - uttOff[u]), capOff[u + 1] - capOff[u]);
        nRows[i][live.size()] = n;
        all = all && n > 0;
      }
      if (all) { rowOff[live.size()] = lldOff[u]; live.push_back(u); }
      frameOff[u + 1] = frameOff[u] + (all ? 1 : 0);
    }
    const int64_t nLld = lld ? lld->frameOff[nUtt] : 0;
    if (!out && !(lld && lld->dOut)) return OSM_B200_OK;
    if (frameOff[nUtt] > maxRows) return hfail(OSM_B200_ERR_INVALID, "output buffer too small");
    if (lld && (nLld > lld->maxRows || (nLld > 0 && !lld->dOut))) return hfail(OSM_B200_ERR_INVALID, "LLD output buffer too small");
    if (live.empty() && nLld == 0) return OSM_B200_OK;
    const float *dRows = nullptr;
    if (dev) {
      if (s->dLldRows.reserve((size_t)lldOff[(size_t)nUtt] * osm_b200_plan_num_elements(p)) != cudaSuccess)
        return hfail(OSM_B200_ERR_NOMEM, "out of device memory (LLD rows)");
      st = osm_b200_plan_run_device_padded(p, dev->pcm, dev->stride, dev->lengths, nUtt, lldOff.data(), s->dLldRows.p, stream);
      if (st == OSM_B200_OK) st = osm_b200_plan_check_device_flags(p, stream);
      dRows = s->dLldRows.p;
    } else {
      st = osm_b200_plan_run_host_resident(p, pcm, uttOff, nUtt, lldOff.data(), &dRows);
    }
    if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    if (nLld > 0 && (st = gather_lld(s, *f, dRows, osm_b200_plan_num_elements(p), lldOff.data(), nUtt, *lld, stream)) != OSM_B200_OK) return st;
    if (live.empty()) return OSM_B200_OK;
    // levels behind the SHS pitch chain: their length at the first end-of-input tick follows the Viterbi level's (data dependent)
    {
      std::vector<int32_t> lag((size_t)nUtt, -1);
      st = dev ? osm_b200_plan_copy_seq_lag_stream(p, lag.data(), nUtt, stream) : osm_b200_plan_copy_seq_lag(p, lag.data(), nUtt);
      if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
      for (size_t k = 0; k < live.size(); k++) {
        const int u = live[k];
        if (lag[u] < 0) continue;
        for (size_t i = 0; i < nI; i++)
          nRows[i][k] = std::max<int64_t>(0, std::min<int64_t>(osm_b200_plan_num_frames_first_eoi_v(f->desc[i] ? f->desc[i].get() : p, uttOff[u + 1] - uttOff[u], lag[u]),
                                                               capOff[u + 1] - capOff[u]));
      }
    }
    const int KF = f->total, KS = f->scratch;
    const size_t need = live.size() * (size_t)KF;
    float *dInst = nullptr;                                            // where the instances write: the sink's row or the scratch row
    if (!f->identity) {
      const size_t needS = live.size() * (size_t)KS;
      if (s->dFuncScratch.reserve_exact(needS) != cudaSuccess) return hfail(OSM_B200_ERR_NOMEM, "out of device memory (functionals scratch rows)");
      dInst = s->dFuncScratch.p;
    }
    // the sink's rows: the caller's device buffer, or the session's, copied to the caller's host buffer below
    float *dSink = out;
    if (!dev) {
      if (s->dFuncOut.reserve_exact(need) != cudaSuccess) return hfail(OSM_B200_ERR_NOMEM, "out of device memory (functionals rows)");
      dSink = s->dFuncOut.p;
    }
    for (size_t i = 0; i < nI; i++) {
      st = osm_b200_functionals_run_device_cols(f->f[i].get(), dRows, osm_b200_plan_num_elements(p), f->cols[i].data(), rowOff.data(), nRows[i].data(),
                                                (int)live.size(), (dInst ? dInst : dSink) + f->off[i], KS, stream);
      if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    }
    if (dInst) {
      st = osm_b200_summary_assemble_device(dInst, KS, f->gSrc.data(), f->gOp.data(), f->gFloor.data(), KF, (int64_t)live.size(), dSink, KF, stream);
      if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
    }
    if (!dev && cudaMemcpy(out, s->dFuncOut.p, need * sizeof(float), cudaMemcpyDeviceToHost) != cudaSuccess) return hfail(OSM_B200_ERR_CUDA, "copy of the functionals rows failed");
    return OSM_B200_OK;
  }
  st = osm_b200_plan_frame_offsets(p, uttOff, nUtt, frameOff);
  if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
  if (!out) return OSM_B200_OK;
  if (frameOff[nUtt] > maxRows) return hfail(OSM_B200_ERR_INVALID, "output buffer too small");
  if (dev) {
    st = osm_b200_plan_run_device_padded(p, dev->pcm, dev->stride, dev->lengths, nUtt, frameOff, out, stream);
    if (st == OSM_B200_OK) st = osm_b200_plan_check_device_flags(p, stream);
  } else {
    st = osm_b200_plan_run_host(p, pcm, uttOff, nUtt, frameOff, out);
  }
  if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
  return OSM_B200_OK;
}

// The host-memory entry points reuse the plans and buffers whose last osm_b200_session_extract_device work may still be in flight on
// its stream: they start after it.
static osm_b200_status after_device_calls(osm_b200_session *s)
{
  if (s && s->evDevice && (cudaSetDevice(s->device) != cudaSuccess || cudaEventSynchronize(s->evDevice) != cudaSuccess))
    return hfail(OSM_B200_ERR_CUDA, std::string("waiting for the last extract_device call: ") + cudaGetErrorString(cudaGetLastError()));
  return OSM_B200_OK;
}

osm_b200_status osm_b200_session_extract_pcm(osm_b200_session *s, const int16_t *pcm, const int64_t *uttOff, int32_t nUtt,
                                             double sampleRate, int32_t nChan, int64_t *frameOff, float *out, int64_t maxRows)
{
  // no exception crosses the C boundary (allocation failures on hostile inputs, std::filesystem / stream errors)
  try {
    osm_b200_status st = after_device_calls(s);
    return st != OSM_B200_OK ? st : osm_b200_session_extract_pcm_impl(s, pcm, uttOff, nUtt, sampleRate, nChan, frameOff, out, maxRows);
  }
  catch (const std::bad_alloc &) { return hfail(OSM_B200_ERR_NOMEM, "out of host memory"); }
  catch (const std::exception &e) { return hfail(OSM_B200_ERR_INVALID, e.what()); }
}

static osm_b200_status extract_device(osm_b200_session *s, const void *d_pcm, int32_t pcm_format, int64_t stride, const int64_t *lengths,
                                      int32_t n_utt, double sample_rate, int32_t n_channels, int64_t *frame_offsets_out, float *d_out,
                                      int64_t max_rows, void *stream, const LldOut *lld)
try {
  if (!s || !lengths || !frame_offsets_out || n_utt < 0) return hfail(OSM_B200_ERR_INVALID, "null argument");
  if (pcm_format != OSM_B200_PCM_S16 && pcm_format != OSM_B200_PCM_F32)
    return hfail(OSM_B200_ERR_INVALID, "pcm_format must be OSM_B200_PCM_S16 (int16) or OSM_B200_PCM_F32 (float32)");
  std::vector<int64_t> uttOff((size_t)n_utt + 1, 0);
  for (int u = 0; u < n_utt; u++) {
    if (lengths[u] < 0 || lengths[u] > stride)
      return hfail(OSM_B200_ERR_INVALID, "utterance " + std::to_string(u) + ": length " + std::to_string(lengths[u]) + " outside 0 .. stride (" +
                                             std::to_string(stride) + ")");
    uttOff[(size_t)u + 1] = uttOff[(size_t)u] + lengths[u];
  }
  const DeviceBatch dev{d_pcm, stride, lengths, reinterpret_cast<cudaStream_t>(stream)};
  // the row-count query touches no device; a run starts behind the previous call's work and marks the end of its own
  const bool run = (d_out || (lld && lld->dOut)) && s->device >= 0;
  if (run && (cudaSetDevice(s->device) != cudaSuccess || (s->evDevice && cudaStreamWaitEvent(dev.stream, s->evDevice, 0) != cudaSuccess)))
    return hfail(OSM_B200_ERR_CUDA, std::string("extract_device: ") + cudaGetErrorString(cudaGetLastError()));
  const osm_b200_status st = osm_b200_session_extract_pcm_impl(s, nullptr, uttOff.data(), n_utt, sample_rate, n_channels, frame_offsets_out,
                                                               d_out, max_rows, pcm_format, &dev, lld);
  if (run && ((!s->evDevice && s->evDevice.create(cudaEventDisableTiming) != cudaSuccess) || cudaEventRecord(s->evDevice, dev.stream) != cudaSuccess))
    return hfail(OSM_B200_ERR_CUDA, std::string("extract_device: ") + cudaGetErrorString(cudaGetLastError()));
  return st;
} catch (const std::bad_alloc &) { return hfail(OSM_B200_ERR_NOMEM, "out of host memory"); }
catch (const std::exception &e) { return hfail(OSM_B200_ERR_INVALID, e.what()); }

osm_b200_status osm_b200_session_extract_device(osm_b200_session *s, const void *d_pcm, int32_t pcm_format, int64_t stride,
                                                const int64_t *lengths, int32_t n_utt, double sample_rate, int32_t n_channels,
                                                int64_t *frame_offsets_out, float *d_out, int64_t max_rows, void *stream)
{
  return extract_device(s, d_pcm, pcm_format, stride, lengths, n_utt, sample_rate, n_channels, frame_offsets_out, d_out, max_rows, stream, nullptr);
}

osm_b200_status osm_b200_session_extract_device_lld(osm_b200_session *s, const void *d_pcm, int32_t pcm_format, int64_t stride,
                                                    const int64_t *lengths, int32_t n_utt, double sample_rate, int32_t n_channels,
                                                    int64_t *frame_offsets_out, float *d_out, int64_t max_rows,
                                                    int64_t *lld_frame_offsets_out, float *d_lld_out, int64_t max_lld_rows, void *stream)
{
  if (!lld_frame_offsets_out) return hfail(OSM_B200_ERR_INVALID, "null argument");
  const LldOut lld{lld_frame_offsets_out, d_lld_out, max_lld_rows};
  return extract_device(s, d_pcm, pcm_format, stride, lengths, n_utt, sample_rate, n_channels, frame_offsets_out, d_out, max_rows, stream, &lld);
}

int32_t osm_b200_session_lld_num_elements(osm_b200_session *s, double sampleRate, int32_t nChan)
{
  if (!s || !s->hasFunc) return 0;
  osm_b200_plan *p;
  osm_b200_session::FuncRt *f;
  if (get_plan(s, sampleRate, nChan, &p) != OSM_B200_OK || get_func(s, sampleRate, nChan, p, &f) != OSM_B200_OK) return 0;
  return (int32_t)f->lldNames.size();
}

const char *osm_b200_session_lld_element_name(osm_b200_session *s, int32_t idx)
{
  return (s && s->curFunc && idx >= 0 && (size_t)idx < s->curFunc->lldNames.size()) ? s->curFunc->lldNames[(size_t)idx].c_str() : nullptr;
}

osm_b200_status osm_b200_session_extract_files(osm_b200_session *s, int32_t n, const char *const *wavPaths,
                                               const char *const *htkPaths, const char *const *csvPaths, int64_t *framesOut)
{
  return osm_b200_session_extract_files_arff(s, n, wavPaths, htkPaths, csvPaths, nullptr, framesOut);
}

extern "C++" {
// run fn(i) for i = 0 .. n-1 on up to `maxThreads` host threads (file reading / formatting: at GPU rates the sinks are the
// bottleneck of a file-based run); returns the first error
template <class Fn>
static bool parallel_files(int n, Fn fn, std::string &err, bool serial = false)
{
  unsigned hw = std::thread::hardware_concurrency();
  int nt = (int)std::min<unsigned>(hw ? hw : 4u, 32u);
  if (const char *e = getenv("OSM_B200_IO_THREADS")) nt = std::max(1, atoi(e));
  nt = std::min(nt, n);
  if (serial) nt = 1;
  std::atomic<int> next(0);
  std::atomic<bool> failed(false);
  std::mutex mu;
  auto worker = [&]() {
    for (;;) {
      const int i = next.fetch_add(1);
      if (i >= n || failed.load()) return;
      std::string e;
      if (!fn(i, e)) { std::lock_guard<std::mutex> lk(mu); if (!failed.exchange(true)) err = e; return; }
    }
  };
  if (nt <= 1) { worker(); return !failed.load(); }
  std::vector<std::thread> th;
  for (int t = 0; t < nt; t++) th.emplace_back(worker);
  for (auto &t : th) t.join();
  return !failed.load();
}

// the options of the sinks of one level, and the plan whose row times their time stamps are
struct SinkOpts { const CsvOpts &csv; const ArffOpts &arff; int parmKind; const osm_b200_plan *timePlan; };

// the sinks of one batch: rows [fo[k], fo[k+1]) of file idx[k] -> its HTK / CSV / ARFF files, files in parallel
static bool write_batch(const SinkOpts &o, const std::vector<int> &idx, const int64_t *fo, const int64_t *nTime, const float *rows, int K,
                        const std::vector<std::string> &names, double period, const char *const *htkPaths, const char *const *csvPaths,
                        const char *const *arffPaths, int64_t *framesOut, std::string &err, const DevText *dt = nullptr,
                        const uint32_t *packed = nullptr, const DevText *dtArff = nullptr)
{
  // several inputs may name the same output file (cArffSink / cCsvSink with append=1 collect every input in one file):
  // those files must be written one after the other, in input order
  bool shared = false;
  {
    std::set<std::string> seen;
    for (const char *const *paths : {htkPaths, csvPaths, arffPaths})
      if (paths)
        for (int i : idx)
          if (paths[i] && !seen.insert(std::string(paths[i])).second) shared = true;
  }
  return parallel_files((int)idx.size(), [&](int k, std::string &e) -> bool {
    const int i = idx[k];
    const float *r = rows + (size_t)fo[k] * K;
    const int64_t nr = fo[k + 1] - fo[k];
    if (framesOut) framesOut[i] = nr;
    if (htkPaths && htkPaths[i] && !write_htk(htkPaths[i], r, nr, K, period, o.parmKind, e, packed ? packed + (size_t)fo[k] * K : nullptr)) return false;
    DevText dk;
    if (dt) dk = DevText{dt->text + fo[k] * dt->slot, dt->slot, dt->len + fo[k], dt->host + fo[k]};
    if (csvPaths && csvPaths[i] && !write_csv(csvPaths[i], r, nr, K, names, period, o.csv, e, nTime[k], dt ? &dk : nullptr, o.timePlan)) return false;
    DevText da;
    if (dtArff) da = DevText{dtArff->text + fo[k] * dtArff->slot, dtArff->slot, dtArff->len + fo[k], dtArff->host + fo[k]};
    if (arffPaths && arffPaths[i] && !write_arff(arffPaths[i], r, nr, K, names, period, o.arff, e, nTime[k], dtArff ? &da : nullptr, o.timePlan)) return false;
    return true;
  }, err, shared);
}
}  // extern "C++"

osm_b200_status osm_b200_session_extract_files_arff(osm_b200_session *s, int32_t n, const char *const *wavPaths,
                                                    const char *const *htkPaths, const char *const *csvPaths,
                                                    const char *const *arffPaths, int64_t *framesOut)
{
  return osm_b200_session_extract_files_lld(s, n, wavPaths, htkPaths, csvPaths, arffPaths, nullptr, nullptr, nullptr, framesOut);
}

// the rows [n][K] of one level in HBM -> their CSV / ARFF value text and HTK payload, formatted on the device, and the rows themselves
// in host memory; false on a CUDA error
static bool device_sink_rows(const float *dRows, int64_t n, int K, bool wantCsv, char csvDelim, bool wantArff, bool wantHtk,
                             std::vector<float> &rows, HostText &csv, HostText &arff, std::vector<uint32_t> &packed)
{
  return cudaMemcpy(rows.data(), dRows, (size_t)n * K * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess &&
         (!wantCsv || device_text(dRows, n, K, csvDelim, false, csv)) &&
         (!wantArff || device_text(dRows, n, K, ',', true, arff)) && (!wantHtk || device_htk(dRows, n, K, packed));
}

// no exception crosses the C boundary (allocation failures on hostile inputs, std::filesystem / stream errors)
osm_b200_status osm_b200_session_extract_files_lld(osm_b200_session *s, int32_t n, const char *const *wavPaths,
                                                   const char *const *htkPaths, const char *const *csvPaths, const char *const *arffPaths,
                                                   const char *const *lldHtkPaths, const char *const *lldCsvPaths,
                                                   const char *const *lldArffPaths, int64_t *framesOut)
try {
  if (!s || !wavPaths || n < 0) return hfail(OSM_B200_ERR_INVALID, "null argument");
  const bool wantLld = lldHtkPaths || lldCsvPaths || lldArffPaths;
  if (wantLld && s->lldLevel.empty()) return hfail(OSM_B200_ERR_INVALID, "LLD paths given, but the session's active sinks read one level: it has no LLD part");
  if (osm_b200_status st = after_device_calls(s); st != OSM_B200_OK) return st;
  // files of one call are grouped by (sample rate, channels); each group is one batched plan run
  std::vector<Wav> wavs(n);
  std::string err;
  if (!parallel_files(n, [&](int i, std::string &e) { return read_wav(wavPaths[i], wavs[i], e); }, err)) return hfail(OSM_B200_ERR_INVALID, err);
  // Inputs that share an output file (append-mode ARFF / CSV) must reach it in input order: within one group write_batch does
  // that; when such a batch mixes formats, every input becomes its own group, taken in input order (one plan run each).
  bool sharedAcross = false;
  {
    std::map<std::string, std::pair<int, int>> owner;                 // path -> (rate, channels/format) of its first writer
    for (const char *const *paths : {htkPaths, csvPaths, arffPaths, lldHtkPaths, lldCsvPaths, lldArffPaths})
      if (paths)
        for (int i = 0; i < n; i++) {
          if (!paths[i]) continue;
          const std::pair<int, int> key{wavs[i].sampleRate, wavs[i].nChan + 4096 * wavs[i].format};
          auto it = owner.find(paths[i]);
          if (it == owner.end()) owner[paths[i]] = key; else if (it->second != key) sharedAcross = true;
        }
  }
  std::vector<std::pair<std::pair<int, int>, std::vector<int>>> groups;
  if (sharedAcross) for (int i = 0; i < n; i++) groups.push_back({{wavs[i].sampleRate, wavs[i].nChan + 4096 * wavs[i].format}, {i}});
  else {
    std::map<std::pair<int, int>, std::vector<int>> byFormat;
    for (int i = 0; i < n; i++) byFormat[{wavs[i].sampleRate, wavs[i].nChan + 4096 * wavs[i].format}].push_back(i);
    for (auto &g : byFormat) groups.push_back({g.first, g.second});
  }
  for (auto &g : groups) {
    const int sr = g.first.first, nc = g.first.second % 4096, fmt = g.first.second / 4096;
    std::vector<int64_t> off(g.second.size() + 1, 0), fo(g.second.size() + 1, 0), nTime(g.second.size(), 0);
    size_t total = 0;
    for (size_t k = 0; k < g.second.size(); k++) { total += wavs[g.second[k]].pcm.size(); off[k + 1] = off[k] + (int64_t)wavs[g.second[k]].frames(); }
    std::vector<unsigned char> pcm(total + 16);
    size_t at = 0;
    for (int idx : g.second) { memcpy(pcm.data() + at, wavs[idx].pcm.data(), wavs[idx].pcm.size()); at += wavs[idx].pcm.size(); }
    osm_b200_plan *p;
    osm_b200_status st = get_plan(s, sr, nc, &p, fmt);
    if (st != OSM_B200_OK) return st;
    const int nG = (int)g.second.size();
    int K = 0;
    std::vector<float> rows;
    std::vector<std::string> names;
    // Device sinks (sinks.cu): the rows stay in HBM after the plan run, the CSV value text and the HTK payload are produced there
    // and copied next to the float rows; the host threads add the per-row prefixes and write.  OSM_B200_DEVICE_SINKS=0: host formatting.
    static const bool devSinks = [] { const char *e = getenv("OSM_B200_DEVICE_SINKS"); return !(e && e[0] == '0'); }();
    const bool wantCsv = csvPaths != nullptr, wantHtk = htkPaths != nullptr, wantArff = arffPaths != nullptr;
    bool devText = false;
    HostText csv, arff;                                     // cArffSink: every value "%e", ',' between them (iocore/arffSink.cpp:300-312)
    std::vector<uint32_t> packed;
    if (s->hasFunc) {
      // a summary configuration (cFunctionals behind the sink's level): one row per input that has frames, as the reference's sinks
      // write it -- instance name, time stamp 0 (the summary's segment starts at 0), the values
      osm_b200_session::FuncRt *f;
      st = get_func(s, sr, nc, p, &f);
      if (st != OSM_B200_OK) return st;
      K = f->total;
      names = f->names;
      rows.resize((size_t)nG * K + 1);
      // the LLD sink's rows of the same plan run: gathered on the device, formatted there as for an LLD-only session, and written by
      // write_batch with the options of the sinks that read its level
      std::vector<int64_t> lfo(wantLld ? (size_t)nG + 1 : 0), lTime(wantLld ? (size_t)nG : 0);
      LldOut lo{lfo.data(), nullptr, 0};
      if (wantLld) {
        st = osm_b200_plan_frame_offsets(f->lld.get(), off.data(), nG, lfo.data());
        if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
        lo.maxRows = lfo[(size_t)nG];
        if (s->dLldOut.reserve((size_t)lo.maxRows * f->lldCols.size() + 1) != cudaSuccess) return hfail(OSM_B200_ERR_NOMEM, "out of device memory (LLD rows)");
        lo.dOut = s->dLldOut.p;
      }
      st = osm_b200_session_extract_pcm_impl(s, pcm.data(), off.data(), nG, sr, nc, fo.data(), rows.data(), nG, fmt, nullptr, wantLld ? &lo : nullptr);
      if (st != OSM_B200_OK) return st;
      for (int k = 0; k < nG; k++) nTime[k] = fo[k + 1] - fo[k];
      if (wantLld) {
        const int KL = (int)f->lldCols.size();
        const int64_t nR = lfo[(size_t)nG];
        std::vector<float> lrows((size_t)nR * KL + 1);
        HostText lcsv, larff;
        std::vector<uint32_t> lpacked;
        const bool lText = devSinks && nR > 0;
        if (nR > 0 && !(lText ? device_sink_rows(s->dLldOut.p, nR, KL, lldCsvPaths, s->lldCsv.delim, lldArffPaths, lldHtkPaths, lrows, lcsv, larff, lpacked)
                              : cudaMemcpy(lrows.data(), s->dLldOut.p, (size_t)nR * KL * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess))
          return hfail(OSM_B200_ERR_CUDA, std::string("device sinks: ") + cudaGetErrorString(cudaGetLastError()));
        for (int k = 0; k < nG; k++) lTime[k] = osm_b200_plan_num_time_frames(f->lld.get(), off[k + 1] - off[k]);
        const DevText dt = lcsv.view(), dtA = larff.view();
        if (!write_batch(SinkOpts{s->lldCsv, s->lldArff, s->lldParmKind, f->lld.get()}, g.second, lfo.data(), lTime.data(), lrows.data(), KL, f->lldNames,
                         osm_b200_plan_frame_period(f->lld.get()), lldHtkPaths, lldCsvPaths, lldArffPaths, nullptr, err, lText && lldCsvPaths ? &dt : nullptr,
                         lText && lldHtkPaths ? lpacked.data() : nullptr, lText && lldArffPaths ? &dtA : nullptr))
          return hfail(OSM_B200_ERR_INVALID, err);
      }
    } else {
      st = osm_b200_plan_frame_offsets(p, off.data(), nG, fo.data());
      if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
      K = osm_b200_plan_num_elements(p);
      const int64_t nR = fo.back();
      rows.resize((size_t)nR * K + 1);
      names.resize(K);
      for (int k = 0; k < K; k++) names[k] = osm_b200_plan_element_name(p, k);
      for (int k = 0; k < nG; k++) nTime[k] = osm_b200_plan_num_time_frames(p, off[k + 1] - off[k]);
      devText = devSinks && nR > 0 && (wantCsv || wantHtk || wantArff);
      if (devText) {
        const float *dRows = nullptr;
        st = osm_b200_plan_run_host_resident(p, pcm.data(), off.data(), nG, fo.data(), &dRows);
        if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
        if (!device_sink_rows(dRows, nR, K, wantCsv, s->csv.delim, wantArff, wantHtk, rows, csv, arff, packed))
          return hfail(OSM_B200_ERR_CUDA, std::string("device sinks: ") + cudaGetErrorString(cudaGetLastError()));
      } else {
        st = osm_b200_plan_run_host(p, pcm.data(), off.data(), nG, fo.data(), rows.data());
        if (st != OSM_B200_OK) return hfail(st, osm_b200_last_error());
      }
    }
    const DevText dt = csv.view(), dtA = arff.view();
    const double period = s->hasFunc ? osm_b200_plan_frame_period(s->curFunc->sum ? s->curFunc->sum.get() : p) : osm_b200_plan_frame_period(p);
    if (!write_batch(SinkOpts{s->csv, s->arff, s->parmKind, s->cur}, g.second, fo.data(), nTime.data(), rows.data(), K, names, period, htkPaths, csvPaths, arffPaths, framesOut, err,
                     devText && wantCsv ? &dt : nullptr, devText && wantHtk ? packed.data() : nullptr, devText && wantArff ? &dtA : nullptr))
      return hfail(OSM_B200_ERR_INVALID, err);
  }
  return OSM_B200_OK;
} catch (const std::bad_alloc &) { return hfail(OSM_B200_ERR_NOMEM, "out of host memory"); }
catch (const std::exception &e) { return hfail(OSM_B200_ERR_INVALID, e.what()); }


// The sink half of osm_b200_session_extract_files_arff on rows the caller already holds (e.g. from
// osm_b200_session_extract_pcm): file i gets rows [frame_offsets[i], frame_offsets[i+1]) of `rows` ([.., num_elements]);
// n_samples[i] = sample frames of utterance i (for the time stamps of rows appended at the end of input).  Files are
// formatted in parallel on host threads.  Needs no device: it works on description-only sessions as well.
osm_b200_status osm_b200_session_write_files(osm_b200_session *s, double sampleRate, int32_t nChan, int32_t n, const int64_t *frameOff,
                                             const int64_t *nSamples, const float *rows, const char *const *htkPaths,
                                             const char *const *csvPaths, const char *const *arffPaths)
{
  if (!s || !frameOff || !rows || n < 0) return hfail(OSM_B200_ERR_INVALID, "null argument");
  osm_b200_plan *p;
  osm_b200_status st = get_plan(s, sampleRate, nChan, &p);
  if (st != OSM_B200_OK) return st;
  int K = osm_b200_plan_num_elements(p);
  std::vector<std::string> names(K);
  for (int k = 0; k < K; k++) names[k] = osm_b200_plan_element_name(p, k);
  std::vector<int> idx(n);
  std::vector<int64_t> nTime(n, 0);
  for (int i = 0; i < n; i++) { idx[i] = i; nTime[i] = nSamples ? osm_b200_plan_num_time_frames(p, nSamples[i]) : 0; }
  if (s->hasFunc) {                                  // summary rows (osm_b200_session_extract_pcm of a cFunctionals configuration)
    osm_b200_session::FuncRt *f;
    st = get_func(s, sampleRate, nChan, p, &f);
    if (st != OSM_B200_OK) return st;
    K = f->total; names = f->names;
    for (int i = 0; i < n; i++) nTime[i] = frameOff[i + 1] - frameOff[i];
  }
  std::string err;
  if (!write_batch(SinkOpts{s->csv, s->arff, s->parmKind, s->cur}, idx, frameOff, nTime.data(), rows, K, names, osm_b200_plan_frame_period(p), htkPaths,
                   csvPaths, arffPaths, nullptr, err))
    return hfail(OSM_B200_ERR_INVALID, err);
  return OSM_B200_OK;
}

// introspection for bindings and tests: the sink formatting options the session took from the configuration
const char *osm_b200_session_sink_options(osm_b200_session *s)
{
  static thread_local std::string out;
  out.clear();
  if (!s) return "";
  char b[1024];
  snprintf(b, sizeof b, "csv: header=%d time=%d index=%d name=%d:'%s' delim=%c\n", (int)s->csv.printHeader, (int)s->csv.timestamp,
           (int)s->csv.number, s->csv.prname, s->csv.instName.c_str(), s->csv.delim);
  out += b;
  snprintf(b, sizeof b, "htk: parmKind=%d\n", s->parmKind);
  out += b;
  snprintf(b, sizeof b, "arff: relation='%s' time=%d index=%d name=%d:'%s' append=%d dummy=%d classes=", s->arff.relation.c_str(),
           (int)s->arff.timestamp, (int)s->arff.number, s->arff.prname, s->arff.instName.c_str(), (int)s->arff.append, (int)s->arff.dummyClass);
  out += b;
  for (size_t c = 0; c < s->arff.classes.size(); c++)
    out += (c ? "," : "") + s->arff.classes[c].first + ":" + s->arff.classes[c].second + ":" + (c < s->arff.targetAll.size() ? s->arff.targetAll[c] : "");
  out += "\n";
  return out.c_str();
}

const char *osm_b200_host_last_error(void) { return g_herr.empty() ? osm_b200_last_error() : g_herr.c_str(); }

int32_t osm_b200_write_htk_device(const char *path, const float *d_rows, int64_t n, int32_t K, double period, int32_t parmKind)
{
  if (!path || (n > 0 && !d_rows) || K <= 0 || n < 0) { g_herr = "null argument"; return 1; }
  std::vector<uint32_t> packed;
  if (!device_htk(d_rows, n, K, packed)) { g_herr = std::string("device sinks: ") + cudaGetErrorString(cudaGetLastError()); return 1; }
  std::string err;
  if (write_htk(path, nullptr, n, K, period, parmKind, err, packed.data())) return 0;
  g_herr = err;
  return 1;
}

int32_t osm_b200_write_csv_device(const char *path, const float *d_rows, int64_t n, int32_t K, const char *const *names, double period,
                                  const char *instName, int32_t frameIndex, int32_t frameTime, int64_t nTimeFrames)
{
  if (!path || (n > 0 && !d_rows) || K <= 0 || n < 0 || !names) { g_herr = "null argument"; return 1; }
  CsvOpts o;
  o.number = frameIndex != 0; o.timestamp = frameTime != 0;
  if (instName && instName[0]) { o.prname = 1; o.instName = instName; }
  std::vector<std::string> nm(K);
  for (int k = 0; k < K; k++) nm[k] = names[k];
  std::vector<float> rows((size_t)n * K + 1);
  HostText t;
  const bool ok = device_text(d_rows, n, K, o.delim, false, t) &&
                  (n == 0 || cudaMemcpy(rows.data(), d_rows, (size_t)n * K * sizeof(float), cudaMemcpyDeviceToHost) == cudaSuccess);
  if (!ok) { g_herr = std::string("device sinks: ") + cudaGetErrorString(cudaGetLastError()); return 1; }
  const DevText dt = t.view();
  std::string err;
  if (write_csv(path, rows.data(), n, K, nm, period, o, err, nTimeFrames, &dt)) return 0;
  g_herr = err;
  return 1;
}

int32_t osm_b200_write_htk(const char *path, const float *rows, int64_t n, int32_t K, double period, int32_t parmKind)
{
  std::string err;
  if (write_htk(path, rows, n, K, period, parmKind, err)) return 0;
  g_herr = err;
  return 1;
}

int32_t osm_b200_write_csv(const char *path, const float *rows, int64_t n, int32_t K, const char *const *names, double period,
                           const char *instName, int32_t frameIndex, int32_t frameTime)
{
  return osm_b200_write_csv_timed(path, rows, n, K, names, period, instName, frameIndex, frameTime, 0);
}

int32_t osm_b200_write_csv_timed(const char *path, const float *rows, int64_t n, int32_t K, const char *const *names, double period,
                                 const char *instName, int32_t frameIndex, int32_t frameTime, int64_t nTimeFrames)
{
  std::string err;
  std::vector<std::string> nm(K);
  for (int k = 0; k < K; k++) nm[k] = names[k];
  CsvOpts o;
  if (instName) { o.instName = instName; o.prname = 1; }
  o.number = frameIndex != 0;
  o.timestamp = frameTime != 0;
  if (write_csv(path, rows, n, K, nm, period, o, err, nTimeFrames)) return 0;
  g_herr = err;
  return 1;
}

int32_t osm_b200_write_arff(const char *path, const float *rows, int64_t n, int32_t K, const char *const *names, double period,
                            const char *relation, const char *instName, int32_t frameIndex, int32_t frameTime,
                            int32_t nClasses, const char *const *classNames, const char *const *classTypes,
                            const char *const *targets, int32_t append, int64_t nTimeFrames)
{
  std::string err;
  std::vector<std::string> nm(K);
  for (int k = 0; k < K; k++) nm[k] = names[k];
  ArffOpts o;
  if (relation) o.relation = relation;
  if (instName && instName[0] && strcmp(instName, "-")) { o.instName = instName; o.prname = 1; }
  o.number = frameIndex != 0;
  o.timestamp = frameTime != 0;
  o.append = append != 0;
  for (int c = 0; c < nClasses; c++) {
    o.classes.push_back({classNames && classNames[c] ? classNames[c] : "class", classTypes && classTypes[c] ? classTypes[c] : "numeric"});
    const char *t = targets ? targets[c] : nullptr;
    o.targetAll.push_back(t ? (strcmp(t, "?") ? arff_escape(t) : std::string("?")) : std::string());
  }
  if (write_arff(path, rows, n, K, nm, period, o, err, nTimeFrames)) return 0;
  g_herr = err;
  return 1;
}

}  // extern "C"

// SMILExtract_b200 -- command line front end over libosm_b200.so's session API, taking the same
// options the reference's SMILExtract takes for the LLD path (progsrc/smilextract/SMILExtract.cpp:
// 42-174): -C config, -I input.wav, plus every option the config declares through \cm[...]
// (-O / -output htk, -csvoutput csv, -instname name, ...).  Batch mode: -I may be given several
// times (or -filelist F with one "wav[ htk[ csv]]" per line); all files go through ONE plan run.
// When the active sinks read a summary level and an LLD level (-csvoutput with -lldcsvoutput of the shipped feature
// sets), that one run writes both: -O / -output / -csvoutput name the summary's files, -lld*output the LLD sinks' files.
#include <cstdio>
#include <cstring>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/osm_b200_host.h"

static std::string replace_ext(const std::string &p, const char *ext)
{
  const size_t d = p.find_last_of('.');
  return (d == std::string::npos ? p : p.substr(0, d)) + ext;
}

int main(int argc, char **argv)
{
  std::string conf, level;
  std::vector<std::string> wavs, htks, csvs, arffs, optN, optV;
  std::string outHtk, outCsv, outArff, htkDir, csvDir;
  std::string sumHtk, sumCsv, lldHtk, lldCsv;             // the same options apart, for a session with an LLD part
  int device = 0;
  for (int i = 1; i < argc; i++) {
    const std::string a = argv[i];
    auto val = [&]() -> std::string { return i + 1 < argc ? std::string(argv[++i]) : std::string(); };
    if (a == "-C" || a == "-configfile") conf = val();
    else if (a == "-I" || a == "-inputfile") wavs.push_back(val());
    else if (a == "-device") device = atoi(val().c_str());
    else if (a == "-level") level = val();
    else if (a == "-filelist") {
      std::ifstream f(val());
      std::string line;
      while (std::getline(f, line)) {
        std::istringstream ls(line);
        std::string w, h, c;
        ls >> w >> h >> c;
        if (w.empty()) continue;
        wavs.push_back(w); htks.resize(wavs.size()); csvs.resize(wavs.size());
        htks.back() = h; csvs.back() = c;
      }
    }
    else if (a == "-h" || a == "-help") {
      printf("usage: SMILExtract_b200 -C <config> -I <in.wav> [-I ...] [-O out.htk] [-csvoutput out.csv] [-lldarffoutput out.arff]\n"
             "       [-filelist list.txt] [-device N] [-level lld] [-<config option> value ...]\n");
      return 0;
    }
    else if (a == "-d" || a == "-debug" || a == "-L" || a == "-components" || a == "-cfgFileTemplate" || a == "-cfgFileDescriptions" || a == "-c" ||
             a == "-ccmdHelp" || a == "-exportHelp" || a == "-noconsoleoutput" || a == "-appendLogfile" || a == "-nologfile") {
      // the reference's boolean switches (progsrc/smilextract/SMILExtract.cpp:60-72) take no value unless an explicit 0 / 1 follows;
      // they steer logging and help output, which this front end does not have: accepted and ignored
      if (i + 1 < argc) { const std::string nx = argv[i + 1]; if (nx == "0" || nx == "1" || nx == "yes" || nx == "no" || nx == "true" || nx == "false") i++; }
    }
    else if (a == "-l" || a == "-loglevel" || a == "-t" || a == "-nticks" || a == "-logfile") (void)val();   // logging / tick limit: accepted, ignored
    else if (a.size() > 1 && a[0] == '-') {
      const std::string n = a.substr(1), v = val();
      optN.push_back(n); optV.push_back(v);
      // the feature-set configurations name their LLD sinks' files -lldhtkoutput / -lldcsvoutput
      // (config/shared/standard_data_output.conf.inc:23,33)
      if (n == "O" || n == "output" || n == "lldhtkoutput") outHtk = v;
      if (n == "csvoutput" || n == "lldcsvoutput") outCsv = v;
      if (n == "lldarffoutput") outArff = v;
      if (n == "O" || n == "output") sumHtk = v;
      if (n == "csvoutput") sumCsv = v;
      if (n == "lldhtkoutput") lldHtk = v;
      if (n == "lldcsvoutput") lldCsv = v;
    }
  }
  if (conf.empty() || wavs.empty()) { fprintf(stderr, "SMILExtract_b200: -C <config> and -I <wav> are required (-h for help)\n"); return 2; }
  htks.resize(wavs.size()); csvs.resize(wavs.size()); arffs.resize(wavs.size());
  // single-file form: -O / -csvoutput name that file's outputs; with several inputs they name a
  // directory-less prefix -> per-file names derived from the input name
  for (size_t k = 0; k < wavs.size(); k++) {
    if (htks[k].empty() && !outHtk.empty()) htks[k] = wavs.size() == 1 ? outHtk : replace_ext(wavs[k], ".htk");
    if (csvs[k].empty() && !outCsv.empty()) csvs[k] = wavs.size() == 1 ? outCsv : replace_ext(wavs[k], ".csv");
    // cArffSink appends when its `append` option says so: every input may go to the same file
    if (!outArff.empty()) arffs[k] = outArff;
  }
  std::vector<const char *> on, ov, pw, ph, pc, pa;
  for (size_t k = 0; k < optN.size(); k++) { on.push_back(optN[k].c_str()); ov.push_back(optV[k].c_str()); }
  for (size_t k = 0; k < wavs.size(); k++) {
    pw.push_back(wavs[k].c_str());
    ph.push_back(htks[k].empty() ? nullptr : htks[k].c_str());
    pc.push_back(csvs[k].empty() ? nullptr : csvs[k].c_str());
    pa.push_back(arffs[k].empty() ? nullptr : arffs[k].c_str());
  }
  osm_b200_session *s = nullptr;
  if (osm_b200_session_open(conf.c_str(), (int)on.size(), on.data(), ov.data(), level.empty() ? nullptr : level.c_str(), device, &s) != OSM_B200_OK) {
    fprintf(stderr, "SMILExtract_b200: %s\n", osm_b200_host_last_error());
    return 1;
  }
  std::vector<int64_t> frames(wavs.size(), 0);
  // the LLD part exists for every input format or for none (16 kHz mono asks the session which)
  const bool both = osm_b200_session_lld_num_elements(s, 16000.0, 1) > 0;
  std::vector<std::string> lh(wavs.size()), lc(wavs.size());
  std::vector<const char *> plh, plc;
  for (size_t k = 0; k < wavs.size() && both; k++) {
    // -filelist names the summary's files; several inputs get the LLD files <input>.lld.htk / .lld.csv
    if (!outHtk.empty()) htks[k] = sumHtk.empty() ? std::string() : (wavs.size() == 1 ? sumHtk : replace_ext(wavs[k], ".htk"));
    if (!outCsv.empty()) csvs[k] = sumCsv.empty() ? std::string() : (wavs.size() == 1 ? sumCsv : replace_ext(wavs[k], ".csv"));
    if (!lldHtk.empty()) lh[k] = wavs.size() == 1 ? lldHtk : replace_ext(wavs[k], ".lld.htk");
    if (!lldCsv.empty()) lc[k] = wavs.size() == 1 ? lldCsv : replace_ext(wavs[k], ".lld.csv");
    ph[k] = htks[k].empty() ? nullptr : htks[k].c_str();
    pc[k] = csvs[k].empty() ? nullptr : csvs[k].c_str();
    plh.push_back(lh[k].empty() ? nullptr : lh[k].c_str());
    plc.push_back(lc[k].empty() ? nullptr : lc[k].c_str());
  }
  const osm_b200_status st = both ? osm_b200_session_extract_files_lld(s, (int)wavs.size(), pw.data(), ph.data(), pc.data(), nullptr,
                                                                       lldHtk.empty() ? nullptr : plh.data(), lldCsv.empty() ? nullptr : plc.data(),
                                                                       outArff.empty() ? nullptr : pa.data(), frames.data())
                                  : osm_b200_session_extract_files_arff(s, (int)wavs.size(), pw.data(), ph.data(), pc.data(), pa.data(), frames.data());
  if (st != OSM_B200_OK) { fprintf(stderr, "SMILExtract_b200: %s\n", osm_b200_host_last_error()); osm_b200_session_close(s); return 1; }
  for (size_t k = 0; k < wavs.size(); k++) fprintf(stderr, "%s: %ld frames\n", wavs[k].c_str(), (long)frames[k]);
  osm_b200_session_close(s);
  return 0;
}

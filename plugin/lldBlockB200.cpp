/*
 * cLldBlockB200 -- see lldBlockB200.hpp.  Host glue only: every number on the LLD rows comes from the CUDA plan
 * behind libosm_b200.so (include/osm_b200.h, include/osm_b200_host.h); nothing is computed on the CPU here.
 *
 * Reference interfaces this file is written against (citations relative to the reference tree):
 *   component registration macros            src/include/core/smileComponent.hpp:216-284
 *   cDataProcessor hooks                      src/core/dataProcessor.cpp:104-325,553-600
 *   sequential block reading of a level       src/core/dataReader.cpp:558-640 (as cWaveSink does, src/iocore/waveSink.cpp:140-201)
 *   writing rows + their time stamps          src/core/dataMemoryLevel.cpp:1190-1226,1535-1590
 *   how the wave level was produced           src/smileutil/smileUtil.c:2516-2536 (int16 -> float, mono mixdown)
 */
#include "lldBlockB200.hpp"

#include <cmath>
#include <cstring>

#define MODULE "cLldBlockB200"

SMILECOMPONENT_STATICS(cLldBlockB200)

SMILECOMPONENT_REGCOMP(cLldBlockB200)
{
  SMILECOMPONENT_REGCOMP_INIT
  scname = COMPONENT_NAME_CLLDBLOCKB200;
  sdescription = COMPONENT_DESCRIPTION_CLLDBLOCKB200;

  SMILECOMPONENT_INHERIT_CONFIGTYPE("cDataProcessor")
  SMILECOMPONENT_IFNOTREGAGAIN(
    ct->setField("graphConf", "The openSMILE configuration file whose low-level-descriptor sub-graph (wave level -> captureTo level) is executed on the GPU. The file is read unchanged.", (const char *)NULL);
    ct->setField("captureTo", "The data memory level of graphConf to produce (default: the level read by its active file sinks).", (const char *)NULL);
    ct->setField("graphOption", "graphOption[n] = name=value : command-line options declared by graphConf through \\cm[...] (without the leading '-').", (const char *)NULL, ARRAY_TYPE);
    ct->setField("device", "The CUDA device to run on. There is no CPU path.", 0);
    ct->setField("blocksize", "The number of wave samples read from the input level per tick while gathering.", 4096);
  )
  SMILECOMPONENT_MAKEINFO(cLldBlockB200);
}

SMILECOMPONENT_CREATE(cLldBlockB200)

cLldBlockB200::cLldBlockB200(const char *_name) :
  cDataProcessor(_name), session_(NULL), plan_(NULL), graphConf_(NULL), captureTo_(NULL), device_(0),
  sampleRate_(0.0), nEl_(0), nRows_(0), nTimeRows_(0), emitted_(0), ran_(false)
{
}

void cLldBlockB200::myFetchConfig()
{
  cDataProcessor::myFetchConfig();
  graphConf_ = getStr("graphConf");
  if (graphConf_ == NULL) COMP_ERR("graphConf is not set: name the configuration file whose LLD graph is to be executed");
  captureTo_ = getStr("captureTo");
  device_ = getInt("device");
  int n = getArraySize("graphOption");
  for (int i = 0; i < n; i++) {
    const char *kv = getStr_f(myvprint("graphOption[%i]", i));
    if (kv == NULL) continue;
    const char *eq = strchr(kv, '=');
    if (eq == NULL) COMP_ERR("graphOption[%i] = '%s' is not of the form name=value", i, kv);
    optNames_.push_back(std::string(kv, eq - kv));
    optValues_.push_back(std::string(eq + 1));
  }
  if (blocksizeR_ <= 0) blocksizeR_ = 4096;
}

void cLldBlockB200::openSession()
{
  if (session_ != NULL) return;
  std::vector<const char *> on, ov;
  for (size_t i = 0; i < optNames_.size(); i++) { on.push_back(optNames_[i].c_str()); ov.push_back(optValues_[i].c_str()); }
  osm_b200_status st = osm_b200_session_open(graphConf_, (int32_t)on.size(), on.empty() ? NULL : &on[0], ov.empty() ? NULL : &ov[0],
                                             captureTo_, device_, &session_);
  if (st != OSM_B200_OK) {
    session_ = NULL;
    COMP_ERR("B200 back end cannot execute '%s': %s", graphConf_, osm_b200_host_last_error());   // -> cComponentException
  }
}

int cLldBlockB200::configureReader(const sDmLevelConfig &c)
{
  cDataProcessor::configureReader(c);
  if (blocksizeR_ < 16) blocksizeR_ = 16;
  reader_->setupSequentialMatrixReading(blocksizeR_, blocksizeR_, 0);
  return 1;
}

int cLldBlockB200::configureWriter(sDmLevelConfig &c)
{
  if (c.T <= 0.0) COMP_ERR("the input level has no sample period: cLldBlockB200 must read a wave level");
  if (reader_->getLevelN() != 1)
    COMP_ERR("the input level has %i elements per sample; the B200 plan takes the mono wave level (cWaveSource.monoMixdown = 1)", reader_->getLevelN());
  sampleRate_ = floor(1.0 / c.T + 0.5);
  openSession();
  // the carrier channel count is only known once samples arrive; names, period and row counts do not depend on it
  if (osm_b200_session_plan(session_, sampleRate_, 1, &plan_) != OSM_B200_OK)
    COMP_ERR("B200 back end: %s", osm_b200_host_last_error());
  nEl_ = osm_b200_plan_num_elements(plan_);
  const double period = osm_b200_plan_frame_period(plan_);
  c.T = period;
  c.frameSizeSec = (double)osm_b200_plan_frame_size_samples(plan_) / sampleRate_;
  c.blocksizeWriter = 1;
  if (c.nT < 1024) c.nT = 1024;          // rows are handed over in pieces of at most the free space of the level
  return 1;
}

// element names "base[k]" with consecutive k become one array field, as the reference's levels have them
// (src/core/dataMemoryLevel.cpp:1158-1169 prints name[idx + arrNameOffset])
int cLldBlockB200::setupNewNames(long nEl)
{
  long i = 0;
  while (i < nEl_) {
    std::string nm = osm_b200_plan_element_name(plan_, (int32_t)i);
    size_t br = nm.rfind('[');
    if (br == std::string::npos || nm.empty() || nm[nm.size() - 1] != ']') { writer_->addField(nm.c_str(), 1); i++; continue; }
    const std::string base = nm.substr(0, br);
    const int first = atoi(nm.c_str() + br + 1);
    long n = 1;
    while (i + n < nEl_) {
      std::string nx = osm_b200_plan_element_name(plan_, (int32_t)(i + n));
      char want[32];
      snprintf(want, sizeof want, "[%d]", first + (int)n);
      if (nx != base + want) break;
      n++;
    }
    writer_->addField(base.c_str(), (int)n, first);
    i += n;
  }
  namesAreSet_ = 1;
  return 1;
}

// The wave level holds v = (sum_c x_c / C) / 32767 of the file's int16 samples (smileUtil.c:2527-2534).  The plan takes
// int16 PCM and performs that conversion itself, so the samples are re-encoded exactly: s = sum_c x_c = round(v * 32767 * C)
// for the smallest channel count C that reproduces every v bit for bit, carried as C int16 values whose sum is s.
bool cLldBlockB200::recoverPcm(const std::vector<float> &wave, std::vector<int16_t> &pcm, int &nCarrier)
{
  for (int C = 1; C <= 8; C++) {
    bool ok = true;
    const size_t n = wave.size();
    pcm.resize(n * (size_t)C);
    for (size_t i = 0; i < n && ok; i++) {
      const long s = lrint((double)wave[i] * 32767.0 * (double)C);
      const float back = ((float)s / (float)C) / (float)32767.0;
      if (back != wave[i] || s > 32767L * C || s < -32768L * C) { ok = false; break; }
      long q = s / C, r = s - q * C;             // r has the sign of s, |r| < C
      for (int c = 0; c < C; c++) {
        long x = q;
        if (r > 0) { x++; r--; } else if (r < 0) { x--; r++; }
        pcm[i * (size_t)C + c] = (int16_t)x;
      }
    }
    if (ok) { nCarrier = C; return true; }
  }
  return false;
}

void cLldBlockB200::runBlock()
{
  ran_ = true;
  std::vector<int16_t> pcm;
  int C = 1;
  if (!recoverPcm(wave_, pcm, C))
    COMP_ERR("the wave level does not hold 16-bit PCM samples (converted by the wave source): the B200 plan computes from int16 PCM only");
  osm_b200_plan *plan = NULL;
  if (osm_b200_session_plan(session_, sampleRate_, C, &plan) != OSM_B200_OK) COMP_ERR("B200 back end: %s", osm_b200_host_last_error());
  const int64_t nSamp = (int64_t)wave_.size();
  int64_t uttOff[2] = {0, nSamp}, frameOff[2] = {0, 0};
  nRows_ = (long)osm_b200_plan_num_frames(plan, nSamp);
  nTimeRows_ = (long)osm_b200_plan_num_time_frames(plan, nSamp);
  rows_.assign((size_t)nRows_ * (size_t)nEl_ + 1, 0.0f);
  pcm.resize(pcm.size() + 16, 0);
  if (osm_b200_session_extract_pcm(session_, &pcm[0], uttOff, 1, sampleRate_, C, frameOff, &rows_[0], nRows_) != OSM_B200_OK)
    COMP_ERR("B200 back end: %s", osm_b200_host_last_error());
  SMILE_IMSG(3, "B200 block: %ld samples (%i-channel carrier) -> %ld rows x %ld elements", (long)nSamp, C, nRows_, nEl_);
  std::vector<float>().swap(wave_);
}

eTickResult cLldBlockB200::myTick(long long t)
{
  if (!ran_) {
    cMatrix *mat = reader_->getNextMatrix(0, 0, DMEM_PAD_NONE);
    if (mat != NULL) {
      wave_.insert(wave_.end(), mat->data, mat->data + mat->nT * mat->N);
      return TICK_SUCCESS;
    }
    if (!isEOI()) return TICK_SOURCE_NOT_AVAIL;
    runBlock();
  }
  if (emitted_ >= nRows_) return TICK_INACTIVE;
  long n = nRows_ - emitted_;
  const long nFree = writer_->getNFree();
  if (n > nFree) n = nFree;
  if (n > 512) n = 512;
  if (n <= 0 || !writer_->checkWrite(n)) return TICK_DEST_NO_SPACE;
  cMatrix out((int)nEl_, (int)n);
  memcpy(out.data, &rows_[(size_t)emitted_ * (size_t)nEl_], sizeof(float) * (size_t)n * (size_t)nEl_);
  for (long i = 0; i < n; i++) {
    // rows appended by window processors at the end of input repeat the last frame's time stamp (dataMemoryLevel.cpp:1698-1708).
    // The time of a row comes from the plan, not from r * level period: the two differ for centred frames, cTonefilt blocks and a
    // cCens level, whose period is its input's times downsampleRatio while its rows keep their input rows' times.
    long r = emitted_ + i;
    if (nTimeRows_ > 0 && r > nTimeRows_ - 1) r = nTimeRows_ - 1;
    out.tmeta[i].time = osm_b200_plan_row_time(plan_, r);
    if (r == 0) out.tmeta[i].time = 0.0;
    out.tmeta[i].lengthSec = (double)osm_b200_plan_frame_size_samples(plan_) / sampleRate_;
  }
  if (!writer_->setNextMatrix(&out)) return TICK_DEST_NO_SPACE;
  emitted_ += n;
  return TICK_SUCCESS;
}

cLldBlockB200::~cLldBlockB200()
{
  if (session_ != NULL) osm_b200_session_close(session_);
}

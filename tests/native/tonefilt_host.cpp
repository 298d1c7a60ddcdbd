// tonefilt_host.cpp -- host build of the block statements of the cTonefilt kernel (opensmile_b200/csrc/tonefilt.cu,
// tonefilt_math.cuh), test infrastructure.  The kernel forms the in-block sums G_b on the FP64 tensor cores; here they are a
// loop over the block's samples.  Segment cuts are an argument: seg = rows per segment (0 = one segment), the state entering
// a segment is chained from the segment aggregates as tonefilt_carry_kernel does.
//   g++ -O2 -ffp-contract=off -shared -fPIC -o tonefilt_host.so tonefilt_host.cpp
#include <cmath>
#include <vector>

#include "../../opensmile_b200/csrc/tonefilt_math.cuh"

namespace {
// rows [a, b) of note k from state z (zr, zi); out = nullptr: the end state only
void run_rows(const float *x, long L, int P, double T, const std::vector<double> &W, int nc, double a, double f, int k, long ra, long rb,
              double &zr, double &zi, float *out, int nNotes)
{
  for (long r = ra; r < rb; r++) {
    double gr = 0.0, gi = 0.0;
    for (int j = 0; j < P; j++) {
      long m = r * P + j;
      if (m >= L) m = L - 1;
      gr += W[(size_t)j * nc + 2 * k] * (double)x[m];
      gi += W[(size_t)j * nc + 2 * k + 1] * (double)x[m];
    }
    osm::tf::block_step(zr, zi, a, gr, gi, f, (long long)r, P, T);
    if (out) out[r * nNotes + k] = osm::tf::tone_value(zr, zi);
  }
}
}  // namespace

extern "C" {

// rows of the cTonefilt level for the tables freq / decay (after the reference's clamps), block length P
long tfh_run(const float *x, long L, int P, double fs, const double *freq, const double *decay, int nNotes, long seg, float *out)
{
  std::vector<double> fr(freq, freq + nNotes), dc(decay, decay + nNotes), W, a;
  const double T = 1.0 / fs;
  osm::tf::block_tables(fr, dc, P, T, W, a);
  const int nc = osm::tf::padded_cols(nNotes);
  const long rows = (L + P - 1) / P;
  const long step = seg > 0 ? seg : (rows > 0 ? rows : 1);
  for (int k = 0; k < nNotes; k++) {
    double cr = 0.0, ci = 0.0;                       // state entering the segment
    for (long s0 = 0; s0 < rows; s0 += step) {
      const long s1 = s0 + step < rows ? s0 + step : rows;
      double zr = cr, zi = ci;
      run_rows(x, L, P, T, W, nc, a[k], fr[k], k, s0, s1, zr, zi, out, nNotes);
      double er = 0.0, ei = 0.0;                     // the segment's aggregate from a zero state, chained as the carry kernel does
      run_rows(x, L, P, T, W, nc, a[k], fr[k], k, s0, s1, er, ei, nullptr, nNotes);
      const double an = pow(a[k], (double)(s1 - s0));
      cr = an * cr + er;
      ci = an * ci + ei;
    }
  }
  return rows;
}

// cChroma on rows [n][nNotes]
void tfh_chroma(const float *t, long n, int nNotes, int K, float silThresh, float *out)
{
  for (long r = 0; r < n; r++) osm::tf::chroma_row(t + r * nNotes, 1, nNotes, K, silThresh, out + r * K, 1);
}
}

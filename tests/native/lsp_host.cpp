// lsp_host.cpp -- host build of the statements of the stand-alone cLpc / cLsp kernel (opensmile_b200/csrc/lsp.cu:
// formant_math.cuh acf_lag + durbin, lsp_math.cuh) (test infrastructure).  The kernel runs the autocorrelation with one
// lane per lag and the rest with one thread per frame; here the lanes are a loop.
//   g++ -O2 -ffp-contract=off -shared -fPIC -o lsp_host.so lsp_host.cpp
#include "../../opensmile_b200/csrc/formant_math.cuh"
#include "../../opensmile_b200/csrc/lsp_math.cuh"

extern "C" {

// one frame x[n] of the level cLpc reads -> a[p], returns the gain
float lsph_lpc(const float *x, int n, int p, float *a)
{
  float r[osm::fm::kMaxLpcOrder + 1];
  for (int l = 0; l <= p; l++) r[l] = osm::fm::acf_lag(x, n, l);
  return osm::fm::durbin(r, p, a);
}

// a[p] -> lsf[p]; returns the roots of the final search
int lsph_lsp(const float *a, int p, float *lsf) { return osm::lsp::lsp_from_lpc(a, p, lsf); }

// roots of one grid search with step delta (no retry, no zero fill)
int lsph_search(const float *a, int p, float *lsf, float delta) { return osm::lsp::lpc_to_lsp(a, p, lsf, osm::lsp::kBisections, delta); }

}

// lsp_math.cuh -- cLsp's LPC -> line spectral pair conversion, written once for the device (lsp.cu) and for a host
// build of the same statements (tests/native/lsp_host.cpp, compared bit for bit with the oracle on the reference's
// LPC rows).  Citations relative to /root/reference/src.  Compile with FMA contraction off (-fmad=false /
// -ffp-contract=off): every float statement below keeps the reference's order and rounding.
#pragma once
#include <math.h>

#ifdef __CUDACC__
#define OSM_LSP_HD __host__ __device__ __forceinline__
#else
#define OSM_LSP_HD inline
#endif

namespace osm {
namespace lsp {

constexpr int kMaxOrder = 16;        // cLpc.p (the graph compiler's limit)
constexpr int kBisections = 10;      // cLsp::processVector passes nb = 10 (lld/lsp.cpp:300): nb + 1 halvings

// cLsp::cheb_poly_eva (lld/lsp.cpp:113-129): float Clenshaw recurrence of order m at x
OSM_LSP_HD float cheb_poly_eva(const float *coef, float x, int m)
{
  float b0 = 0.0f, b1 = 0.0f;
  x *= 2.0f;
  for (int k = m; k > 0; k--) {
    const float tmp = b0;
    b0 = x * b0 - b1 + coef[m - k];
    b1 = tmp;
  }
  return -b1 + 0.5f * x * b0 + coef[m];
}

// SIGN_CHANGE(a, b): the float product compared with 0.0 (an underflowing product is no sign change)
OSM_LSP_HD bool sign_change(float a, float b) { return (double)(a * b) < 0.0; }

// acos of a float: the reference calls acos(float) through <math.h> in C++, i.e. the float overload (glibc's acosf; the
// device's acosf may differ from it by an ulp or two)
OSM_LSP_HD float x2angle(float x) { return acosf(x); }

// cLsp::lpc_to_lsp (lld/lsp.cpp:145-269): roots of P'(z) and Q'(z) on the x = cos(w) axis, alternating, searched
// downwards from x = 1 with step delta * (1 - 0.9 x^2) (halved near a root), each refined by nb + 1 bisections.
// Writes freq[j] for every root found and returns their number (the roots are found in order j = 0, 1, ...).
OSM_LSP_HD int lpc_to_lsp(const float *a, int lpcrdr, float *freq, int nb, float delta)
{
  float P[kMaxOrder / 2 + 1], Q[kMaxOrder / 2 + 1];
  const int m = lpcrdr / 2;
  P[0] = 1.0f;
  Q[0] = 1.0f;
  for (int i = 0; i < m; i++) {
    P[i + 1] = (a[i] + a[lpcrdr - 1 - i]) - P[i];
    Q[i + 1] = (a[i] - a[lpcrdr - 1 - i]) + Q[i];
  }
  for (int i = 0; i < m; i++) {
    P[i] = 2 * P[i];
    Q[i] = 2 * Q[i];
  }
  float xr = 0.0f, xl = 1.0f, xm = 0.0f;
  int roots = 0;
  for (int j = 0; j < lpcrdr; j++) {
    const float *pt = (j & 1) ? Q : P;
    float psuml = cheb_poly_eva(pt, xl, m);
    bool flag = true;
    while (flag && ((double)xr >= -1.0)) {
      float dd = delta * (1.0f - 0.9f * xl * xl);
      if ((double)fabsf(psuml) < .2) dd *= 0.5f;
      xr = xl - dd;
      float psumr = cheb_poly_eva(pt, xr, m);
      const float temp_psumr = psumr, temp_xr = xr;
      if (sign_change(psumr, psuml)) {
        roots++;
        for (int k = 0; k <= nb; k++) {
          xm = 0.5f * (xl + xr);
          const float psumm = cheb_poly_eva(pt, xm, m);
          if (!sign_change(psumm, psuml)) { psuml = psumm; xl = xm; }
          else { psumr = psumm; xr = xm; }
        }
        if ((double)xm > 1.0) xm = 1.0f;
        else if ((double)xm < -1.0) xm = -1.0f;
        freq[j] = x2angle(xm);
        xl = xm;
        flag = false;
      } else {
        psuml = temp_psumr;
        xl = temp_xr;
      }
    }
  }
  return roots;
}

// cLsp::processVector (lld/lsp.cpp:289-313): grid 0.2 first, 0.05 when it misses roots, then zeros from the last root on.
// Returns the number of roots of the final search.
OSM_LSP_HD int lsp_from_lpc(const float *a, int p, float *lsf)
{
  int roots = lpc_to_lsp(a, p, lsf, kBisections, 0.2f);
  if (roots != p) {
    roots = lpc_to_lsp(a, p, lsf, kBisections, 0.05f);
    for (int i = roots; i < p; i++) lsf[i] = 0.0f;
  }
  return roots;
}

}  // namespace lsp
}  // namespace osm

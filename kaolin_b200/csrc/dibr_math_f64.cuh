// dibr_math_f64.cuh — the <double> instantiation of the reference's per-pixel arithmetic
// (rasterization_cuda.cu:85-188,266-399, dibr_soft_mask_cuda.cu:74-182,266-349 with
// scalar_t = double).  The rasterize trees use the contraction pattern read from the SASS of the
// reference's <double> forward kernel (the reference object compiled for the tests: DMUL + DFMA(.., -prod),
// (w0 + w1) + w2, DADD of the copysign eps, three IEEE divisions; pixel centres computed in
// float and widened), i.e. the <float> trees of dibr_math.cuh with double operations, so face_idx
// is decided by the same comparisons.  The soft-mask distances / gradients follow the source
// expressions with the same fma placement as the <float> trees, which is also the per-edge tree of
// the reference's <double> soft-mask kernel.  face_idx, the weights, the interpolated features and
// the forward soft mask are bit-compared with the reference's <double> kernels
// (tests/test_f64_matrix_gpu.py); the gradients are compared to 1e-13 of their scale, as both sides
// sum them with double atomics in different orders.
#pragma once
#include "dibr_math.cuh"

namespace dibr64 {

using dibr::dadd; using dibr::dsub; using dibr::dmul; using dibr::ddiv;

#if defined(__CUDA_ARCH__)
DIBR_HD double dfma(double a, double b, double c) { return __fma_rn(a, b, c); }
#else
DIBR_HD double dfma(double a, double b, double c) { return fma(a, b, c); }
#endif

// inside <=> !(w0 < 0 || w1 < 0 || w2 < 0)   (NaN counts as inside, as in the reference)
DIBR_HD bool raster_weights(double eps, double x0, double y0, double ax, double ay, double bx, double by, double cx,
                            double cy, double& w0, double& w1, double& w2) {
  const double aex = dsub(ax, x0), aey = dsub(ay, y0), bex = dsub(bx, x0), bey = dsub(by, y0);
  const double cex = dsub(cx, x0), cey = dsub(cy, y0);
  const double u0 = dfma(bex, cey, -dmul(bey, cex));
  const double u1 = dfma(aey, cex, -dmul(aex, cey));
  const double u2 = dfma(aex, bey, -dmul(aey, bex));
  double norm = dadd(dadd(u0, u1), u2);
  norm = dadd(norm, copysign(fabs(eps), norm));
  w0 = ddiv(u0, norm); w1 = ddiv(u1, norm); w2 = ddiv(u2, norm);
  return !(w0 < 0.0 || w1 < 0.0 || w2 < 0.0);
}
DIBR_HD double raster_interp(double r0, double r1, double r2, double w0, double w1, double w2) {
  return dfma(r2, w2, dfma(r0, w0, dmul(r1, w1)));
}

#define DIBR64_EPS 1e-7
DIBR_HD double soft_min_dist(double x0, double y0, const double v[6], float multiplier, int& edgeid) {
  double pdis[6];
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const double x1 = v[2 * i], y1 = v[2 * i + 1];
    const int j = (i + 1) % 3;
    const double x2 = v[2 * j], y2 = v[2 * j + 1];
    const double A = dsub(y2, y1), B = dsub(x1, x2);
    const double C = dfma(y1, x2, -dmul(x1, y2));
    const double AA = dmul(A, A), BB = dmul(B, B), AB = dmul(A, B);
    const double down = dadd(dadd(AA, BB), DIBR64_EPS);
    const double up = dadd(C, dfma(y0, B, dmul(x0, A)));
    const double x3 = ddiv(dfma(-A, C, dfma(x0, BB, -dmul(y0, AB))), down);
    const double y3 = ddiv(dfma(-B, C, dfma(y0, AA, -dmul(x0, AB))), down);
    const double direct = dfma(dsub(x3, x1), dsub(x3, x2), dmul(dsub(y3, y1), dsub(y3, y2)));
    pdis[i] = direct > 0.0 ? (double)((4.f * multiplier) * multiplier) : ddiv(dmul(up, up), down);
  }
#pragma unroll
  for (int i = 0; i < 3; i++) {
    const double dx = dsub(x0, v[2 * i]), dy = dsub(y0, v[2 * i + 1]);
    pdis[3 + i] = dfma(dx, dx, dmul(dy, dy));
  }
  edgeid = 0;
  double d = pdis[0];
#pragma unroll
  for (int i = 1; i < 6; i++) {
    if (d > pdis[i]) { d = pdis[i]; edgeid = i; }
  }
  return d;
}
DIBR_HD double soft_prob(double d2, float sigmainv, float multiplier) {
  return exp(-ddiv(ddiv(dmul((double)sigmainv, d2), (double)multiplier), (double)multiplier));
}

// dibr_soft_mask_cuda.cu:276-347 with scalar_t = double
DIBR_HD void soft_backward_terms(double x0, double y0, const double v[6], int edgeid, double prob, double allprob,
                                 double dLdp, float sigmainv, float multiplier, double g[6]) {
#pragma unroll
  for (int i = 0; i < 6; i++) g[i] = 0.0;
  const double m = (double)multiplier;
  const double dLdz = dmul(ddiv(dmul(dmul(-(double)sigmainv, dLdp), dsub(1.0, allprob)),
                                dadd(dsub(1.0, prob), DIBR64_EPS)), prob);
  if (edgeid >= 3) {
    const int k = edgeid - 3;
    const double two = dadd(dLdz, dLdz);
    g[2 * k] = ddiv(dmul(two, dsub(v[2 * k], x0)), m);
    g[2 * k + 1] = ddiv(dmul(two, dsub(v[2 * k + 1], y0)), m);
  } else {
    const int k = edgeid, j = (edgeid + 1) % 3;
    const double x1 = v[2 * k], y1 = v[2 * k + 1], x2 = v[2 * j], y2 = v[2 * j + 1];
    const double A = dsub(y2, y1), B = dsub(x1, x2);
    const double C = dfma(y1, x2, -dmul(x1, y2));
    const double up = dadd(C, dfma(y0, B, dmul(x0, A)));
    const double down = dadd(dfma(B, B, dmul(A, A)), DIBR64_EPS);
    const double dissquare = ddiv(dmul(up, up), down);
    const double dzdA = ddiv(dmul(2.0, dfma(x0, up, -dmul(A, dissquare))), down);
    const double dzdB = ddiv(dmul(2.0, dfma(y0, up, -dmul(B, dissquare))), down);
    const double dzdC = ddiv(dmul(2.0, up), down);
    g[2 * k] = ddiv(dmul(dLdz, dfma(-y2, dzdC, dzdB)), m);
    g[2 * k + 1] = ddiv(dmul(dLdz, dfma(x2, dzdC, -dzdA)), m);
    g[2 * j] = ddiv(dmul(dLdz, dfma(y1, dzdC, -dzdB)), m);
    g[2 * j + 1] = ddiv(dmul(dLdz, dfma(-x1, dzdC, dzdA)), m);
  }
}

// rasterization_cuda.cu:292-399 with scalar_t = double: out6[j] += sum_d dldI_d * dI_d/dp_j
struct BwdGeom { double n1ax, n1ay, n2ax, n2ay, d1bx, d1by, d1cx, d1cy, d2bx, d2by, d2cx, d2cy, k3sq; };
DIBR_HD void raster_backward_geom(const double p[6], double aw, double bw, double cw, float eps, BwdGeom& G) {
  const double ax = p[0], ay = p[1], bx = p[2], by = p[3], cx = p[4], cy = p[5];
  const double pp = dsub(by, ay), n = dsub(cx, ax), m = dsub(bx, ax), q = dsub(cy, ay);
  double k3 = dfma(m, q, -dmul(pp, n));
  k3 = dadd(k3, copysign(fabs((double)eps), k3));
  const double y0 = dfma(cy, cw, dfma(ay, aw, dmul(by, bw)));
  const double x0 = dfma(cx, cw, dfma(ax, aw, dmul(bx, bw)));
  const double t = dsub(y0, ay), s = dsub(x0, ax);
  const double k1 = dfma(q, s, -dmul(n, t)), k2 = dfma(m, t, -dmul(pp, s));
  const double tk3 = dmul(t, k3), sk3 = dmul(s, k3);
  const double dw1ds = dmul(q, k3), dw1dm = -dmul(q, k1), dw2dm = dfma(-q, k2, tk3), dw1dn = dfma(pp, k1, -tk3);
  const double dw1dp = dmul(n, k1), dw1dq = dfma(-m, k1, sk3), dw1dt = -dmul(n, k3), dw2dp = dfma(n, k2, -sk3);
  const double dw2ds = -dmul(pp, k3), dw2dt = dmul(m, k3), dw2dn = dmul(pp, k2), dw2dq = -dmul(m, k2);
  G.n1ay = dadd(dw1dt, dadd(dw1dp, dw1dq)); G.n1ax = dadd(dw1ds, dadd(dw1dm, dw1dn));
  G.n2ax = dadd(dw2ds, dadd(dw2dm, dw2dn)); G.n2ay = dadd(dw2dt, dadd(dw2dp, dw2dq));
  G.d1bx = dw1dm; G.d1by = dw1dp; G.d1cx = dw1dn; G.d1cy = dw1dq;
  G.d2bx = dw2dm; G.d2by = dw2dp; G.d2cx = dw2dn; G.d2cy = dw2dq;
  G.k3sq = dmul(k3, k3);
}
DIBR_HD void raster_backward_feature(const BwdGeom& G, double g, double c0, double c1, double c2, double out[6]) {
  const double d1 = dsub(c1, c0), d2 = dsub(c2, c0), dl = ddiv(g, G.k3sq);
  out[0] = dmul(dfma(-G.n2ax, d2, -dmul(G.n1ax, d1)), dl);
  out[1] = dmul(dfma(-G.n2ay, d2, -dmul(G.n1ay, d1)), dl);
  out[2] = dmul(dfma(G.d1bx, d1, dmul(G.d2bx, d2)), dl);
  out[3] = dmul(dfma(G.d1by, d1, dmul(G.d2by, d2)), dl);
  out[4] = dmul(dfma(G.d1cx, d1, dmul(G.d2cx, d2)), dl);
  out[5] = dmul(dfma(G.d1cy, d1, dmul(G.d2cy, d2)), dl);
}

}  // namespace dibr64

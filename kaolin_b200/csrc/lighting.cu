// lighting.cu — diffuse shading right after the rasterizer (kaolin/render/lighting/sg.py, sh.py),
// behind the C ABI of include/dibr_b200.h:
//
//   general reduced SG inner product   out(N,3) = sum_m <sg_n, other_m>     (the _C.render.sg operator)
//   SG_INNER_PRODUCT                    per-point cosine lobe (1.17, normal, 2.133) . lights, clamp, albedo/pi
//   SG_FITTED                           Stephen Hill's fitted irradiance, mean over lights, clamp, albedo/pi
//   SH9                                 sum_k band_k(normal) c_k lights_k, x albedo
//   SPECULAR                            sg_warp_specular_term: the GGX lobe of (normal, roughness) warped
//                                       by the view . lights, times Smith visibility, Fresnel and n.l
//
// One kernel template per direction, instantiated per Kind; the general op, SG_INNER_PRODUCT and
// SPECULAR differ only in where the sg side comes from (per-point arrays, the cosine lobe of the
// normal, or the warped distribution lobe) and in the epilogue.
//
// Layout of the work: a CTA of 256 threads takes tiles of 1024 points, four consecutive points per
// thread, so that the 12-byte rows of a thread's points are three 16-byte loads (scalar loads when
// the base is not 16-byte aligned or the tile is partial).  The point data stays in registers for
// the whole light loop: it is read from HBM exactly once for every L.  Lights are staged in shared
// memory 64 at a time, with the per-light terms the formulas share precomputed in fp32; with L <= 64
// they are staged once per CTA, above that once per tile and chunk (from L2).
//
// Light gradients are deterministic: the backward grid has a fixed number of CTAs for a given N,
// each warp sums its four-point partials with a fixed shuffle tree, the eight warps are summed in
// warp order into a per-CTA slot of the workspace, and a finalize kernel sums the CTA slots in CTA
// order in fp64.  No float atomics are used anywhere.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/dibr_b200.h"
#include "op_layouts.h"

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kPts = 4;                     // points per thread per tile
constexpr int kTile = kThreads * kPts;
constexpr int kChunk = 64;                  // lights staged in shared memory at a time
constexpr int kSms = 132;                   // persistent grids: Cfg::kFwdBlocks CTAs on each of H100's 132 SMs
constexpr int kBwdCtas = kSms * 2;          // 2 resident CTAs per SM (__launch_bounds__ below); also the
                                            // number of per-CTA partial slots in the workspace
constexpr float kPi = 3.14159265358979323846f;
constexpr float kTwoPi = 6.28318530717958647692f;

enum Kind { GENERAL = 0, LOBE = 1, FITTED = 2, SH9 = 3, SPECULAR = 4, SHADE = 5 };

template <int K> struct Cfg {
  // per-point floats in registers (SPECULAR: the warped lobe a, w, ws, then V(ndl) V(ndv), (1-ldh)^5, ndl;
  // SHADE: unit normal, roughness, view, and SPECULAR's 8 besides)
  static constexpr int kIn = K == GENERAL ? 7 : K == SPECULAR ? 8 : K == SHADE ? 7 : 3;
  static constexpr int kRec = (K == GENERAL || K == LOBE || K == SPECULAR || K == SHADE) ? 8 : 16;  // floats per staged light
  static constexpr int kAcc = K == SH9 ? 9 : 7;                      // per-light gradient partials
  // resident forward CTAs per SM: the SPECULAR prologue needs more than 64 registers, and SHADE holds
  // both lobes' state (normal, warped lobe and epilogue factors, two sums) for each of its points
  static constexpr int kFwdBlocks = K == SPECULAR ? 3 : K == SHADE ? 2 : 4;
  // points per thread: kPts, except in SHADE's backward, whose per-point state (both lobes' sums,
  // their gradients and the normal's) does not fit 128 registers at 4 points
  static constexpr int pts(bool bwd) { return bwd && K == SHADE ? 2 : kPts; }
};

struct Args {
  int64_t n;
  int L;
  // GENERAL: the sg side; SPECULAR: view and roughness in the slots GENERAL's direction and sharpness
  // use (the layout, and with it every kernel's parameter offsets, is the same for all kinds)
  const float* p_amp;
  union { const float* p_dir; const float* view; };
  union { const float* p_sharp; const float* rough; };
  const float* normal; const float* albedo;                         // shading models
  const float* l_amp; const float* l_dir; const float* l_sharp;   // lights / "other" (SH9: l_amp = 9 coefficients)
  float* out;
  const float* grad_out;
  float* g_amp;                                                     // GENERAL: sg-side gradients
  union { float* g_dir; float* g_view; };
  union { float* g_sharp; float* g_rough; };
  float* g_normal; float* g_albedo;
  float* gl_amp; float* gl_dir; float* gl_sharp;                    // light gradients
  float* partial;                                                   // [grid][L][kAcc]
};                                  // SPECULAR: albedo = spec_albedo, g_albedo = grad_spec_albedo

// ---------------------------------------------------------------------------------------------
// P-point row loads / stores (P = kPts except in SHADE's backward): P C / 4 16-byte accesses when
// aligned and P C is a multiple of 4, scalar accesses otherwise.
template <int C, int P>
__device__ __forceinline__ void load_rows(const float* __restrict__ base, int64_t p0, int64_t n, float (&v)[P][C]) {
  const float* src = base + p0 * C;
  if ((P * C) % 4 == 0 && p0 + P <= n && (reinterpret_cast<uintptr_t>(src) & 15) == 0) {
#pragma unroll
    for (int q = 0; q < P * C / 4; ++q) {
      const float4 t = __ldg(reinterpret_cast<const float4*>(src) + q);
      v[(4 * q) / C][(4 * q) % C] = t.x;
      v[(4 * q + 1) / C][(4 * q + 1) % C] = t.y;
      v[(4 * q + 2) / C][(4 * q + 2) % C] = t.z;
      v[(4 * q + 3) / C][(4 * q + 3) % C] = t.w;
    }
  } else {
#pragma unroll
    for (int p = 0; p < P; ++p)
#pragma unroll
      for (int c = 0; c < C; ++c) v[p][c] = (p0 + p < n) ? __ldg(src + p * C + c) : 0.f;
  }
}

template <int C, int P>
__device__ __forceinline__ void store_rows(float* __restrict__ base, int64_t p0, int64_t n, const float (&v)[P][C]) {
  float* dst = base + p0 * C;
  if ((P * C) % 4 == 0 && p0 + P <= n && (reinterpret_cast<uintptr_t>(dst) & 15) == 0) {
#pragma unroll
    for (int q = 0; q < P * C / 4; ++q)
      reinterpret_cast<float4*>(dst)[q] = make_float4(v[(4 * q) / C][(4 * q) % C], v[(4 * q + 1) / C][(4 * q + 1) % C],
                                                      v[(4 * q + 2) / C][(4 * q + 2) % C], v[(4 * q + 3) / C][(4 * q + 3) % C]);
  } else {
#pragma unroll
    for (int p = 0; p < P; ++p)
      if (p0 + p < n)
#pragma unroll
        for (int c = 0; c < C; ++c) dst[p * C + c] = v[p][c];
  }
}

// ---------------------------------------------------------------------------------------------
// Light staging: record m of the current chunk from light `l`.
template <int K>
__device__ __forceinline__ void stage_light(const Args& a, int l, float* rec) {
  if (K == SH9) {
#pragma unroll
    for (int k = 0; k < 9; ++k) rec[k] = __ldg(a.l_amp + k);
  } else if (K == FITTED) {
    const float lb = __ldg(a.l_sharp + l);
    const float eml = expf(-lb), em2l = eml * eml, rl = 1.f / lb;
    const float scale = 1.f + 2.f * em2l - rl;
    const float bias = (eml - em2l) * rl - em2l;
    const float x = sqrtf(1.f - scale);
    const float dscale = -4.f * em2l + rl * rl;
    const float dbias = (2.f * em2l - eml) * rl - (eml - em2l) * rl * rl + 2.f * em2l;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      rec[k] = __ldg(a.l_dir + 3 * l + k);
      rec[3 + k] = kTwoPi * (__ldg(a.l_amp + 3 * l + k) / lb);
    }
    rec[6] = scale; rec[7] = bias; rec[8] = x; rec[9] = (1.f / (4.f * 0.36f)) * x;
    rec[10] = rl; rec[11] = dscale; rec[12] = dbias; rec[13] = -dscale / (2.f * x);
    rec[14] = kTwoPi / lb; rec[15] = 0.f;
  } else {
    const float lb = __ldg(a.l_sharp + l);
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      rec[k] = __ldg(a.l_amp + 3 * l + k);
      rec[3 + k] = __ldg(a.l_dir + 3 * l + k) * lb;
    }
    rec[6] = lb; rec[7] = 0.f;
  }
}

// Stage lights [c0, c0 + cnt) into shared memory (caller synchronises).
template <int K>
__device__ __forceinline__ void stage_chunk(const Args& a, int c0, int cnt, float* s_light) {
  for (int m = threadIdx.x; m < cnt; m += kThreads) stage_light<K>(a, c0 + m, s_light + m * Cfg<K>::kRec);
}

// ---------------------------------------------------------------------------------------------
// SG inner product of one (sg, other) pair: v = lambda d + Lambda D, lm = lambda + Lambda.
struct SgTerm { float um, E, X, c; };

__device__ __forceinline__ SgTerm sg_term(float vx, float vy, float vz, float lm) {
  SgTerm t;
  t.um = sqrtf(vx * vx + vy * vy + vz * vz);
  t.E = expf(t.um - lm);
  t.X = expf(-2.f * t.um);
  t.c = kTwoPi * t.E * (1.f - t.X) / t.um;
  return t;
}

// The sg side of point p: GENERAL reads it, LOBE builds the cosine lobe of the normal.
template <int K>
__device__ __forceinline__ void sg_side(const float* in, float* amp, float* dir, float& sharp) {
  if constexpr (K == GENERAL) {
    amp[0] = in[0]; amp[1] = in[1]; amp[2] = in[2];
    dir[0] = in[3]; dir[1] = in[4]; dir[2] = in[5];
    sharp = in[6];
  } else if constexpr (K == SPECULAR) {
    amp[0] = amp[1] = amp[2] = in[0];
    dir[0] = in[1]; dir[1] = in[2]; dir[2] = in[3];
    sharp = in[4];
  } else {
    amp[0] = amp[1] = amp[2] = 1.17f;
    dir[0] = in[0]; dir[1] = in[1]; dir[2] = in[2];
    sharp = 2.133f;
  }
}

struct Fit { float mu, x0, nn, y; bool b; };

__device__ __forceinline__ Fit fitted_term(const float* n, const float* r) {
  Fit f;
  f.mu = n[0] * r[0] + n[1] * r[1] + n[2] * r[2];
  f.x0 = 0.36f * f.mu;
  f.nn = f.x0 + r[9];
  f.b = fabsf(f.x0) <= r[9];
  f.y = f.b ? f.nn * f.nn / r[8] : fminf(fmaxf(f.mu, 0.f), 1.f);
  return f;
}

// SH9 bands of a (not necessarily unit) normal, times the band constants c_k.
__device__ __forceinline__ void sh9_bands(const float* n, float* b) {
  const float x = n[0], y = n[1], z = n[2];
  const float b1 = 2.f * kPi / 3.f, b2 = kPi / 4.f;
  b[0] = 0.28209479177f * kPi;
  b[1] = (-0.4886025119f * y) * b1;
  b[2] = (0.4886025119f * z) * b1;
  b[3] = (-0.4886025119f * x) * b1;
  b[4] = (1.0925484305920792f * (x * y)) * b2;
  b[5] = (-1.0925484305920792f * (y * z)) * b2;
  b[6] = (0.94617469575f * (z * z) - 0.31539156525f) * b2;
  b[7] = ((-1.0925484305920792f * x) * z) * b2;
  b[8] = (0.5462742152960396f * (x * x - y * y)) * b2;
}

// Forward contribution of one light to the pre-epilogue sum of one point.
template <int K>
__device__ __forceinline__ void pair_fwd(const float* in, const float* r, float* acc) {
  if constexpr (K == FITTED) {
    const Fit f = fitted_term(in, r);
    const float res = r[6] * f.y + r[7];
    acc[0] += res * r[3]; acc[1] += res * r[4]; acc[2] += res * r[5];
  } else if constexpr (K == SH9) {
    float b[9];
    sh9_bands(in, b);
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < 9; ++k) s += b[k] * r[k];
    acc[0] += s;
  } else {
    float amp[3], dir[3], sh;
    sg_side<K>(in, amp, dir, sh);
    const SgTerm t = sg_term(sh * dir[0] + r[3], sh * dir[1] + r[4], sh * dir[2] + r[5], sh + r[6]);
    acc[0] += amp[0] * r[0] * t.c; acc[1] += amp[1] * r[1] * t.c; acc[2] += amp[2] * r[2] * t.c;
  }
}

// Backward of one (point, light) pair: gpre = d loss / d pre-epilogue sum.  Adds the light's
// partials to la[kAcc] and, when `point` is set, the point's gradient to pg[kIn].
template <int K>
__device__ __forceinline__ void pair_bwd(const float* in, const float* gpre, const float* r, float* la, float* pg, bool point) {
  if constexpr (K == FITTED) {
    const Fit f = fitted_term(in, r);
    const float res = r[6] * f.y + r[7];
    const float G = gpre[0] * r[3] + gpre[1] * r[4] + gpre[2] * r[5];
    const float dydmu = f.b ? 2.f * f.nn * 0.36f / r[8] : ((f.mu >= 0.f && f.mu <= 1.f) ? 1.f : 0.f);
    const float dydl = f.b ? r[13] * (f.nn / r[8]) * (2.f * (1.f / (4.f * 0.36f)) - f.nn / r[8]) : 0.f;
    const float drdl = r[11] * f.y + r[6] * dydl + r[12];
    const float gmu = G * (r[6] * dydmu);
    la[0] += gpre[0] * res * r[14]; la[1] += gpre[1] * res * r[14]; la[2] += gpre[2] * res * r[14];
    la[3] += gmu * in[0]; la[4] += gmu * in[1]; la[5] += gmu * in[2];
    la[6] += G * drdl - G * res * r[10];
    if (point) { pg[0] += gmu * r[0]; pg[1] += gmu * r[1]; pg[2] += gmu * r[2]; }
  } else if constexpr (K == SH9) {
    float b[9];
    sh9_bands(in, b);
#pragma unroll
    for (int k = 0; k < 9; ++k) la[k] += gpre[0] * b[k];
    if (point) {
      const float x = in[0], y = in[1], z = in[2];
      const float b1 = 2.f * kPi / 3.f, b2 = kPi / 4.f;
      const float c1 = 0.4886025119f * b1, c2 = 1.0925484305920792f * b2;
      const float gx = -c1 * r[3] + c2 * y * r[4] - c2 * z * r[7] + 2.f * 0.5462742152960396f * b2 * x * r[8];
      const float gy = -c1 * r[1] + c2 * x * r[4] - c2 * z * r[5] - 2.f * 0.5462742152960396f * b2 * y * r[8];
      const float gz = c1 * r[2] - c2 * y * r[5] + 2.f * 0.94617469575f * b2 * z * r[6] - c2 * x * r[7];
      pg[0] += gpre[0] * gx; pg[1] += gpre[0] * gy; pg[2] += gpre[0] * gz;
    }
  } else {
    float amp[3], dir[3], sh;
    sg_side<K>(in, amp, dir, sh);
    const float vx = sh * dir[0] + r[3], vy = sh * dir[1] + r[4], vz = sh * dir[2] + r[5];
    const SgTerm t = sg_term(vx, vy, vz, sh + r[6]);
    const float t0 = gpre[0] * amp[0], t1 = gpre[1] * amp[1], t2 = gpre[2] * amp[2];
    const float Gc = t0 * r[0] + t1 * r[1] + t2 * r[2];
    const float dcdum = t.c + (2.f * kTwoPi * t.E * t.X - t.c) / t.um;
    const float s = Gc * dcdum / t.um;
    const float gx = s * vx, gy = s * vy, gz = s * vz;
    la[0] += t0 * t.c; la[1] += t1 * t.c; la[2] += t2 * t.c;
    la[3] += gx; la[4] += gy; la[5] += gz;
    la[6] += Gc * t.c;
    if (point) {
      pg[0] += gx; pg[1] += gy; pg[2] += gz;       // times the sg sharpness at the end
      if constexpr (K == GENERAL) {
        pg[3] += gpre[0] * r[0] * t.c; pg[4] += gpre[1] * r[1] * t.c; pg[5] += gpre[2] * r[2] * t.c;
        pg[6] += dir[0] * gx + dir[1] * gy + dir[2] * gz - Gc * t.c;
      } else if constexpr (K == SPECULAR) {     // one amplitude for the three channels
        pg[3] += (gpre[0] * r[0] + gpre[1] * r[1] + gpre[2] * r[2]) * t.c;
        pg[4] += dir[0] * gx + dir[1] * gy + dir[2] * gz - Gc * t.c;
      }
    }
  }
}

// ---------------------------------------------------------------------------------------------
// SPECULAR (sg_warp_specular_term), the reference's arithmetic in fp32.  x = normal n, roughness,
// view v of one point.  The lobe of sg_distribution_term is (1 / (pi m2), n, 2 / m2) with m2 =
// roughness^2; sg_warp_distribution turns it into (a, w, ws) with w = -v - 2 ((-v).n) n and
// ws = (2 / m2) / (4 max(n.v, 1e-4)).  The epilogue multiplies the lights' sum by the Smith terms
// V(ndl) V(ndv), Fresnel s + (1 - s) (1 - ldh)^5 and ndl.
__device__ __forceinline__ float clamp01(float v) { return v < 0.f ? 0.f : (v > 1.f ? 1.f : v); }   // NaN stays NaN
__device__ __forceinline__ bool in01(float v) { return v >= 0.f && v <= 1.f; }   // where torch.clamp(v, 0, 1) passes a gradient

struct Spec {
  float m2, a, sh0, nv, cnv, ws, w[3];                                      // the warped lobe
  float ndl_raw, ndl, ndv, q1, q2, V1, V2, hat[3], hn, ldh_raw, om, p5;    // the epilogue's factors
};

__device__ __forceinline__ Spec spec_geom(const float* x) {
  Spec s;
  const float* n = x;
  const float* v = x + 4;
  s.m2 = x[3] * x[3];
  s.sh0 = 2.f / s.m2;
  s.a = 1.f / (kPi * s.m2);
  s.nv = n[0] * v[0] + n[1] * v[1] + n[2] * v[2];
  s.cnv = s.nv < 1e-4f ? 1e-4f : s.nv;
  s.ws = s.sh0 / (4.f * s.cnv);
  const float t = 2.f * -s.nv;                       // 2 ((-v).n)
#pragma unroll
  for (int k = 0; k < 3; ++k) s.w[k] = -v[k] - t * n[k];
  s.ndl_raw = n[0] * s.w[0] + n[1] * s.w[1] + n[2] * s.w[2];
  s.ndl = clamp01(s.ndl_raw);
  s.ndv = clamp01(s.nv);
  const float h0 = s.w[0] + v[0], h1 = s.w[1] + v[1], h2 = s.w[2] + v[2];
  s.hn = sqrtf(h0 * h0 + h1 * h1 + h2 * h2);
  s.hat[0] = h0 / s.hn; s.hat[1] = h1 / s.hn; s.hat[2] = h2 / s.hn;
  s.ldh_raw = s.w[0] * s.hat[0] + s.w[1] * s.hat[1] + s.w[2] * s.hat[2];
  s.q1 = sqrtf(s.m2 + (1.f - s.m2) * s.ndl * s.ndl);
  s.q2 = sqrtf(s.m2 + (1.f - s.m2) * s.ndv * s.ndv);
  s.V1 = 1.f / (s.ndl + s.q1);
  s.V2 = 1.f / (s.ndv + s.q2);
  s.om = 1.f - clamp01(s.ldh_raw);
  const float om2 = s.om * s.om;
  s.p5 = om2 * om2 * s.om;
  return s;
}

__device__ __forceinline__ void load_spec_raw(const Args& a, int64_t p0, float (&x)[kPts][7]) {
  float n[kPts][3], r[kPts][1], v[kPts][3];
  load_rows<3>(a.normal, p0, a.n, n);
  load_rows<1>(a.rough, p0, a.n, r);
  load_rows<3>(a.view, p0, a.n, v);
#pragma unroll
  for (int p = 0; p < kPts; ++p) {
#pragma unroll
    for (int k = 0; k < 3; ++k) { x[p][k] = n[p][k]; x[p][4 + k] = v[p][k]; }
    x[p][3] = r[p][0];
  }
}

// Epilogue backward of one point: from the lights' sums acc, grad_out g and spec albedo sa, the
// gradient gpre of the sums, grad_spec_albedo gs, and eg = d loss / d (n.w, n.v, ldh) where their
// clamps pass a gradient, and d loss / d m2 through the Smith terms.
__device__ __forceinline__ void spec_epilogue_bwd(const Spec& s, const float* acc, const float* g, const float* sa,
                                                  float* gpre, float* gs, float* eg) {
  const float G = s.V1 * s.V2;
  float gG = 0.f, gndl = 0.f, gp5 = 0.f;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float F = sa[k] + (1.f - sa[k]) * s.p5;
    const float gy = ((acc[k] * G) * F) * s.ndl >= 0.f ? g[k] : 0.f;   // clamp(min=0)
    gpre[k] = gy * G * F * s.ndl;
    const float gF = gy * acc[k] * G * s.ndl;
    gs[k] = gF * (1.f - s.p5);
    gp5 += gF * (1.f - sa[k]);
    gG += gy * acc[k] * F * s.ndl;
    gndl += gy * acc[k] * G * F;
  }
  // V(x) = 1 / (x + q), q = sqrt(m2 + (1 - m2) x^2):  dV = -V^2 ((1 + (1 - m2) x / q) dx + (1 - x^2) / (2 q) dm2)
  const float d1 = -gG * s.V2 * s.V1 * s.V1, d2 = -gG * s.V1 * s.V2 * s.V2;
  gndl += d1 * (1.f + (1.f - s.m2) * s.ndl / s.q1);
  const float gndv = d2 * (1.f + (1.f - s.m2) * s.ndv / s.q2);
  eg[3] = d1 * (1.f - s.ndl * s.ndl) / (2.f * s.q1) + d2 * (1.f - s.ndv * s.ndv) / (2.f * s.q2);
  const float om2 = s.om * s.om;
  eg[0] = in01(s.ndl_raw) ? gndl : 0.f;
  eg[1] = in01(s.nv) ? gndv : 0.f;
  eg[2] = in01(s.ldh_raw) ? -5.f * (om2 * om2) * gp5 : 0.f;
}

// Prologue backward of one point: pg holds the light loop's d loss / d (ws w) (3), d / da and d / dws;
// writes d loss / d normal, roughness, view.
__device__ __forceinline__ void spec_point_bwd(const float* x, const Spec& s, const float* pg, const float* eg,
                                               float* gn, float& gr, float* gv) {
  const float* n = x;
  const float* v = x + 4;
  float gw[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) gw[k] = s.ws * pg[k];
  const float gsh0 = pg[4] / (4.f * s.cnv);
  const float gm2 = eg[3] - pg[3] * s.a / s.m2 - gsh0 * s.sh0 / s.m2;
  float gnv = eg[1] + (s.nv >= 1e-4f ? -pg[4] * s.ws / s.cnv : 0.f);
  // ldh = w . hat, hat = h / |h|, h = w + v
  const float hg = s.hat[0] * s.w[0] + s.hat[1] * s.w[1] + s.hat[2] * s.w[2];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    const float gh = eg[2] * (s.w[k] - s.hat[k] * hg) / s.hn;
    gw[k] += eg[2] * s.hat[k] + gh;
    gv[k] = gh;
  }
  // ndl = n . w
#pragma unroll
  for (int k = 0; k < 3; ++k) { gn[k] = eg[0] * s.w[k]; gw[k] += eg[0] * n[k]; }
  // w = -v + 2 (n.v) n, and every n.v
  gnv += 2.f * (gw[0] * n[0] + gw[1] * n[1] + gw[2] * n[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    gn[k] += 2.f * s.nv * gw[k] + gnv * v[k];
    gv[k] += gnv * n[k] - gw[k];
  }
  gr = gm2 * 2.f * x[3];
}

template <int K>
__device__ __forceinline__ void load_points(const Args& a, int64_t p0, float (&in)[kPts][Cfg<K>::kIn]) {
  if constexpr (K == GENERAL) {
    float am[kPts][3], di[kPts][3], sh[kPts][1];
    load_rows<3>(a.p_amp, p0, a.n, am);
    load_rows<3>(a.p_dir, p0, a.n, di);
    load_rows<1>(a.p_sharp, p0, a.n, sh);
#pragma unroll
    for (int p = 0; p < kPts; ++p) {
#pragma unroll
      for (int k = 0; k < 3; ++k) { in[p][k] = am[p][k]; in[p][3 + k] = di[p][k]; }
      in[p][6] = sh[p][0];
    }
  } else if constexpr (K == SPECULAR) {
    float x[kPts][7];
    load_spec_raw(a, p0, x);
#pragma unroll
    for (int p = 0; p < kPts; ++p) {
      const Spec s = spec_geom(x[p]);
      in[p][0] = s.a; in[p][1] = s.w[0]; in[p][2] = s.w[1]; in[p][3] = s.w[2]; in[p][4] = s.ws;
      in[p][5] = s.V1 * s.V2; in[p][6] = s.p5; in[p][7] = s.ndl;
    }
  } else {
    load_rows<3>(a.normal, p0, a.n, in);
  }
}

__device__ __forceinline__ float clamp0(float v) { return v < 0.f ? 0.f : v; }   // torch.clamp(min=0): NaN stays NaN

// ---------------------------------------------------------------------------------------------
template <int K>
__global__ void __launch_bounds__(kThreads, Cfg<K>::kFwdBlocks) lighting_fwd_kernel(Args a) {
  constexpr int R = Cfg<K>::kRec;
  __shared__ __align__(16) float s_light[kChunk * R];
  const int64_t tiles = (a.n + kTile - 1) / kTile;
  const int nchunks = (a.L + kChunk - 1) / kChunk;
  if (nchunks == 1) { stage_chunk<K>(a, 0, a.L, s_light); __syncthreads(); }
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t p0 = tile * kTile + (int64_t)threadIdx.x * kPts;
    float in[kPts][Cfg<K>::kIn];
    load_points<K>(a, p0, in);
    float acc[kPts][3] = {};
    for (int c = 0; c < nchunks; ++c) {
      const int cnt = min(kChunk, a.L - c * kChunk);
      if (nchunks > 1) { __syncthreads(); stage_chunk<K>(a, c * kChunk, cnt, s_light); __syncthreads(); }
      for (int m = 0; m < cnt; ++m) {
        float r[R];
#pragma unroll
        for (int q = 0; q < R / 4; ++q) *reinterpret_cast<float4*>(r + 4 * q) = reinterpret_cast<const float4*>(s_light + m * R)[q];
#pragma unroll
        for (int p = 0; p < kPts; ++p) pair_fwd<K>(in[p], r, acc[p]);
      }
    }
    if constexpr (K == SPECULAR) {
      float sa[kPts][3], o[kPts][3];
      load_rows<3>(a.albedo, p0, a.n, sa);
#pragma unroll
      for (int p = 0; p < kPts; ++p)
#pragma unroll
        for (int k = 0; k < 3; ++k)
          o[p][k] = clamp0(((acc[p][k] * in[p][5]) * (sa[p][k] + (1.f - sa[p][k]) * in[p][6])) * in[p][7]);
      store_rows<3>(a.out, p0, a.n, o);
    } else if (K == GENERAL) {
      store_rows<3>(a.out, p0, a.n, acc);
    } else if (K == SH9 && !a.albedo) {
      float o[kPts][1];
#pragma unroll
      for (int p = 0; p < kPts; ++p) o[p][0] = acc[p][0];
      store_rows<1>(a.out, p0, a.n, o);
    } else {
      float al[kPts][3] = {};
      if (a.albedo) load_rows<3>(a.albedo, p0, a.n, al);
      float o[kPts][3];
#pragma unroll
      for (int p = 0; p < kPts; ++p)
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (K == SH9) { o[p][k] = al[p][k] * acc[p][0]; continue; }
          const float e = clamp0(K == FITTED ? (a.L > 0 ? acc[p][k] / (float)a.L : 0.f) : acc[p][k]);
          o[p][k] = a.albedo ? e * (al[p][k] / kPi) : e;
        }
      store_rows<3>(a.out, p0, a.n, o);
    }
  }
}

template <int K>
__global__ void __launch_bounds__(kThreads, 2) lighting_bwd_kernel(Args a) {
  constexpr int R = Cfg<K>::kRec, A = Cfg<K>::kAcc, I = Cfg<K>::kIn;
  __shared__ __align__(16) float s_light[kChunk * R];
  __shared__ float s_red[kWarps][kChunk][A];
  const int64_t tiles = (a.n + kTile - 1) / kTile;
  const int nchunks = (a.L + kChunk - 1) / kChunk;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool want_light = a.partial != nullptr;
  const bool want_point = K == GENERAL    ? (a.g_amp || a.g_dir || a.g_sharp)
                          : K == SPECULAR ? (a.g_normal || a.g_rough || a.g_view)
                                          : a.g_normal != nullptr;
  const bool has_albedo = a.albedo != nullptr;
  // forward sums are needed for the clamp mask (SG models) or for grad_albedo (SH9)
  const bool need_pre = K == LOBE || K == FITTED || K == SPECULAR || (K == SH9 && a.g_albedo);
  float* part = want_light ? a.partial + (size_t)blockIdx.x * a.L * A : nullptr;
  if (want_light)
    for (int i = threadIdx.x; i < a.L * A; i += kThreads) part[i] = 0.f;
  if (nchunks == 1) { stage_chunk<K>(a, 0, a.L, s_light); }
  __syncthreads();
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t p0 = tile * kTile + (int64_t)threadIdx.x * kPts;
    float in[kPts][I];
    load_points<K>(a, p0, in);
    float g[kPts][3] = {}, al[kPts][3] = {};
    if (K == SH9 && !has_albedo) {        // sh9_irradiance: grad_out is (N,)
      float g1[kPts][1];
      load_rows<1>(a.grad_out, p0, a.n, g1);
#pragma unroll
      for (int p = 0; p < kPts; ++p) g[p][0] = g1[p][0];
    } else {
      load_rows<3>(a.grad_out, p0, a.n, g);
    }
    if (has_albedo) load_rows<3>(a.albedo, p0, a.n, al);
    // phase 1: the pre-epilogue sums
    float pre[kPts][3] = {};
    if (need_pre) {
      for (int c = 0; c < nchunks; ++c) {
        const int cnt = min(kChunk, a.L - c * kChunk);
        if (nchunks > 1) { __syncthreads(); stage_chunk<K>(a, c * kChunk, cnt, s_light); __syncthreads(); }
        for (int m = 0; m < cnt; ++m) {
          float r[R];
#pragma unroll
          for (int q = 0; q < R / 4; ++q) *reinterpret_cast<float4*>(r + 4 * q) = reinterpret_cast<const float4*>(s_light + m * R)[q];
#pragma unroll
          for (int p = 0; p < kPts; ++p) pair_fwd<K>(in[p], r, pre[p]);
        }
      }
    }
    // epilogue backward: gpre = d loss / d pre, and grad_albedo
    float gpre[kPts][3];
    float ga[kPts][3];
    float eg[kPts][4];                      // SPECULAR: spec_epilogue_bwd
    float sx[kPts][7];
    if constexpr (K == SPECULAR) load_spec_raw(a, p0, sx);
#pragma unroll
    for (int p = 0; p < kPts; ++p) {
      const bool valid = p0 + p < a.n;
      if constexpr (K == SPECULAR) {
        spec_epilogue_bwd(spec_geom(sx[p]), pre[p], g[p], al[p], gpre[p], ga[p], eg[p]);
      } else if (K == SH9) {
        gpre[p][0] = has_albedo ? g[p][0] * al[p][0] + g[p][1] * al[p][1] + g[p][2] * al[p][2] : g[p][0];
        gpre[p][1] = gpre[p][2] = 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) ga[p][k] = g[p][k] * pre[p][0];
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          if (K == GENERAL) { gpre[p][k] = g[p][k]; ga[p][k] = 0.f; continue; }
          const float x = K == FITTED ? (a.L > 0 ? pre[p][k] / (float)a.L : 0.f) : pre[p][k];
          const float gE = has_albedo ? g[p][k] * (al[p][k] / kPi) : g[p][k];
          gpre[p][k] = x >= 0.f ? (K == FITTED ? gE / (float)a.L : gE) : 0.f;
          ga[p][k] = g[p][k] * clamp0(x) / kPi;
        }
      }
      if (!valid) gpre[p][0] = gpre[p][1] = gpre[p][2] = 0.f;
    }
    if (a.g_albedo) store_rows<3>(a.g_albedo, p0, a.n, ga);
    // phase 2: light partials and per-point gradients
    float pg[kPts][I] = {};
    if (want_light || want_point) {
      for (int c = 0; c < nchunks; ++c) {
        const int cnt = min(kChunk, a.L - c * kChunk);
        if (nchunks > 1) { __syncthreads(); stage_chunk<K>(a, c * kChunk, cnt, s_light); __syncthreads(); }
        for (int m = 0; m < cnt; ++m) {
          float r[R];
#pragma unroll
          for (int q = 0; q < R / 4; ++q) *reinterpret_cast<float4*>(r + 4 * q) = reinterpret_cast<const float4*>(s_light + m * R)[q];
          float la[A] = {};
#pragma unroll
          for (int p = 0; p < kPts; ++p)
            if (p0 + p < a.n) pair_bwd<K>(in[p], gpre[p], r, la, pg[p], want_point);
          if (want_light) {
#pragma unroll
            for (int j = 0; j < A; ++j) {
#pragma unroll
              for (int o = 16; o > 0; o >>= 1) la[j] += __shfl_xor_sync(0xffffffffu, la[j], o);
            }
            if (lane == 0)
#pragma unroll
              for (int j = 0; j < A; ++j) s_red[warp][m][j] = la[j];
          }
        }
        if (want_light) {
          __syncthreads();
          for (int i = threadIdx.x; i < cnt * A; i += kThreads) {
            const int m = i / A, j = i - m * A;
            float s = 0.f;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) s += s_red[w][m][j];
            part[(size_t)(c * kChunk + m) * A + j] += s;
          }
          __syncthreads();
        }
      }
    }
    if (want_point) {
      if constexpr (K == GENERAL) {
        float o[kPts][3], o1[kPts][1];
        if (a.g_amp) {
#pragma unroll
          for (int p = 0; p < kPts; ++p) { o[p][0] = pg[p][3]; o[p][1] = pg[p][4]; o[p][2] = pg[p][5]; }
          store_rows<3>(a.g_amp, p0, a.n, o);
        }
        if (a.g_dir) {
#pragma unroll
          for (int p = 0; p < kPts; ++p) { o[p][0] = in[p][6] * pg[p][0]; o[p][1] = in[p][6] * pg[p][1]; o[p][2] = in[p][6] * pg[p][2]; }
          store_rows<3>(a.g_dir, p0, a.n, o);
        }
        if (a.g_sharp) {
#pragma unroll
          for (int p = 0; p < kPts; ++p) o1[p][0] = pg[p][6];
          store_rows<1>(a.g_sharp, p0, a.n, o1);
        }
      } else if constexpr (K == SPECULAR) {
        load_spec_raw(a, p0, sx);
        float on[kPts][3], orr[kPts][1], ov[kPts][3];
#pragma unroll
        for (int p = 0; p < kPts; ++p) spec_point_bwd(sx[p], spec_geom(sx[p]), pg[p], eg[p], on[p], orr[p][0], ov[p]);
        if (a.g_normal) store_rows<3>(a.g_normal, p0, a.n, on);
        if (a.g_rough) store_rows<1>(a.g_rough, p0, a.n, orr);
        if (a.g_view) store_rows<3>(a.g_view, p0, a.n, ov);
      } else {
        float o[kPts][3];
        const float s = K == LOBE ? 2.133f : 1.f;
#pragma unroll
        for (int p = 0; p < kPts; ++p) { o[p][0] = s * pg[p][0]; o[p][1] = s * pg[p][1]; o[p][2] = s * pg[p][2]; }
        store_rows<3>(a.g_normal, p0, a.n, o);
      }
    }
  }
}

// Sums the per-CTA partials of each light in CTA order, in fp64, and writes the light gradients.
template <int K>
__global__ void __launch_bounds__(128) lighting_finalize_kernel(Args a, int ctas) {
  constexpr int A = Cfg<K>::kAcc;
  const int m = blockIdx.x * blockDim.x + threadIdx.x;
  if (m >= a.L) return;
  double s[A];
#pragma unroll
  for (int j = 0; j < A; ++j) s[j] = 0.0;
  for (int c = 0; c < ctas; ++c) {
    const float* q = a.partial + ((size_t)c * a.L + m) * A;
#pragma unroll
    for (int j = 0; j < A; ++j) s[j] += (double)q[j];
  }
  if (K == SH9) {
    if (a.gl_amp)
#pragma unroll
      for (int j = 0; j < 9; ++j) a.gl_amp[j] = (float)s[j];
    return;
  }
  if (a.gl_amp)
#pragma unroll
    for (int k = 0; k < 3; ++k) a.gl_amp[3 * m + k] = (float)s[k];
  if (K == FITTED) {
    if (a.gl_dir)
#pragma unroll
      for (int k = 0; k < 3; ++k) a.gl_dir[3 * m + k] = (float)s[3 + k];
    if (a.gl_sharp) a.gl_sharp[m] = (float)s[6];
    return;
  }
  // v = lambda d + Lambda D:  dL/dD = Lambda sum(gv),  dL/dLambda = D . sum(gv) - sum(Gc c)
  const double lb = __ldg(a.l_sharp + m);
  const double D0 = __ldg(a.l_dir + 3 * m), D1 = __ldg(a.l_dir + 3 * m + 1), D2 = __ldg(a.l_dir + 3 * m + 2);
  if (a.gl_dir)
#pragma unroll
    for (int k = 0; k < 3; ++k) a.gl_dir[3 * m + k] = (float)(lb * s[3 + k]);
  if (a.gl_sharp) a.gl_sharp[m] = (float)(D0 * s[3] + D1 * s[4] + D2 * s[5] - s[6]);
}

template <int K>
int launch_fwd(const Args& a, cudaStream_t st) {
  const int64_t tiles = (a.n + kTile - 1) / kTile;
  if (tiles == 0) return 0;
  const int64_t ctas = (int64_t)kSms * Cfg<K>::kFwdBlocks;
  lighting_fwd_kernel<K><<<(unsigned)(tiles < ctas ? tiles : ctas), kThreads, 0, st>>>(a);
  return (int)cudaGetLastError();
}

template <int K>
int launch_bwd(const Args& a, cudaStream_t st) {
  const int64_t tiles = (a.n + kTile - 1) / kTile;
  const int ctas = (int)(tiles < kBwdCtas ? tiles : kBwdCtas);
  if (ctas > 0) lighting_bwd_kernel<K><<<ctas, kThreads, 0, st>>>(a);
  if (a.partial && a.L > 0) lighting_finalize_kernel<K><<<(a.L + 127) / 128, 128, 0, st>>>(a, ctas);
  return (int)cudaGetLastError();
}

// The workspace of a backward whose light gradients take `floats` partial sums per light.
dibr_layout::LightingLayout partials(int floats, int lights) { return dibr_layout::lighting_layout(kBwdCtas, floats, lights); }

// The partial sums of l in the workspace, or NULL when it does not fit.
float* carve_partials(const dibr_layout::LightingLayout& l, void* workspace, size_t workspace_bytes) {
  char* o = dibr_layout::carve(workspace, workspace_bytes, l.bytes);
  return o ? dibr_layout::piece<float>(o, l.partial) : nullptr;
}

// ---------------------------------------------------------------------------------------------
// SHADE (sg_shade of kaolin/render/easy_render/mesh.py): deferred shading of a (B, H, W) G-buffer, one
// point per pixel.  A background pixel (face_idx < 0) gives exactly 0 and takes no part in the light
// gradients; a covered one normalises its normal as F.normalize does, generates its view ray, and
// evaluates the LOBE (diffuse) and SPECULAR pairs against each staged light, so each light is staged
// and read once for both terms.  Both lobes' light partials go into the same 7-float slot: the
// finalize step is linear in them.  A warp whose 32 pixels are all background skips the light loop.
constexpr int kCam = 16;   // floats per view: R (row-major), tan_x, tan_y, x0, y0, camera width, height, 0

struct ShadeArgs {
  Args a;                  // a.n = B H W pixels; the lights, their gradients and the partial slots
  int H, W;
  const int64_t* face_idx;
  const float* cam;
  const float* normal; const float* albedo; const float* spec_albedo; const float* rough;
  float* diffuse; float* specular; float* img;
  const float* g_diffuse; const float* g_specular; const float* g_img;
  float* g_normal; float* g_albedo; float* g_spec_albedo; float* g_rough;
};

// Which of a thread's P pixels are covered; whether any of its warp's are.
template <int P>
__device__ __forceinline__ bool shade_mask(const ShadeArgs& s, int64_t p0, bool (&cov)[P]) {
  bool any = false;
#pragma unroll
  for (int q = 0; q < P; ++q) {
    cov[q] = p0 + q < s.a.n && __ldg(s.face_idx + p0 + q) >= 0;
    any |= cov[q];
  }
  return __any_sync(0xffffffffu, any);
}

// The view of pixel (i, j): -normalize(R^T d), d the pinhole ray of kaolin/render/camera/raygen.py
// through the pixel centre of the custom-resolution grid (scale = camera size / G-buffer size), in the
// reference's fp32 operations and their order.
__device__ __forceinline__ void shade_view(const float* __restrict__ cam, int H, int W, int i, int j, float* v) {
  const float cw = __ldg(cam + 13), ch = __ldg(cam + 14);
  const float sx = __fdiv_rn(cw, (float)W), sy = __fdiv_rn(ch, (float)H);
  const float px = __fsub_rn(__fadd_rn(__fmul_rn(sx, (float)j), __fmul_rn(sx, 0.5f)), __ldg(cam + 11));
  const float py = __fadd_rn(__fadd_rn(__fmul_rn(sy, (float)i), __fmul_rn(sy, 0.5f)), __ldg(cam + 12));
  const float d0 = __fmul_rn(__fsub_rn(__fmul_rn(2.f, __fdiv_rn(px, cw)), 1.f), __ldg(cam + 9));
  const float d1 = __fmul_rn(-__fsub_rn(__fmul_rn(2.f, __fdiv_rn(py, ch)), 1.f), __ldg(cam + 10));
  float w[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) w[k] = __ldg(cam + k) * d0 + __ldg(cam + 3 + k) * d1 - __ldg(cam + 6 + k);
  const float len = sqrtf(w[0] * w[0] + w[1] * w[1] + w[2] * w[2]);
#pragma unroll
  for (int k = 0; k < 3; ++k) v[k] = -(w[k] / len);
}

// Per pixel: x7 = (unit normal, roughness, view), the raw layout of spec_geom; dn = max(|normal|, 1e-12).
template <int P>
__device__ __forceinline__ void shade_points(const ShadeArgs& s, int64_t p0, float (&x7)[P][7], float (&dn)[P]) {
  float x[P][3], r[P][1];
  load_rows<3>(s.normal, p0, s.a.n, x);
  load_rows<1>(s.rough, p0, s.a.n, r);
  const int64_t hw = (int64_t)s.H * s.W;
  int64_t b = p0 / hw;
  const int rem = (int)(p0 - b * hw);
  int i = rem / s.W, j = rem - i * s.W;
#pragma unroll
  for (int q = 0; q < P; ++q) {
    const float len = sqrtf(x[q][0] * x[q][0] + x[q][1] * x[q][1] + x[q][2] * x[q][2]);
    dn[q] = len < 1e-12f ? 1e-12f : len;       // clamp_min: NaN stays NaN
#pragma unroll
    for (int k = 0; k < 3; ++k) x7[q][k] = x[q][k] / dn[q];
    x7[q][3] = r[q][0];
    if (p0 + q < s.a.n) shade_view(s.cam + kCam * b, s.H, s.W, i, j, x7[q] + 4);
    else x7[q][4] = x7[q][5] = x7[q][6] = 0.f;
    if (++j == s.W) { j = 0; if (++i == s.H) { i = 0; ++b; } }
  }
}

// SPECULAR's per-point record (load_points<SPECULAR>) from x7.
__device__ __forceinline__ void shade_spec_in(const float* x7, float* in) {
  const Spec g = spec_geom(x7);
  in[0] = g.a; in[1] = g.w[0]; in[2] = g.w[1]; in[3] = g.w[2]; in[4] = g.ws;
  in[5] = g.V1 * g.V2; in[6] = g.p5; in[7] = g.ndl;
}

template <int P>
__device__ __forceinline__ void shade_pairs_fwd(const float* s_light, int cnt, const float (&x7)[P][7],
                                                const float (&sp)[P][8], float (&accd)[P][3], float (&accs)[P][3]) {
  constexpr int R = Cfg<SHADE>::kRec;
  for (int m = 0; m < cnt; ++m) {
    float r[R];
#pragma unroll
    for (int q = 0; q < R / 4; ++q) *reinterpret_cast<float4*>(r + 4 * q) = reinterpret_cast<const float4*>(s_light + m * R)[q];
#pragma unroll
    for (int p = 0; p < P; ++p) {
      pair_fwd<LOBE>(x7[p], r, accd[p]);
      pair_fwd<SPECULAR>(sp[p], r, accs[p]);
    }
  }
}

template <int P>
__global__ void __launch_bounds__(kThreads, Cfg<SHADE>::kFwdBlocks) shade_fwd_kernel(ShadeArgs s) {
  constexpr int T = kThreads * P;
  __shared__ __align__(16) float s_light[kChunk * Cfg<SHADE>::kRec];
  const Args& a = s.a;
  const int64_t tiles = (a.n + T - 1) / T;
  const int nchunks = (a.L + kChunk - 1) / kChunk;
  if (nchunks == 1) { stage_chunk<SHADE>(a, 0, a.L, s_light); __syncthreads(); }
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t p0 = tile * T + (int64_t)threadIdx.x * P;
    bool cov[P];
    const bool active = shade_mask(s, p0, cov);
    float x7[P][Cfg<SHADE>::kIn] = {}, dn[P], sp[P][8] = {};
    float accd[P][3] = {}, accs[P][3] = {}, al[P][3] = {}, sa[P][3] = {};
    if (active) {
      shade_points(s, p0, x7, dn);
#pragma unroll
      for (int p = 0; p < P; ++p) shade_spec_in(x7[p], sp[p]);
    }
    for (int c = 0; c < nchunks; ++c) {
      const int cnt = min(kChunk, a.L - c * kChunk);
      if (nchunks > 1) { __syncthreads(); stage_chunk<SHADE>(a, c * kChunk, cnt, s_light); __syncthreads(); }
      if (active) shade_pairs_fwd(s_light, cnt, x7, sp, accd, accs);
    }
    if (active) {
      load_rows<3>(s.albedo, p0, a.n, al);
      load_rows<3>(s.spec_albedo, p0, a.n, sa);
    }
    float od[P][3], os[P][3], oi[P][3];
#pragma unroll
    for (int p = 0; p < P; ++p)
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const float d = clamp0(accd[p][k]) * (al[p][k] / kPi);
        const float e = clamp0(((accs[p][k] * sp[p][5]) * (sa[p][k] + (1.f - sa[p][k]) * sp[p][6])) * sp[p][7]);
        od[p][k] = cov[p] ? d : 0.f;
        os[p][k] = cov[p] ? e : 0.f;
        oi[p][k] = cov[p] ? d + e : 0.f;
      }
    store_rows<3>(s.diffuse, p0, a.n, od);
    store_rows<3>(s.specular, p0, a.n, os);
    store_rows<3>(s.img, p0, a.n, oi);
  }
}

// d loss / d diffuse and d loss / d specular of each pixel: each output's gradient plus img's.
template <int P>
__device__ __forceinline__ void shade_grads(const ShadeArgs& s, int64_t p0, float (&gd)[P][3], float (&gs)[P][3]) {
  if (s.g_diffuse) load_rows<3>(s.g_diffuse, p0, s.a.n, gd);
  if (s.g_specular) load_rows<3>(s.g_specular, p0, s.a.n, gs);
  if (s.g_img) {
    float gi[P][3];
    load_rows<3>(s.g_img, p0, s.a.n, gi);
#pragma unroll
    for (int p = 0; p < P; ++p)
#pragma unroll
      for (int k = 0; k < 3; ++k) { gd[p][k] += gi[p][k]; gs[p][k] += gi[p][k]; }
  }
}

template <int P>
__global__ void __launch_bounds__(kThreads, 2) shade_bwd_kernel(ShadeArgs s) {
  constexpr int R = Cfg<SHADE>::kRec, A = Cfg<SHADE>::kAcc, T = kThreads * P;
  __shared__ __align__(16) float s_light[kChunk * R];
  __shared__ float s_red[kWarps][kChunk][A];
  const Args& a = s.a;
  const int64_t tiles = (a.n + T - 1) / T;
  const int nchunks = (a.L + kChunk - 1) / kChunk;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool want_light = a.partial != nullptr;
  const bool want_point = s.g_normal || s.g_rough;
  float* part = want_light ? a.partial + (size_t)blockIdx.x * a.L * A : nullptr;
  if (want_light)
    for (int i = threadIdx.x; i < a.L * A; i += kThreads) part[i] = 0.f;
  if (nchunks == 1) { stage_chunk<SHADE>(a, 0, a.L, s_light); }
  __syncthreads();
  for (int64_t tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    const int64_t p0 = tile * T + (int64_t)threadIdx.x * P;
    bool cov[P];
    const bool active = shade_mask(s, p0, cov);
    float x7[P][7] = {}, dn[P] = {}, sp[P][8] = {};
    float gd[P][3] = {}, gs[P][3] = {}, al[P][3] = {}, sa[P][3] = {};
    if (active) {
      shade_points(s, p0, x7, dn);
#pragma unroll
      for (int p = 0; p < P; ++p) shade_spec_in(x7[p], sp[p]);
      shade_grads(s, p0, gd, gs);
      load_rows<3>(s.albedo, p0, a.n, al);
      load_rows<3>(s.spec_albedo, p0, a.n, sa);
    }
    // phase 1: both lobes' sums, for the clamp masks and the epilogues
    float pred[P][3] = {}, pres[P][3] = {};
    for (int c = 0; c < nchunks; ++c) {
      const int cnt = min(kChunk, a.L - c * kChunk);
      if (nchunks > 1) { __syncthreads(); stage_chunk<SHADE>(a, c * kChunk, cnt, s_light); __syncthreads(); }
      if (active) shade_pairs_fwd(s_light, cnt, x7, sp, pred, pres);
    }
    // epilogue backward: the LOBE epilogue of the diffuse term, spec_epilogue_bwd of the specular one
    float gpd[P][3], gps[P][3], ga[P][3], gsa[P][3], eg[P][4] = {};
#pragma unroll
    for (int p = 0; p < P; ++p) {
      if (cov[p]) {
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          gpd[p][k] = pred[p][k] >= 0.f ? gd[p][k] * (al[p][k] / kPi) : 0.f;
          ga[p][k] = gd[p][k] * clamp0(pred[p][k]) / kPi;
        }
        spec_epilogue_bwd(spec_geom(x7[p]), pres[p], gs[p], sa[p], gps[p], gsa[p], eg[p]);
      } else {
#pragma unroll
        for (int k = 0; k < 3; ++k) gpd[p][k] = gps[p][k] = ga[p][k] = gsa[p][k] = 0.f;
      }
    }
    if (s.g_albedo) store_rows<3>(s.g_albedo, p0, a.n, ga);
    if (s.g_spec_albedo) store_rows<3>(s.g_spec_albedo, p0, a.n, gsa);
    // phase 2: light partials of both lobes into one slot, and the per-pixel gradients
    float pgd[P][3] = {}, pgs[P][5] = {};
    if (want_light || want_point) {
      for (int c = 0; c < nchunks; ++c) {
        const int cnt = min(kChunk, a.L - c * kChunk);
        if (nchunks > 1) { __syncthreads(); stage_chunk<SHADE>(a, c * kChunk, cnt, s_light); __syncthreads(); }
        for (int m = 0; m < cnt; ++m) {
          float la[A] = {};
          if (active) {
            float r[R];
#pragma unroll
            for (int q = 0; q < R / 4; ++q) *reinterpret_cast<float4*>(r + 4 * q) = reinterpret_cast<const float4*>(s_light + m * R)[q];
#pragma unroll
            for (int p = 0; p < P; ++p)
              if (cov[p]) {
                pair_bwd<LOBE>(x7[p], gpd[p], r, la, pgd[p], want_point);
                pair_bwd<SPECULAR>(sp[p], gps[p], r, la, pgs[p], want_point);
              }
            if (want_light) {
#pragma unroll
              for (int j = 0; j < A; ++j) {
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) la[j] += __shfl_xor_sync(0xffffffffu, la[j], o);
              }
            }
          }
          if (want_light && lane == 0)
#pragma unroll
            for (int j = 0; j < A; ++j) s_red[warp][m][j] = la[j];
        }
        if (want_light) {
          __syncthreads();
          for (int i = threadIdx.x; i < cnt * A; i += kThreads) {
            const int m = i / A, j = i - m * A;
            float sum = 0.f;
#pragma unroll
            for (int w = 0; w < kWarps; ++w) sum += s_red[w][m][j];
            part[(size_t)(c * kChunk + m) * A + j] += sum;
          }
          __syncthreads();
        }
      }
    }
    if (want_point) {
      float on[P][3] = {}, orr[P][1] = {};
#pragma unroll
      for (int p = 0; p < P; ++p) {
        if (!cov[p]) continue;
        float gn[3], gv[3];
        spec_point_bwd(x7[p], spec_geom(x7[p]), pgs[p], eg[p], gn, orr[p][0], gv);
#pragma unroll
        for (int k = 0; k < 3; ++k) gn[k] += 2.133f * pgd[p][k];
        // n = x / max(|x|, eps): (g - n (n.g)) / |x| where |x| >= eps, g / eps below
        const float* n = x7[p];
        const float ng = dn[p] > 1e-12f ? n[0] * gn[0] + n[1] * gn[1] + n[2] * gn[2] : 0.f;
#pragma unroll
        for (int k = 0; k < 3; ++k) on[p][k] = (gn[k] - n[k] * ng) / dn[p];
      }
      if (s.g_normal) store_rows<3>(s.g_normal, p0, a.n, on);
      if (s.g_rough) store_rows<1>(s.g_rough, p0, a.n, orr);
    }
  }
}

int launch_shade_fwd(const ShadeArgs& s, cudaStream_t st) {
  constexpr int P = Cfg<SHADE>::pts(false);
  const int64_t tiles = (s.a.n + kThreads * P - 1) / (kThreads * P);
  if (tiles == 0) return 0;
  const int64_t ctas = (int64_t)kSms * Cfg<SHADE>::kFwdBlocks;
  shade_fwd_kernel<P><<<(unsigned)(tiles < ctas ? tiles : ctas), kThreads, 0, st>>>(s);
  return (int)cudaGetLastError();
}

int launch_shade_bwd(const ShadeArgs& s, cudaStream_t st) {
  constexpr int P = Cfg<SHADE>::pts(true);
  const int64_t tiles = (s.a.n + kThreads * P - 1) / (kThreads * P);
  const int ctas = (int)(tiles < kBwdCtas ? tiles : kBwdCtas);
  if (ctas > 0) shade_bwd_kernel<P><<<ctas, kThreads, 0, st>>>(s);
  if (s.a.partial && s.a.L > 0) lighting_finalize_kernel<SHADE><<<(s.a.L + 127) / 128, 128, 0, st>>>(s.a, ctas);
  return (int)cudaGetLastError();
}

}  // namespace

extern "C" {

size_t dibr_b200_sg_inner_product_workspace_bytes(int num_other) {
  return num_other < 0 ? 0 : partials(Cfg<GENERAL>::kAcc, num_other).bytes;
}

int dibr_b200_sg_inner_product_forward(int64_t num_sg, int num_other, const float* amplitude, const float* direction,
                                       const float* sharpness, const float* other_amplitude,
                                       const float* other_direction, const float* other_sharpness, float* out,
                                       dibr_b200_stream_t stream) {
  if (num_sg < 0 || num_other < 0) return DIBR_B200_EINVAL;
  if (num_sg == 0) return 0;
  if (!amplitude || !direction || !sharpness || !out) return DIBR_B200_EINVAL;
  if (num_other > 0 && (!other_amplitude || !other_direction || !other_sharpness)) return DIBR_B200_EINVAL;
  Args a = {};
  a.n = num_sg; a.L = num_other;
  a.p_amp = amplitude; a.p_dir = direction; a.p_sharp = sharpness;
  a.l_amp = other_amplitude; a.l_dir = other_direction; a.l_sharp = other_sharpness;
  a.out = out;
  return launch_fwd<GENERAL>(a, (cudaStream_t)stream);
}

int dibr_b200_sg_inner_product_backward(int64_t num_sg, int num_other, const float* grad_out, const float* amplitude,
                                        const float* direction, const float* sharpness, const float* other_amplitude,
                                        const float* other_direction, const float* other_sharpness,
                                        float* grad_amplitude, float* grad_direction, float* grad_sharpness,
                                        float* grad_other_amplitude, float* grad_other_direction,
                                        float* grad_other_sharpness, void* workspace, size_t workspace_bytes,
                                        dibr_b200_stream_t stream) {
  if (num_sg < 0 || num_other < 0) return DIBR_B200_EINVAL;
  if (num_sg > 0 && (!grad_out || !amplitude || !direction || !sharpness)) return DIBR_B200_EINVAL;
  if (num_other > 0 && (!other_amplitude || !other_direction || !other_sharpness)) return DIBR_B200_EINVAL;
  Args a = {};
  a.n = num_sg; a.L = num_other;
  a.p_amp = amplitude; a.p_dir = direction; a.p_sharp = sharpness;
  a.l_amp = other_amplitude; a.l_dir = other_direction; a.l_sharp = other_sharpness;
  a.grad_out = grad_out;
  a.g_amp = grad_amplitude; a.g_dir = grad_direction; a.g_sharp = grad_sharpness;
  a.gl_amp = grad_other_amplitude; a.gl_dir = grad_other_direction; a.gl_sharp = grad_other_sharpness;
  if (num_other > 0 && (a.gl_amp || a.gl_dir || a.gl_sharp)) {
    if (!workspace) return DIBR_B200_EINVAL;
    a.partial = carve_partials(partials(Cfg<GENERAL>::kAcc, num_other), workspace, workspace_bytes);
    if (!a.partial) return DIBR_B200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (num_other == 0) {   // empty sum: every sg-side gradient is zero
    const size_t b3 = (size_t)num_sg * 3 * sizeof(float);
    if (grad_amplitude && cudaMemsetAsync(grad_amplitude, 0, b3, st) != cudaSuccess) return (int)cudaGetLastError();
    if (grad_direction && cudaMemsetAsync(grad_direction, 0, b3, st) != cudaSuccess) return (int)cudaGetLastError();
    if (grad_sharpness && cudaMemsetAsync(grad_sharpness, 0, b3 / 3, st) != cudaSuccess) return (int)cudaGetLastError();
    return 0;
  }
  return launch_bwd<GENERAL>(a, st);
}

// The workspace of a diffuse backward with light gradients; SH9 has one light of 9 coefficients.
static dibr_layout::LightingLayout diffuse_partials(int model, int num_lights) {
  switch (model) {
    case DIBR_B200_LIGHT_SG_INNER_PRODUCT: return partials(Cfg<LOBE>::kAcc, num_lights);
    case DIBR_B200_LIGHT_SG_FITTED: return partials(Cfg<FITTED>::kAcc, num_lights);
    default: return partials(Cfg<SH9>::kAcc, 1);
  }
}

size_t dibr_b200_diffuse_workspace_bytes(int model, int num_lights) {
  if (num_lights < 0) return 0;
  switch (model) {
    case DIBR_B200_LIGHT_SG_INNER_PRODUCT: case DIBR_B200_LIGHT_SG_FITTED: case DIBR_B200_LIGHT_SH9:
      return diffuse_partials(model, num_lights).bytes;
    default: return 0;
  }
}

static int diffuse_args(Args& a, int model, int64_t num_points, int num_lights, const float* light_amplitude,
                        const float* light_direction, const float* light_sharpness, const float* normal,
                        const float* albedo) {
  if (num_points < 0 || num_lights < 0) return DIBR_B200_EINVAL;
  if (model == DIBR_B200_LIGHT_SH9) {
    if (num_lights != 1 || !light_amplitude) return DIBR_B200_EINVAL;
  } else if (model == DIBR_B200_LIGHT_SG_INNER_PRODUCT || model == DIBR_B200_LIGHT_SG_FITTED) {
    if (num_lights > 0 && (!light_amplitude || !light_direction || !light_sharpness)) return DIBR_B200_EINVAL;
  } else {
    return DIBR_B200_EINVAL;
  }
  if (num_points > 0 && !normal) return DIBR_B200_EINVAL;
  a = Args{};
  a.n = num_points; a.L = num_lights;
  a.normal = normal; a.albedo = albedo;
  a.l_amp = light_amplitude; a.l_dir = light_direction; a.l_sharp = light_sharpness;
  return 0;
}

int dibr_b200_diffuse_forward(int model, int64_t num_points, int num_lights, const float* light_amplitude,
                              const float* light_direction, const float* light_sharpness, const float* normal,
                              const float* albedo, float* out, dibr_b200_stream_t stream) {
  Args a;
  const int rc = diffuse_args(a, model, num_points, num_lights, light_amplitude, light_direction, light_sharpness,
                              normal, albedo);
  if (rc) return rc;
  if (num_points > 0 && !out) return DIBR_B200_EINVAL;
  a.out = out;
  cudaStream_t st = (cudaStream_t)stream;
  switch (model) {
    case DIBR_B200_LIGHT_SG_INNER_PRODUCT: return launch_fwd<LOBE>(a, st);
    case DIBR_B200_LIGHT_SG_FITTED: return launch_fwd<FITTED>(a, st);
    default: return launch_fwd<SH9>(a, st);
  }
}

int dibr_b200_diffuse_backward(int model, int64_t num_points, int num_lights, const float* light_amplitude,
                               const float* light_direction, const float* light_sharpness, const float* normal,
                               const float* albedo, const float* grad_out, float* grad_normal, float* grad_albedo,
                               float* grad_light_amplitude, float* grad_light_direction,
                               float* grad_light_sharpness, void* workspace, size_t workspace_bytes,
                               dibr_b200_stream_t stream) {
  Args a;
  const int rc = diffuse_args(a, model, num_points, num_lights, light_amplitude, light_direction, light_sharpness,
                              normal, albedo);
  if (rc) return rc;
  if (num_points > 0 && !grad_out) return DIBR_B200_EINVAL;
  if (grad_albedo && !albedo) return DIBR_B200_EINVAL;
  a.grad_out = grad_out;
  a.g_normal = grad_normal; a.g_albedo = grad_albedo;
  a.gl_amp = grad_light_amplitude;
  if (model != DIBR_B200_LIGHT_SH9) { a.gl_dir = grad_light_direction; a.gl_sharp = grad_light_sharpness; }
  if (num_lights > 0 && (a.gl_amp || a.gl_dir || a.gl_sharp)) {
    if (!workspace) return DIBR_B200_EINVAL;
    a.partial = carve_partials(diffuse_partials(model, num_lights), workspace, workspace_bytes);
    if (!a.partial) return DIBR_B200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (num_lights == 0) {   // empty sum: zero irradiance, zero per-point gradients
    const size_t b3 = (size_t)num_points * 3 * sizeof(float);
    if (grad_normal && cudaMemsetAsync(grad_normal, 0, b3, st) != cudaSuccess) return (int)cudaGetLastError();
    if (grad_albedo && cudaMemsetAsync(grad_albedo, 0, b3, st) != cudaSuccess) return (int)cudaGetLastError();
    return 0;
  }
  switch (model) {
    case DIBR_B200_LIGHT_SG_INNER_PRODUCT: return launch_bwd<LOBE>(a, st);
    case DIBR_B200_LIGHT_SG_FITTED: return launch_bwd<FITTED>(a, st);
    default: return launch_bwd<SH9>(a, st);
  }
}

size_t dibr_b200_specular_workspace_bytes(int num_lights) {
  return num_lights < 0 ? 0 : partials(Cfg<SPECULAR>::kAcc, num_lights).bytes;
}

static int specular_args(Args& a, int64_t num_points, int num_lights, const float* light_amplitude,
                         const float* light_direction, const float* light_sharpness, const float* normal,
                         const float* roughness, const float* view, const float* spec_albedo) {
  if (num_points < 0 || num_lights < 0) return DIBR_B200_EINVAL;
  if (num_lights > 0 && (!light_amplitude || !light_direction || !light_sharpness)) return DIBR_B200_EINVAL;
  if (num_points > 0 && (!normal || !roughness || !view || !spec_albedo)) return DIBR_B200_EINVAL;
  a = Args{};
  a.n = num_points; a.L = num_lights;
  a.normal = normal; a.rough = roughness; a.view = view; a.albedo = spec_albedo;
  a.l_amp = light_amplitude; a.l_dir = light_direction; a.l_sharp = light_sharpness;
  return 0;
}

int dibr_b200_specular_forward(int64_t num_points, int num_lights, const float* light_amplitude,
                               const float* light_direction, const float* light_sharpness, const float* normal,
                               const float* roughness, const float* view, const float* spec_albedo, float* out,
                               dibr_b200_stream_t stream) {
  Args a;
  const int rc = specular_args(a, num_points, num_lights, light_amplitude, light_direction, light_sharpness, normal,
                               roughness, view, spec_albedo);
  if (rc) return rc;
  if (num_points > 0 && !out) return DIBR_B200_EINVAL;
  a.out = out;
  return launch_fwd<SPECULAR>(a, (cudaStream_t)stream);
}

int dibr_b200_specular_backward(int64_t num_points, int num_lights, const float* light_amplitude,
                                const float* light_direction, const float* light_sharpness, const float* normal,
                                const float* roughness, const float* view, const float* spec_albedo,
                                const float* grad_out, float* grad_normal, float* grad_roughness, float* grad_view,
                                float* grad_spec_albedo, float* grad_light_amplitude, float* grad_light_direction,
                                float* grad_light_sharpness, void* workspace, size_t workspace_bytes,
                                dibr_b200_stream_t stream) {
  Args a;
  const int rc = specular_args(a, num_points, num_lights, light_amplitude, light_direction, light_sharpness, normal,
                               roughness, view, spec_albedo);
  if (rc) return rc;
  if (num_points > 0 && !grad_out) return DIBR_B200_EINVAL;
  a.grad_out = grad_out;
  a.g_normal = grad_normal; a.g_rough = grad_roughness; a.g_view = grad_view; a.g_albedo = grad_spec_albedo;
  a.gl_amp = grad_light_amplitude; a.gl_dir = grad_light_direction; a.gl_sharp = grad_light_sharpness;
  if (num_lights > 0 && (a.gl_amp || a.gl_dir || a.gl_sharp)) {
    if (!workspace) return DIBR_B200_EINVAL;
    a.partial = carve_partials(partials(Cfg<SPECULAR>::kAcc, num_lights), workspace, workspace_bytes);
    if (!a.partial) return DIBR_B200_EWORKSPACE;
  }
  cudaStream_t st = (cudaStream_t)stream;
  if (num_lights == 0) {   // empty sum: zero output, zero per-point gradients
    const size_t b1 = (size_t)num_points * sizeof(float), b3 = 3 * b1;
    if (grad_normal && cudaMemsetAsync(grad_normal, 0, b3, st) != cudaSuccess) return (int)cudaGetLastError();
    if (grad_roughness && cudaMemsetAsync(grad_roughness, 0, b1, st) != cudaSuccess) return (int)cudaGetLastError();
    if (grad_view && cudaMemsetAsync(grad_view, 0, b3, st) != cudaSuccess) return (int)cudaGetLastError();
    if (grad_spec_albedo && cudaMemsetAsync(grad_spec_albedo, 0, b3, st) != cudaSuccess) return (int)cudaGetLastError();
    return 0;
  }
  return launch_bwd<SPECULAR>(a, st);
}

size_t dibr_b200_sg_shade_workspace_bytes(int num_lights) {
  return num_lights < 0 ? 0 : partials(Cfg<SHADE>::kAcc, num_lights).bytes;
}

static int shade_args(ShadeArgs& s, int batch, int height, int width, int num_lights, const float* camera,
                      const int64_t* face_idx, const float* albedo, const float* spec_albedo, const float* roughness,
                      const float* normals, const float* light_amplitude, const float* light_direction,
                      const float* light_sharpness) {
  if (batch < 0 || height < 0 || width < 0 || num_lights < 0) return DIBR_B200_EINVAL;
  if (height > 16384 || width > 16384) return DIBR_B200_ESIZE;
  if (num_lights > 0 && (!light_amplitude || !light_direction || !light_sharpness)) return DIBR_B200_EINVAL;
  const int64_t n = (int64_t)batch * height * width;
  if (n > 0 && (!camera || !face_idx || !albedo || !spec_albedo || !roughness || !normals)) return DIBR_B200_EINVAL;
  s = ShadeArgs{};
  s.a.n = n; s.a.L = num_lights;
  s.a.l_amp = light_amplitude; s.a.l_dir = light_direction; s.a.l_sharp = light_sharpness;
  s.H = height; s.W = width;
  s.face_idx = face_idx; s.cam = camera;
  s.normal = normals; s.albedo = albedo; s.spec_albedo = spec_albedo; s.rough = roughness;
  return 0;
}

int dibr_b200_sg_shade_forward(int batch, int height, int width, int num_lights, const float* camera,
                               const int64_t* face_idx, const float* albedo, const float* spec_albedo,
                               const float* roughness, const float* normals, const float* light_amplitude,
                               const float* light_direction, const float* light_sharpness, float* diffuse,
                               float* specular, float* img, dibr_b200_stream_t stream) {
  ShadeArgs s;
  const int rc = shade_args(s, batch, height, width, num_lights, camera, face_idx, albedo, spec_albedo, roughness,
                            normals, light_amplitude, light_direction, light_sharpness);
  if (rc) return rc;
  if (s.a.n > 0 && (!diffuse || !specular || !img)) return DIBR_B200_EINVAL;
  s.diffuse = diffuse; s.specular = specular; s.img = img;
  return launch_shade_fwd(s, (cudaStream_t)stream);
}

int dibr_b200_sg_shade_backward(int batch, int height, int width, int num_lights, const float* camera,
                                const int64_t* face_idx, const float* albedo, const float* spec_albedo,
                                const float* roughness, const float* normals, const float* light_amplitude,
                                const float* light_direction, const float* light_sharpness,
                                const float* grad_diffuse, const float* grad_specular, const float* grad_img,
                                float* grad_albedo, float* grad_spec_albedo, float* grad_roughness,
                                float* grad_normals, float* grad_light_amplitude, float* grad_light_direction,
                                float* grad_light_sharpness, void* workspace, size_t workspace_bytes,
                                dibr_b200_stream_t stream) {
  ShadeArgs s;
  const int rc = shade_args(s, batch, height, width, num_lights, camera, face_idx, albedo, spec_albedo, roughness,
                            normals, light_amplitude, light_direction, light_sharpness);
  if (rc) return rc;
  s.g_diffuse = grad_diffuse; s.g_specular = grad_specular; s.g_img = grad_img;
  s.g_albedo = grad_albedo; s.g_spec_albedo = grad_spec_albedo; s.g_rough = grad_roughness; s.g_normal = grad_normals;
  s.a.gl_amp = grad_light_amplitude; s.a.gl_dir = grad_light_direction; s.a.gl_sharp = grad_light_sharpness;
  const bool want_light = num_lights > 0 && (s.a.gl_amp || s.a.gl_dir || s.a.gl_sharp);
  if (want_light) {
    if (!workspace) return DIBR_B200_EINVAL;
    s.a.partial = carve_partials(partials(Cfg<SHADE>::kAcc, num_lights), workspace, workspace_bytes);
    if (!s.a.partial) return DIBR_B200_EWORKSPACE;
  }
  if (!want_light && !grad_albedo && !grad_spec_albedo && !grad_roughness && !grad_normals) return 0;
  return launch_shade_bwd(s, (cudaStream_t)stream);
}

}  // extern "C"

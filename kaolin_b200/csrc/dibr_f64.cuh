// dibr_f64.cuh — the float64 instantiation of the DIB-R path (SURVEY.md §8 a11: the reference
// dispatches float and double, rasterization_cuda.cu:218/427, dibr_soft_mask_cuda.cu:205/376).
// Included inside dibr_b200.cu's unnamed namespace: it reuses the binning infrastructure.
//
// Double callers are rare (the reference's tests parametrise the dtype; training runs in fp32), so
// this path is built for exactness, not speed:
//   * f64_prep_kernel turns the double vertices into CONSERVATIVE float bboxes (mins rounded down,
//     maxes rounded up, tight and enlarged) + a validity byte per face; the fp32 binning kernels
//     (bin pyramid, exact integer rectangles of those float boxes) then enumerate a superset of the
//     faces every pixel has to look at;
//   * dibr_f64_fwd_kernel: one thread per pixel walks the bins of its tile and decides every
//     candidate with the reference's own double arithmetic (dibr_math_f64.cuh): the half-open bbox
//     test on the double bbox, the DMUL/DFMA edge functions, eps by copysign, IEEE divisions, strict
//     '>' with ties to the lowest index; the soft mask visits the tile's candidates in index order
//     (the shared-memory sort of the fp32 path) and applies the double enlarged-bbox test, the
//     first knum hits count;
//   * dibr_f64_bwd_kernel: the same walk, gradients scattered with native double atomics.
#include "dibr_math_f64.cuh"

struct F64Args {
  Scene s;
  int D, K, mode;
  float eps, sigmainv, multiplier;                        // C floats, as the reference kernels take them
  double scale;                                           // the multiplier the vertices are scaled by, in double
  double margin;                                          // boxlen * multiplier, in double
  const double* xy; const double* z; const double* feat;  // (NF,3,2) unscaled, (NF,3), (NF,3,D)
  double* out_feat; int64_t* idx; double* out_w; double* out_soft;
  const double* g_feat; const double* g_soft; const double* soft;
  double* g_xy; double* g_ff;
};

__global__ void __launch_bounds__(256) f64_prep_kernel(int64_t NF, const double* __restrict__ xy, const double* __restrict__ z,
                                                       const double* __restrict__ fnz,
                                                       const uint8_t* __restrict__ valid_in, double m, double margin,
                                                       float* __restrict__ xyf, float* __restrict__ bt, float* __restrict__ bl,
                                                       uint8_t* __restrict__ valid) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NF) return;
  double v[6];
  // a NaN depth makes the face's float vertices NaN: the binning then drops it from both sets, as it
  // drops a face with a NaN in face_vertices_image (bin_faces_kernel)
  const bool nan_z = z && (isnan(z[i * 3]) || isnan(z[i * 3 + 1]) || isnan(z[i * 3 + 2]));
#pragma unroll
  for (int k = 0; k < 6; ++k) { v[k] = __dmul_rn(xy[i * 6 + k], m); xyf[i * 6 + k] = nan_z ? NAN : (float)v[k]; }
  const double xmin = fmin(fmin(v[0], v[2]), v[4]), ymin = fmin(fmin(v[1], v[3]), v[5]);
  const double xmax = fmax(fmax(v[0], v[2]), v[4]), ymax = fmax(fmax(v[1], v[3]), v[5]);
  reinterpret_cast<float4*>(bt)[i] = make_float4(__double2float_rd(xmin), __double2float_rd(ymin),
                                                 __double2float_ru(xmax), __double2float_ru(ymax));
  reinterpret_cast<float4*>(bl)[i] = make_float4(__double2float_rd(xmin - margin), __double2float_rd(ymin - margin),
                                                 __double2float_ru(xmax + margin), __double2float_ru(ymax + margin));
  bool ok = true;
  if (fnz) ok = ok && fnz[i] >= 0.0;
  if (valid_in) ok = ok && valid_in[i] != 0;
  valid[i] = ok ? 1 : 0;
}

__device__ __forceinline__ void f64_face(const F64Args& a, int64_t g, double m, double v[6], double bb[4]) {
#pragma unroll
  for (int k = 0; k < 6; ++k) v[k] = __dmul_rn(__ldg(a.xy + g * 6 + k), m);   // face_vertices_image * multiplier (torch, double)
  bb[0] = fmin(fmin(v[0], v[2]), v[4]); bb[1] = fmin(fmin(v[1], v[3]), v[5]);
  bb[2] = fmax(fmax(v[0], v[2]), v[4]); bb[3] = fmax(fmax(v[1], v[3]), v[5]);
}

// Visits, in face-index order, the soft-mask candidates of the calling thread's pixel (CTA-collective:
// every thread of the tile calls it).  hit(face, v[6]) is invoked for faces whose double enlarged bbox
// holds the pixel; it returns false to stop (knum reached).
template <typename Hit>
__device__ __forceinline__ void f64_soft_walk(const F64Args& a, const TileCtx& c, TileSmem& sm, bool uncovered,
                                              double x0, double y0, Hit hit) {
  const Scene& s = a.s;
  const int maxf = s.F;
  bool want = uncovered;
  int lo = -1;
  while (true) {
    int hi;
    const int n = soft_window(s, c, sm, lo, maxf, hi);
    soft_sort(sm, n);
    for (int j = 0; j < n; ++j) {
      const unsigned long long key = sm.sorted[j];
      if (want && (((uint32_t)key) & c.sel) == c.sel) {
        const int f = (int)(key >> 32);
        double v[6], bb[4];
        f64_face(a, c.fbase + f, a.scale, v, bb);
        // dibr.py:33-39 in double: [min - boxlen*m, max + boxlen*m]; dibr_soft_mask_cuda.cu:95
        if (!(x0 < bb[0] - a.margin || x0 >= bb[2] + a.margin || y0 < bb[1] - a.margin || y0 >= bb[3] + a.margin))
          want = hit(f, v);
      }
    }
    const bool all_done = __syncthreads_and(!want);
    if (hi == 0x7fffffff || all_done) break;
    lo = hi;
  }
}

template <bool BWD>
__global__ void __launch_bounds__(kThreads) dibr_f64_kernel(const __grid_constant__ F64Args a) {
  __shared__ __align__(128) TileSmem sm;
  const Scene& s = a.s;
  const TileCtx c = make_tile_ctx(s, blockIdx.z, blockIdx.x, blockIdx.y);   // grid = (tiles_x, tiles_y, views)
  load_bin_table(s, c, sm);
  __syncthreads();
  const double x0 = (double)c.x0, y0 = (double)c.y0;     // computed in float, widened (rasterization_cuda.cu:85-86)
  int best = -1;
  if (!BWD && (a.mode & DIBR_B200_RASTER)) {
    double bz = -INFINITY, b0 = 0.0, b1 = 0.0, b2 = 0.0;
    for (int l = 0; l < s.L; ++l) {
      const BinRef bin = sm.bin[0][l];
      for (int i = 0; i < bin.n; ++i) {
        const int4 e = __ldg(bin.ptr + i);
        const int x_lo = e.y & 0xffff, x_hi = (int)((unsigned)e.y >> 16), y_lo = e.z & 0xffff, y_hi = (int)((unsigned)e.z >> 16);
        if (c.px < x_lo || c.px >= x_hi || c.py < y_lo || c.py >= y_hi) continue;
        double v[6], bb[4];
        f64_face(a, c.fbase + e.x, a.scale, v, bb);
        if (x0 < bb[0] || x0 >= bb[2] || y0 < bb[1] || y0 >= bb[3]) continue;
        double w0, w1, w2;
        if (!dibr64::raster_weights((double)a.eps, x0, y0, v[0], v[1], v[2], v[3], v[4], v[5], w0, w1, w2)) continue;
        const double* zp = a.z + (c.fbase + e.x) * 3;
        const double zv = dibr64::raster_interp(__ldg(zp), __ldg(zp + 1), __ldg(zp + 2), w0, w1, w2);
        if (!(zv <= bz) || (zv == bz && e.x < best)) { bz = zv; best = e.x; b0 = w0; b1 = w1; b2 = w2; }
      }
    }
    if (c.in_img) {
      a.idx[c.pix] = (int64_t)best;
      double* wp = a.out_w + c.pix * 3;
      wp[0] = b0; wp[1] = b1; wp[2] = b2;
      double* fp = a.out_feat + c.pix * a.D;
      const double* ff = a.feat + (c.fbase + max(best, 0)) * 3 * a.D;
      for (int d = 0; d < a.D; ++d)
        fp[d] = best >= 0 ? dibr64::raster_interp(__ldg(ff + d), __ldg(ff + a.D + d), __ldg(ff + 2 * a.D + d), b0, b1, b2) : 0.0;
    }
  } else {
    best = c.in_img ? (int)a.idx[c.pix] : 0;
  }
  const bool uncovered = c.in_img && best < 0;

  if (!BWD) {
    if (!(a.mode & DIBR_B200_SOFT_MASK)) return;
    double allprob = 1.0;
    int kid = 0;
    if (__syncthreads_or(uncovered)) {
      f64_soft_walk(a, c, sm, uncovered, x0, y0, [&](int, const double* v) {
        int edgeid;
        const double d2 = dibr64::soft_min_dist(x0, y0, v, a.multiplier, edgeid);
        allprob = dibr::dmul(allprob, dibr::dsub(1.0, dibr64::soft_prob(d2, a.sigmainv, a.multiplier)));
        return ++kid < a.K;
      });
    }
    if (c.in_img) a.out_soft[c.pix] = uncovered ? dibr::dsub(1.0, allprob) : 1.0;
    return;
  }

  // ---- backward
  if (a.g_feat && c.in_img && best >= 0) {
    const int64_t face = c.fbase + best;
    double p[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) p[k] = __ldg(a.xy + face * 6 + k);        // UNSCALED (rasterization.py:360-368)
    const double* wp = a.out_w + c.pix * 3;
    const double w0 = wp[0], w1 = wp[1], w2 = wp[2];
    dibr64::BwdGeom G;
    dibr64::raster_backward_geom(p, w0, w1, w2, a.eps, G);
    double vsum[6] = {0, 0, 0, 0, 0, 0};
    const double* cf = a.feat + face * 3 * a.D;
    double* gf = a.g_ff + face * 3 * a.D;
    for (int d = 0; d < a.D; ++d) {
      const double g = a.g_feat[c.pix * a.D + d];
      double t6[6];
      dibr64::raster_backward_feature(G, g, __ldg(cf + d), __ldg(cf + a.D + d), __ldg(cf + 2 * a.D + d), t6);
#pragma unroll
      for (int j = 0; j < 6; ++j) vsum[j] += t6[j];
      atomicAdd(gf + d, g * w0); atomicAdd(gf + a.D + d, g * w1); atomicAdd(gf + 2 * a.D + d, g * w2);
    }
#pragma unroll
    for (int j = 0; j < 6; ++j) atomicAdd(a.g_xy + face * 6 + j, vsum[j]);
  }
  if (a.g_soft && __syncthreads_or(uncovered)) {
    const double dLdp = uncovered ? a.g_soft[c.pix] : 0.0;
    const double allprob = uncovered ? a.soft[c.pix] : 0.0;
    int kid = 0;
    f64_soft_walk(a, c, sm, uncovered, x0, y0, [&](int f, const double* v) {
      int edgeid;
      const double d2 = dibr64::soft_min_dist(x0, y0, v, a.multiplier, edgeid);
      const double prob = dibr64::soft_prob(d2, a.sigmainv, a.multiplier);
      double g[6];
      dibr64::soft_backward_terms(x0, y0, v, edgeid, prob, allprob, dLdp, a.sigmainv, a.multiplier, g);
      double* gp = a.g_xy + (c.fbase + f) * 6;
#pragma unroll
      for (int j = 0; j < 6; ++j)
        if (g[j] != 0.0) atomicAdd(gp + j, g[j]);
      return ++kid < a.K;
    });
  }
}

// Lays out the float scene of a double call (scaled vertices, conservative bboxes, validity) in the
// workspace, after setup_scene's pieces; a null workspace is too small.  Host only: nothing is
// enqueued.  `multiplier` is the C float the reference's kernels take: it places the pixel centres.
int f64_scene(Scene& s, int B, int F, int H, int W, float multiplier, void* ws, size_t ws_bytes) {
  if (!ws) return DIBR_B200_EWORKSPACE;
  return setup_scene(s, B, (int64_t)B * F, F, H, W, multiplier, 0.f, 0, true, ws, ws_bytes);
}

// Fills the float scene laid out by f64_scene from the double inputs, scaled by the double
// multiplier `scale` (face_vertices_image * multiplier in torch, rasterization.py:320, dibr.py:32),
// and bins it.  `fvz` (nullable) only marks faces with a NaN depth, which are binned in no set.
int f64_bins(const Scene& s, const double* fvi, const double* fvz, const double* fnz, const uint8_t* valid,
             double scale, double margin, int sets, cudaStream_t st) {
  if (s.NF > 0)
    f64_prep_kernel<<<(unsigned)((s.NF + 255) / 256), 256, 0, st>>>(
        s.NF, fvi, fvz, fnz, valid, scale, margin, const_cast<float*>(s.xy), const_cast<float*>(s.bbox_tight),
        const_cast<float*>(s.bbox_large), const_cast<uint8_t*>(s.valid));
  return build_bins(s, sets, st);     // with no faces: zeroed counters, every pixel takes the empty path
}

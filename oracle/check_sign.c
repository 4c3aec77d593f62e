/* TEST INFRASTRUCTURE — NOT PRODUCT CODE.
 *
 * Brute-force CPU restatement of the reference's point-in-mesh test (kaolin.ops.mesh.check_sign, CUDA
 * path), in float and double:
 *   oracle_mesh_intersection_count_*   kernel mesh_intersection_cuda.cu:105-219: every point against
 *                                      every face, the count of crossed faces
 *   oracle_check_sign_*                wrapper check_sign.py:45-57,138-155: per view maxlen over all
 *                                      vertices (NaN propagating), verts and points / maxlen, the corners
 *                                      gathered, count % 2 == 1
 * Every floating-point step is written as the reference's <float> / <double> kernels compile it for
 * sm_90a (nvcc 12.9 -O3, read from their SASS), with the FMAs spelled out: build with
 * -ffp-contract=off (oracle/check_sign.py) so the compiler adds none.
 */
#include <math.h>
#include <stdint.h>

#define DEFINE_CHECK_SIGN(T, SFX, FMA, MIN, MAX)                                                             \
  /* mesh_intersection_cuda.cu:69-83 on (y, z) pairs */                                                     \
  static T signed_area_##SFX(T ax, T ay, T bx, T by, T cx, T cy) {                                          \
    if (cx > bx || (bx == cx && cy < by)) return -FMA(by - cy, ax - cx, (cx - bx) * (ay - cy));              \
    return FMA(cy - by, ax - bx, (bx - cx) * (ay - by));                                                     \
  }                                                                                                          \
  /* :85-93 */                                                                                               \
  static int above_##SFX(T vx, T vy, T lx, T ly, T rx, T ry) {                                               \
    return FMA(rx - lx, vy - ly, -((ry - ly) * (vx - lx))) > 0;                                              \
  }                                                                                                          \
  /* :131-214 for one (point, face) */                                                                       \
  static int crosses_##SFX(const T* q, const T* p1, const T* p2, const T* p3) {                             \
    const T qx = q[0], qy = q[1], qz = q[2], q2x = qx + (T)10;                                               \
    /* :48-56 bbox_check: float bounds */                                                                    \
    const float ymin = (float)MIN(p1[1], MIN(p2[1], p3[1])), ymax = (float)MAX(p1[1], MAX(p2[1], p3[1]));   \
    const float zmin = (float)MIN(p1[2], MIN(p2[2], p3[2])), zmax = (float)MAX(p1[2], MAX(p2[2], p3[2]));   \
    if (qy < (T)ymin || (T)ymax < qy || qz < (T)zmin || (T)zmax < qz) return 0;                              \
    /* :59-64 signed_volume = dot(cross(b - a, c - a), d - a) */                                             \
    const T ex = p1[0] - qx, ey = p1[1] - qy, ez = p1[2] - qz;                                               \
    const T fx = p2[0] - qx, fy = p2[1] - qy, fz = p2[2] - qz;                                               \
    const T gx = p3[0] - qx, gy = p3[1] - qy, gz = p3[2] - qz;                                               \
    const T ex2 = p1[0] - q2x, fx2 = p2[0] - q2x, gx2 = p3[0] - q2x;                                         \
    const T cx = FMA(ey, fz, -(ez * fy)), cy = FMA(ez, fx, -(ex * fz)), cz = FMA(ex, fy, -(ey * fx));        \
    const T cy2 = FMA(ez, fx2, -(ex2 * fz)), cz2 = FMA(ex2, fy, -(ey * fx2));                                \
    const T vol1 = FMA(cz, gz, FMA(cx, gx, cy * gy)), vol2 = FMA(cz2, gz, FMA(cx, gx2, cy2 * gy));           \
    if ((vol1 > 0) == (vol2 > 0)) return 0;                                                                  \
    const T d1 = signed_area_##SFX(qy, qz, p1[1], p1[2], p2[1], p2[2]);                                      \
    const T d2 = signed_area_##SFX(qy, qz, p2[1], p2[2], p3[1], p3[2]);                                      \
    if (!(d1 * d2 >= 0)) return 0;                                                                           \
    const T d3 = signed_area_##SFX(qy, qz, p3[1], p3[2], p1[1], p1[2]);                                      \
    if (!(d3 * d1 >= 0 && d2 * d3 >= 0)) return 0;                                                          \
    int edge;                                                                                                \
    const T *v1, *v2, *other = 0;                                                                            \
    if (qy == p1[1] && qz == p1[2]) { edge = 0; v1 = p2; v2 = p3; }                                          \
    else if (qy == p2[1] && qz == p2[2]) { edge = 0; v1 = p1; v2 = p3; }                                     \
    else if (qy == p3[1] && qz == p3[2]) { edge = 0; v1 = p1; v2 = p2; }                                     \
    else if (d1 == 0) { edge = 1; v1 = p1; v2 = p2; other = p3; }                                           \
    else if (d2 == 0) { edge = 1; v1 = p2; v2 = p3; other = p1; }                                           \
    else if (d3 == 0) { edge = 1; v1 = p3; v2 = p1; other = p2; }                                           \
    else return 1;                                                                                           \
    if (v1[1] > v2[1] || (v1[1] == v2[1] && v1[2] > v2[2])) { const T* t = v1; v1 = v2; v2 = t; }           \
    if (edge) return !above_##SFX(other[1], other[2], v1[1], v1[2], v2[1], v2[2]);                           \
    return above_##SFX(qy, qz, v1[1], v1[2], v2[1], v2[2]) && v1[1] < qy && v2[1] >= qy;                     \
  }                                                                                                          \
  void oracle_mesh_intersection_count_##SFX(int n, const T* points, int m, const T* v1, const T* v2,        \
                                            const T* v3, T* out) {                                          \
    _Pragma("omp parallel for schedule(dynamic, 64)")                                                        \
    for (int j = 0; j < n; ++j) {                                                                            \
      int64_t c = 0;                                                                                         \
      for (int k = 0; k < m; ++k) c += crosses_##SFX(points + 3 * (int64_t)j, v1 + 3 * (int64_t)k,           \
                                                     v2 + 3 * (int64_t)k, v3 + 3 * (int64_t)k);              \
      out[j] = (T)c;                                                                                         \
    }                                                                                                        \
  }                                                                                                          \
  static T nan_max_##SFX(T a, T b) { return (a > b || a != a) ? a : b; }                                     \
  static T nan_min_##SFX(T a, T b) { return (a < b || a != a) ? a : b; }                                     \
  /* verts (B, V, 3), faces (F, 3), points (B, N, 3); scratch: 9F + 4N values; out (B, N) */                \
  int oracle_check_sign_##SFX(int B, int V, int F, int N, const T* verts, const int64_t* faces,             \
                              const T* points, T* scratch, uint8_t* out) {                                  \
    T* corners = scratch;                                                                                    \
    T* q = scratch + 9 * (int64_t)F;                                                                         \
    T* counts = q + 3 * (int64_t)N;                                                                          \
    for (int64_t f = 0; f < 3 * (int64_t)F; ++f)                                                             \
      if (faces[f] < 0 || faces[f] >= V) return -1;                                                          \
    for (int b = 0; b < B; ++b) {                                                                            \
      const T* v = verts + (int64_t)b * V * 3;                                                               \
      T len[3];                                                                                              \
      for (int a = 0; a < 3; ++a) {                                                                          \
        T mn = v[a], mx = v[a];                                                                              \
        for (int i = 1; i < V; ++i) { mn = nan_min_##SFX(mn, v[3 * (int64_t)i + a]);                         \
                                      mx = nan_max_##SFX(mx, v[3 * (int64_t)i + a]); }                       \
        len[a] = mx - mn;                                                                                    \
      }                                                                                                      \
      const T maxlen = nan_max_##SFX(nan_max_##SFX(len[0], len[1]), len[2]);                                \
      for (int64_t f = 0; f < F; ++f)                                                                        \
        for (int k = 0; k < 3; ++k)                                                                          \
          for (int a = 0; a < 3; ++a) corners[(k * (int64_t)F + f) * 3 + a] = v[faces[3 * f + k] * 3 + a] / maxlen; \
      for (int64_t i = 0; i < 3 * (int64_t)N; ++i) q[i] = points[(int64_t)b * N * 3 + i] / maxlen;           \
      oracle_mesh_intersection_count_##SFX(N, q, F, corners, corners + 3 * (int64_t)F,                       \
                                           corners + 6 * (int64_t)F, counts);                                \
      for (int64_t i = 0; i < N; ++i) out[(int64_t)b * N + i] = fmod(counts[i], 2) == 1;                    \
    }                                                                                                        \
    return 0;                                                                                                \
  }

DEFINE_CHECK_SIGN(float, f32, fmaf, fminf, fmaxf)
DEFINE_CHECK_SIGN(double, f64, fma, fmin, fmax)

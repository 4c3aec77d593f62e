// TEST-ONLY: compiles kaolin_b200/csrc/dibr_math.cuh as plain C++ (g++,
// -ffp-contract=off) and evaluates, for every (pixel, face) pair of a scene,
// both raster_weights (the forward's test) and raster_weights_of (the weights
// the rasterize backward recomputes for the face it is given), so that
// tests/test_known_face_weights.py can compare them bit for bit.
#include <cstdint>
#include "../../kaolin_b200/csrc/dibr_math.cuh"

using namespace dibr;

extern "C" {

// xy: (F,3,2) already multiplied.  inside: (H,W,F); w_fwd, w_of: (H,W,F,3).
void hm_known_face_weights(int H, int W, int F, const float* xy, float multiplier, float eps,
                           uint8_t* inside, float* w_fwd, float* w_of) {
  const PixelGrid g = make_grid(multiplier, W, H);
  const RasterConst rc = make_raster_const(eps);
  for (int iy = 0; iy < H; iy++) for (int ix = 0; ix < W; ix++) {
    const float x0 = pix_x(g, ix), y0 = pix_y(g, iy);
    for (int f = 0; f < F; f++) {
      const float* p = xy + 6 * (int64_t)f;
      const int64_t o = ((int64_t)iy * W + ix) * F + f;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      inside[o] = raster_weights(rc, x0, y0, p[0], p[1], p[2], p[3], p[4], p[5], a0, a1, a2) ? 1 : 0;
      w_fwd[3 * o] = a0; w_fwd[3 * o + 1] = a1; w_fwd[3 * o + 2] = a2;
      raster_weights_of(rc, x0, y0, p[0], p[1], p[2], p[3], p[4], p[5], w_of[3 * o], w_of[3 * o + 1],
                        w_of[3 * o + 2]);
    }
  }
}

}  // extern "C"

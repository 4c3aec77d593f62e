// TEST INFRASTRUCTURE — not product code.
// pybind11 shim that exposes the reference's point-to-mesh distance operators, compiled unmodified from
// their sources (oracle/build_ref_point_mesh.py), under the module name `kaolin_ref_point_mesh_C`.
// Mirrors the registration the reference does in kaolin/csrc/bindings.cpp:106-109.
#include <torch/extension.h>
#include "metrics/unbatched_triangle_distance.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("unbatched_triangle_distance_forward_cuda", &kaolin::unbatched_triangle_distance_forward_cuda);
  m.def("unbatched_triangle_distance_backward_cuda", &kaolin::unbatched_triangle_distance_backward_cuda);
}

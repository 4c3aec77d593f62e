// TEST INFRASTRUCTURE — not product code.
// pybind11 shim that exposes the reference's point-in-mesh operator, compiled unmodified from its
// sources (oracle/build_ref_check_sign.py), under the module name `kaolin_ref_check_sign_C`.
// Mirrors the registration the reference does in kaolin/csrc/bindings.cpp:48-49.
#include <torch/extension.h>
#include "ops/mesh/mesh_intersection.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("unbatched_mesh_intersection_cuda", &kaolin::unbatched_mesh_intersection_cuda);
}

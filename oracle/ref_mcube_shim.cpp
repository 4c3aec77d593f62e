// TEST INFRASTRUCTURE — not product code.
// pybind11 shim that exposes the reference's marching-cubes operator, compiled unmodified from its
// sources (oracle/build_ref_mcube.py), under the module name `kaolin_ref_mcube_C`.
// Mirrors the registration the reference does in kaolin/csrc/bindings.cpp:54-55.
#include <torch/extension.h>
#include "ops/conversions/unbatched_mcube/unbatched_mcube.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("unbatched_mcube_forward_cuda", &kaolin::unbatched_mcube_forward_cuda);
}

// TEST INFRASTRUCTURE — not product code.
// pybind11 shim that exposes the reference's spherical-Gaussian operator pair, compiled unmodified
// from its sources (oracle/build_ref_sg.py), under the module name `kaolin_ref_sg_C`.
// Mirrors the registration the reference does in kaolin/csrc/bindings.cpp:129-133.
#include <torch/extension.h>
#include "render/sg/unbatched_reduced_sg_inner_product.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("unbatched_reduced_sg_inner_product_forward_cuda", &kaolin::unbatched_reduced_sg_inner_product_forward_cuda);
  m.def("unbatched_reduced_sg_inner_product_backward_cuda", &kaolin::unbatched_reduced_sg_inner_product_backward_cuda);
}

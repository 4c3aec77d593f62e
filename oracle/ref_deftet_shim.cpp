// TEST INFRASTRUCTURE — not product code.
// pybind11 shim that exposes the reference's DefTet sparse-render operator pair, compiled unmodified
// from its sources (oracle/build_ref_deftet.py), under the module name `kaolin_ref_deftet_C`.
// Mirrors the registration the reference does in kaolin/csrc/bindings.cpp:116-117.
#include <torch/extension.h>
#include "render/mesh/deftet.h"

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.def("deftet_sparse_render_forward_cuda", &kaolin::deftet_sparse_render_forward_cuda);
  m.def("deftet_sparse_render_backward_cuda", &kaolin::deftet_sparse_render_backward_cuda);
}

// Python module `blackbird_b200._bb`: one extension holding the C++20 control plane and the
// sm_90a data plane.  Sub-binders live in bind_*.cpp.
#include <pybind11/pybind11.h>

namespace py = pybind11;

void bind_common(py::module_& m);
void bind_gpu(py::module_& m);
void bind_control(py::module_& m);

PYBIND11_MODULE(_bb, m) {
  m.doc() = "blackbird_b200 native core (C++20 control plane + sm_90a data plane)";
  bind_common(m);
  bind_control(m);
  bind_gpu(m);
}

// pybind11 surface of the lingvo_b200 native extension (`lingvo_b200.ops._C`).
#include <torch/extension.h>

namespace lb {
torch::Tensor gemm_bf16(const torch::Tensor& a, const torch::Tensor& b, bool a_kmajor,
                        bool b_kmajor, const c10::optional<torch::Tensor>& bias, int64_t act,
                        const c10::optional<torch::Tensor>& aux, int64_t aux_mode,
                        const c10::optional<torch::Tensor>& row_scale,
                        const c10::optional<torch::Tensor>& out,
                        const c10::optional<torch::Tensor>& row_ptrs);
void RegisterAll(pybind11::module& m);
}  // namespace lb

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "lingvo_b200 sm_90a kernels";
  m.def("gemm_bf16", &lb::gemm_bf16, py::arg("a"), py::arg("b"), py::arg("a_kmajor") = true,
        py::arg("b_kmajor") = true, py::arg("bias") = py::none(), py::arg("act") = 0,
        py::arg("aux") = py::none(), py::arg("aux_mode") = 0, py::arg("row_scale") = py::none(),
        py::arg("out") = py::none(), py::arg("row_ptrs") = py::none());
  lb::RegisterAll(m);
}

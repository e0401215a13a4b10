// egpu_tables_op.cc — the PyTorch operator egpu::bestfit_tables (DESIGN.md §2.10): argument checks on the
// host, outputs from the caching allocator, one launch of bestfit_tables_kernel on the current stream.  No
// synchronisation and no host copy, so the operator can be captured into a CUDA graph.  The fake (shape)
// implementation is registered from Python (tables.py).
#include <ATen/core/Tensor.h>
#include <ATen/ops/empty.h>
#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>
#include <torch/library.h>

#include <cstdint>
#include <limits>
#include <tuple>

#include "egpu_tables.h"

namespace {

void check_int32_contiguous(const at::Tensor& t, const char* name) {
    TORCH_CHECK(t.scalar_type() == at::kInt, "bestfit_tables: ", name, " must be int32, got ", t.scalar_type());
    TORCH_CHECK(t.is_contiguous(), "bestfit_tables: ", name, " must be contiguous");
}

// Checks in the order of the Python fake implementation, device last, so that every refusal but the
// device's can be met with CPU tensors.
std::tuple<at::Tensor, at::Tensor> bestfit_tables(const at::Tensor& free_core, const at::Tensor& free_mem,
                                                  const at::Tensor& d_valid, const at::Tensor& req_core,
                                                  const at::Tensor& req_mem) {
    check_int32_contiguous(free_core, "free_core");
    check_int32_contiguous(free_mem, "free_mem");
    check_int32_contiguous(d_valid, "d_valid");
    check_int32_contiguous(req_core, "req_core");
    check_int32_contiguous(req_mem, "req_mem");
    TORCH_CHECK_VALUE(free_core.dim() == 2 && free_mem.sizes() == free_core.sizes(),
                      "bestfit_tables: free_core and free_mem must both be [N, D], got ", free_core.sizes(), " and ",
                      free_mem.sizes());
    const int64_t N = free_core.size(0), D = free_core.size(1);
    TORCH_CHECK_VALUE(D >= 1 && D <= 64, "bestfit_tables: D must be in [1, 64], got ", D);
    TORCH_CHECK_VALUE(d_valid.dim() == 1 && d_valid.size(0) == N, "bestfit_tables: d_valid must be [N] = [", N,
                      "], got ", d_valid.sizes());
    TORCH_CHECK_VALUE(req_core.dim() == 1 && req_mem.sizes() == req_core.sizes(),
                      "bestfit_tables: req_core and req_mem must both be [P], got ", req_core.sizes(), " and ",
                      req_mem.sizes());
    const int64_t P = req_core.size(0);
    constexpr int64_t kMax = std::numeric_limits<int32_t>::max();
    TORCH_CHECK_VALUE(N <= kMax && P <= kMax, "bestfit_tables: N and P must be below 2^31, got ", N, " and ", P);
    const at::Device dev = free_core.device();
    for (const at::Tensor* t : {&free_core, &free_mem, &d_valid, &req_core, &req_mem})
        TORCH_CHECK(t->is_cuda() && t->device() == dev, "bestfit_tables: every tensor must be on one CUDA device, got ",
                    t->device(), " and ", dev);

    at::Tensor idx = at::empty({N, P}, free_core.options().dtype(at::kChar));
    at::Tensor key = at::empty({N, P}, free_core.options());
    if (N == 0 || P == 0) return {idx, key};
    const c10::cuda::CUDAGuard guard(dev);
    const cudaError_t err = egpu::tables_launch(
        free_core.data_ptr<int32_t>(), free_mem.data_ptr<int32_t>(), d_valid.data_ptr<int32_t>(), static_cast<int>(N),
        static_cast<int>(D), req_core.data_ptr<int32_t>(), req_mem.data_ptr<int32_t>(), static_cast<int>(P),
        idx.data_ptr<int8_t>(), key.data_ptr<int32_t>(), dev.index(), c10::cuda::getCurrentCUDAStream(dev.index()).stream());
    TORCH_CHECK(err == cudaSuccess, "bestfit_tables: launch failed: ", cudaGetErrorString(err));
    return {idx, key};
}

}  // namespace

TORCH_LIBRARY(egpu, m) {
    m.def("bestfit_tables(Tensor free_core, Tensor free_mem, Tensor d_valid, Tensor req_core, Tensor req_mem) -> "
          "(Tensor, Tensor)");
}

// The CPU registration only refuses (the device check above): a CPU caller gets the same messages as a CUDA one.
TORCH_LIBRARY_IMPL(egpu, CUDA, m) { m.impl("bestfit_tables", &bestfit_tables); }
TORCH_LIBRARY_IMPL(egpu, CPU, m) { m.impl("bestfit_tables", &bestfit_tables); }

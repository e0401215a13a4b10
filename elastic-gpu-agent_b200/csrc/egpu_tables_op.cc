// egpu_tables_op.cc — the PyTorch operators egpu::bestfit_tables (DESIGN.md §2.10), egpu::place_tables (§2.11),
// egpu::place_pods (§2.12), egpu::place_gangs (§2.13), egpu::preempt_pods (§2.14) and egpu::preempt_gangs (§2.15):
// argument checks on the host, outputs and scratch from the caching allocator, one launch of bestfit_tables_kernel,
// place_tables_kernel, place_pods_kernel, place_gangs_kernel, preempt_pods_kernel or preempt_gangs_kernel on the
// current stream.  No synchronisation and no host copy, so every operator can be captured
// into a CUDA graph.  The fake (shape) implementations are registered from Python (tables.py).
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

void check_int32_contiguous(const char* op, const at::Tensor& t, const char* name) {
    TORCH_CHECK(t.scalar_type() == at::kInt, op, ": ", name, " must be int32, got ", t.scalar_type());
    TORCH_CHECK(t.is_contiguous(), op, ": ", name, " must be contiguous");
}

// The checks of both operators, in the order of the Python fake implementations, device last, so that every
// refusal but the device's can be met with CPU tensors.  Returns (N, D, P).
std::tuple<int64_t, int64_t, int64_t> check_inputs(const char* op, const at::Tensor& free_core, const at::Tensor& free_mem,
                                                   const at::Tensor& d_valid, const at::Tensor& req_core,
                                                   const at::Tensor& req_mem) {
    check_int32_contiguous(op, free_core, "free_core");
    check_int32_contiguous(op, free_mem, "free_mem");
    check_int32_contiguous(op, d_valid, "d_valid");
    check_int32_contiguous(op, req_core, "req_core");
    check_int32_contiguous(op, req_mem, "req_mem");
    TORCH_CHECK_VALUE(free_core.dim() == 2 && free_mem.sizes() == free_core.sizes(), op,
                      ": free_core and free_mem must both be [N, D], got ", free_core.sizes(), " and ", free_mem.sizes());
    const int64_t N = free_core.size(0), D = free_core.size(1);
    TORCH_CHECK_VALUE(D >= 1 && D <= 64, op, ": D must be in [1, 64], got ", D);
    TORCH_CHECK_VALUE(d_valid.dim() == 1 && d_valid.size(0) == N, op, ": d_valid must be [N] = [", N, "], got ",
                      d_valid.sizes());
    TORCH_CHECK_VALUE(req_core.dim() == 1 && req_mem.sizes() == req_core.sizes(), op,
                      ": req_core and req_mem must both be [P], got ", req_core.sizes(), " and ", req_mem.sizes());
    const int64_t P = req_core.size(0);
    constexpr int64_t kMax = std::numeric_limits<int32_t>::max();
    TORCH_CHECK_VALUE(N <= kMax && P <= kMax, op, ": N and P must be below 2^31, got ", N, " and ", P);
    const at::Device dev = free_core.device();
    for (const at::Tensor* t : {&free_core, &free_mem, &d_valid, &req_core, &req_mem})
        TORCH_CHECK(t->is_cuda() && t->device() == dev, op, ": every tensor must be on one CUDA device, got ", t->device(),
                    " and ", dev);
    return {N, D, P};
}

std::tuple<at::Tensor, at::Tensor> bestfit_tables(const at::Tensor& free_core, const at::Tensor& free_mem,
                                                  const at::Tensor& d_valid, const at::Tensor& req_core,
                                                  const at::Tensor& req_mem) {
    const auto [N, D, P] = check_inputs("bestfit_tables", free_core, free_mem, d_valid, req_core, req_mem);
    const at::Device dev = free_core.device();
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

// DESIGN.md §2.11.  Scratch comes from the caching allocator on the current stream, so the call stays capturable.
std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> place_tables(
    const at::Tensor& free_core, const at::Tensor& free_mem, const at::Tensor& d_valid, const at::Tensor& req_core,
    const at::Tensor& req_mem) {
    const auto [N, D, P] = check_inputs("place_tables", free_core, free_mem, d_valid, req_core, req_mem);
    const at::Device dev = free_core.device();
    const c10::cuda::CUDAGuard guard(dev);
    at::Tensor node = at::empty({P}, free_core.options());
    at::Tensor dv_out = at::empty({P}, free_core.options().dtype(at::kChar));
    at::Tensor fc_out = at::empty({N, D}, free_core.options());
    at::Tensor fm_out = at::empty({N, D}, free_core.options());
    at::Tensor info = at::empty({2}, free_core.options());
    if (N == 0 || P == 0) {  // nothing to place, or nowhere to place it
        node.fill_(-1);
        dv_out.fill_(-1);
        fc_out.copy_(free_core);
        fm_out.copy_(free_mem);
        info.zero_();
        return {node, dv_out, fc_out, fm_out, info};
    }
    at::Tensor scratch = at::empty({static_cast<int64_t>(egpu::place_scratch_bytes(static_cast<int>(P)))},
                                   free_core.options().dtype(at::kByte));
    const cudaError_t err = egpu::place_launch(
        free_core.data_ptr<int32_t>(), free_mem.data_ptr<int32_t>(), d_valid.data_ptr<int32_t>(), static_cast<int>(N),
        static_cast<int>(D), req_core.data_ptr<int32_t>(), req_mem.data_ptr<int32_t>(), static_cast<int>(P),
        node.data_ptr<int32_t>(), dv_out.data_ptr<int8_t>(), fc_out.data_ptr<int32_t>(), fm_out.data_ptr<int32_t>(),
        info.data_ptr<int32_t>(), scratch.data_ptr(), dev.index(), c10::cuda::getCurrentCUDAStream(dev.index()).stream());
    TORCH_CHECK(err == cudaSuccess, "place_tables: launch failed: ", cudaGetErrorString(err));
    return {node, dv_out, fc_out, fm_out, info};
}

// DESIGN.md §2.12.  The checks of check_inputs, then pod_offsets' dtype, layout, shape and device; its values are
// the kernel's to check (they are device data).  Returns G.
int64_t check_pod_offsets(const char* op, const at::Tensor& free_core, const at::Tensor& pod_offsets) {
    check_int32_contiguous(op, pod_offsets, "pod_offsets");
    TORCH_CHECK_VALUE(pod_offsets.dim() == 1 && pod_offsets.size(0) >= 1, op, ": pod_offsets must be [G + 1], got ",
                      pod_offsets.sizes());
    TORCH_CHECK_VALUE(pod_offsets.size(0) <= std::numeric_limits<int32_t>::max(), op,
                      ": G + 1 must be below 2^31, got ", pod_offsets.size(0));
    TORCH_CHECK(pod_offsets.is_cuda() && pod_offsets.device() == free_core.device(), op,
                ": every tensor must be on one CUDA device, got ", pod_offsets.device(), " and ", free_core.device());
    return pod_offsets.size(0) - 1;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> place_pods(
    const at::Tensor& free_core, const at::Tensor& free_mem, const at::Tensor& d_valid, const at::Tensor& req_core,
    const at::Tensor& req_mem, const at::Tensor& pod_offsets) {
    const auto [N, D, P] = check_inputs("place_pods", free_core, free_mem, d_valid, req_core, req_mem);
    const int64_t G = check_pod_offsets("place_pods", free_core, pod_offsets);
    const at::Device dev = free_core.device();
    const c10::cuda::CUDAGuard guard(dev);
    at::Tensor node = at::empty({G}, free_core.options());
    at::Tensor dv_out = at::empty({P}, free_core.options().dtype(at::kChar));
    at::Tensor fc_out = at::empty({N, D}, free_core.options());
    at::Tensor fm_out = at::empty({N, D}, free_core.options());
    at::Tensor info = at::empty({3}, free_core.options());
    if (N == 0 || P == 0) {  // nothing to place, or nowhere to place it
        node.fill_(-1);
        dv_out.fill_(-1);
        fc_out.copy_(free_core);
        fm_out.copy_(free_mem);
        info.zero_();
        return {node, dv_out, fc_out, fm_out, info};
    }
    at::Tensor scratch = at::empty({static_cast<int64_t>(egpu::pods_scratch_bytes(static_cast<int>(G)))},
                                   free_core.options().dtype(at::kByte));
    const cudaError_t err = egpu::pods_launch(
        free_core.data_ptr<int32_t>(), free_mem.data_ptr<int32_t>(), d_valid.data_ptr<int32_t>(), static_cast<int>(N),
        static_cast<int>(D), req_core.data_ptr<int32_t>(), req_mem.data_ptr<int32_t>(), static_cast<int>(P),
        pod_offsets.data_ptr<int32_t>(), static_cast<int>(G), node.data_ptr<int32_t>(), dv_out.data_ptr<int8_t>(),
        fc_out.data_ptr<int32_t>(), fm_out.data_ptr<int32_t>(), info.data_ptr<int32_t>(), scratch.data_ptr(), dev.index(),
        c10::cuda::getCurrentCUDAStream(dev.index()).stream());
    TORCH_CHECK(err == cudaSuccess, "place_pods: launch failed: ", cudaGetErrorString(err));
    return {node, dv_out, fc_out, fm_out, info};
}

// DESIGN.md §2.13.  place_pods' checks naming place_gangs, then gang_offsets' and gang_min's dtype and layout, shapes
// and device; their values are the kernel's to check (they are device data).  Returns J.
int64_t check_gangs(const char* op, const at::Tensor& free_core, const at::Tensor& gang_offsets,
                    const at::Tensor& gang_min) {
    check_int32_contiguous(op, gang_offsets, "gang_offsets");
    check_int32_contiguous(op, gang_min, "gang_min");
    TORCH_CHECK_VALUE(gang_offsets.dim() == 1 && gang_offsets.size(0) >= 1, op,
                      ": gang_offsets must be [J + 1], got ", gang_offsets.sizes());
    TORCH_CHECK_VALUE(gang_offsets.size(0) <= std::numeric_limits<int32_t>::max(), op,
                      ": J + 1 must be below 2^31, got ", gang_offsets.size(0));
    const int64_t J = gang_offsets.size(0) - 1;
    TORCH_CHECK_VALUE(gang_min.dim() == 1 && gang_min.size(0) == J, op, ": gang_min must be [J] = [", J,
                      "], got ", gang_min.sizes());
    for (const at::Tensor* t : {&gang_offsets, &gang_min})
        TORCH_CHECK(t->is_cuda() && t->device() == free_core.device(), op,
                    ": every tensor must be on one CUDA device, got ", t->device(), " and ", free_core.device());
    return J;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> place_gangs(
    const at::Tensor& free_core, const at::Tensor& free_mem, const at::Tensor& d_valid, const at::Tensor& req_core,
    const at::Tensor& req_mem, const at::Tensor& pod_offsets, const at::Tensor& gang_offsets,
    const at::Tensor& gang_min) {
    const auto [N, D, P] = check_inputs("place_gangs", free_core, free_mem, d_valid, req_core, req_mem);
    const int64_t G = check_pod_offsets("place_gangs", free_core, pod_offsets);
    const int64_t J = check_gangs("place_gangs", free_core, gang_offsets, gang_min);
    const at::Device dev = free_core.device();
    const c10::cuda::CUDAGuard guard(dev);
    at::Tensor node = at::empty({G}, free_core.options());
    at::Tensor dv_out = at::empty({P}, free_core.options().dtype(at::kChar));
    at::Tensor placed = at::empty({J}, free_core.options());
    at::Tensor fc_out = at::empty({N, D}, free_core.options());
    at::Tensor fm_out = at::empty({N, D}, free_core.options());
    at::Tensor info = at::empty({3}, free_core.options());
    if (N == 0 || P == 0) {  // nothing to place, or nowhere to place it
        node.fill_(-1);
        dv_out.fill_(-1);
        placed.zero_();
        fc_out.copy_(free_core);
        fm_out.copy_(free_mem);
        info.zero_();
        return {node, dv_out, placed, fc_out, fm_out, info};
    }
    at::Tensor scratch =
        at::empty({static_cast<int64_t>(egpu::gangs_scratch_bytes(static_cast<int>(G), static_cast<int>(J)))},
                  free_core.options().dtype(at::kByte));
    const cudaError_t err = egpu::gangs_launch(
        free_core.data_ptr<int32_t>(), free_mem.data_ptr<int32_t>(), d_valid.data_ptr<int32_t>(), static_cast<int>(N),
        static_cast<int>(D), req_core.data_ptr<int32_t>(), req_mem.data_ptr<int32_t>(), static_cast<int>(P),
        pod_offsets.data_ptr<int32_t>(), static_cast<int>(G), gang_offsets.data_ptr<int32_t>(),
        gang_min.data_ptr<int32_t>(), static_cast<int>(J), node.data_ptr<int32_t>(), dv_out.data_ptr<int8_t>(),
        placed.data_ptr<int32_t>(), fc_out.data_ptr<int32_t>(), fm_out.data_ptr<int32_t>(), info.data_ptr<int32_t>(),
        scratch.data_ptr(), dev.index(), c10::cuda::getCurrentCUDAStream(dev.index()).stream());
    TORCH_CHECK(err == cudaSuccess, "place_gangs: launch failed: ", cudaGetErrorString(err));
    return {node, dv_out, placed, fc_out, fm_out, info};
}

// DESIGN.md §2.14.  place_pods' checks naming preempt_pods, then the dtype and layout of the six new tensors, their
// shapes, and their device; their values are the kernel's to check (they are device data).  preempt_gangs (§2.15)
// has no pod_prio (its priority is per gang) and passes nullptr.  Returns (Q, H).
std::tuple<int64_t, int64_t> check_running(const char* op, const at::Tensor& free_core, int64_t G,
                                           const at::Tensor* pod_prio, const at::Tensor& run_core,
                                           const at::Tensor& run_mem, const at::Tensor& run_dev,
                                           const at::Tensor& run_offsets, const at::Tensor& run_prio,
                                           const at::Tensor& node_offsets) {
    if (pod_prio) check_int32_contiguous(op, *pod_prio, "pod_prio");
    check_int32_contiguous(op, run_core, "run_core");
    check_int32_contiguous(op, run_mem, "run_mem");
    TORCH_CHECK(run_dev.scalar_type() == at::kChar, op, ": run_dev must be int8, got ", run_dev.scalar_type());
    TORCH_CHECK(run_dev.is_contiguous(), op, ": run_dev must be contiguous");
    check_int32_contiguous(op, run_offsets, "run_offsets");
    check_int32_contiguous(op, run_prio, "run_prio");
    check_int32_contiguous(op, node_offsets, "node_offsets");
    const int64_t N = free_core.size(0);
    if (pod_prio)
        TORCH_CHECK_VALUE(pod_prio->dim() == 1 && pod_prio->size(0) == G, op, ": pod_prio must be [G] = [", G,
                          "], got ", pod_prio->sizes());
    TORCH_CHECK_VALUE(run_core.dim() == 1 && run_mem.sizes() == run_core.sizes() && run_dev.sizes() == run_core.sizes(),
                      op, ": run_core, run_mem and run_dev must all be [Q], got ", run_core.sizes(), ", ",
                      run_mem.sizes(), " and ", run_dev.sizes());
    TORCH_CHECK_VALUE(run_offsets.dim() == 1 && run_offsets.size(0) >= 1, op, ": run_offsets must be [H + 1], got ",
                      run_offsets.sizes());
    const int64_t Q = run_core.size(0), H = run_offsets.size(0) - 1;
    constexpr int64_t kMax = std::numeric_limits<int32_t>::max();
    TORCH_CHECK_VALUE(Q < kMax && H < kMax, op, ": Q and H + 1 must be below 2^31, got ", Q, " and ", H + 1);
    TORCH_CHECK_VALUE(run_prio.dim() == 1 && run_prio.size(0) == H, op, ": run_prio must be [H] = [", H, "], got ",
                      run_prio.sizes());
    TORCH_CHECK_VALUE(node_offsets.dim() == 1 && node_offsets.size(0) == N + 1, op, ": node_offsets must be [N + 1] = [",
                      N + 1, "], got ", node_offsets.sizes());
    for (const at::Tensor* t : {pod_prio, &run_core, &run_mem, &run_dev, &run_offsets, &run_prio, &node_offsets})
        TORCH_CHECK(!t || t->is_cuda() && t->device() == free_core.device(), op,
                    ": every tensor must be on one CUDA device, got ", t->device(), " and ", free_core.device());
    return {Q, H};
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> preempt_pods(
    const at::Tensor& free_core, const at::Tensor& free_mem, const at::Tensor& d_valid, const at::Tensor& req_core,
    const at::Tensor& req_mem, const at::Tensor& pod_offsets, const at::Tensor& pod_prio, const at::Tensor& run_core,
    const at::Tensor& run_mem, const at::Tensor& run_dev, const at::Tensor& run_offsets, const at::Tensor& run_prio,
    const at::Tensor& node_offsets) {
    const auto [N, D, P] = check_inputs("preempt_pods", free_core, free_mem, d_valid, req_core, req_mem);
    const int64_t G = check_pod_offsets("preempt_pods", free_core, pod_offsets);
    const auto [Q, H] = check_running("preempt_pods", free_core, G, &pod_prio, run_core, run_mem, run_dev, run_offsets,
                                      run_prio, node_offsets);
    const at::Device dev = free_core.device();
    const c10::cuda::CUDAGuard guard(dev);
    at::Tensor node = at::empty({G}, free_core.options());
    at::Tensor dv_out = at::empty({P}, free_core.options().dtype(at::kChar));
    at::Tensor evicted = at::empty({H}, free_core.options());
    at::Tensor fc_out = at::empty({N, D}, free_core.options());
    at::Tensor fm_out = at::empty({N, D}, free_core.options());
    at::Tensor info = at::empty({3}, free_core.options());
    if (N == 0 || P == 0) {  // nothing to place, or nowhere to place it
        node.fill_(-1);
        dv_out.fill_(-1);
        evicted.fill_(-1);
        fc_out.copy_(free_core);
        fm_out.copy_(free_mem);
        info.zero_();
        return {node, dv_out, evicted, fc_out, fm_out, info};
    }
    at::Tensor scratch =
        at::empty({static_cast<int64_t>(egpu::preempt_scratch_bytes(static_cast<int>(N), static_cast<int>(G)))},
                  free_core.options().dtype(at::kByte));
    const cudaError_t err = egpu::preempt_launch(
        free_core.data_ptr<int32_t>(), free_mem.data_ptr<int32_t>(), d_valid.data_ptr<int32_t>(), static_cast<int>(N),
        static_cast<int>(D), req_core.data_ptr<int32_t>(), req_mem.data_ptr<int32_t>(), static_cast<int>(P),
        pod_offsets.data_ptr<int32_t>(), pod_prio.data_ptr<int32_t>(), static_cast<int>(G), run_core.data_ptr<int32_t>(),
        run_mem.data_ptr<int32_t>(), run_dev.data_ptr<int8_t>(), static_cast<int>(Q), run_offsets.data_ptr<int32_t>(),
        run_prio.data_ptr<int32_t>(), static_cast<int>(H), node_offsets.data_ptr<int32_t>(), node.data_ptr<int32_t>(),
        dv_out.data_ptr<int8_t>(), evicted.data_ptr<int32_t>(), fc_out.data_ptr<int32_t>(), fm_out.data_ptr<int32_t>(),
        info.data_ptr<int32_t>(), scratch.data_ptr(), dev.index(), c10::cuda::getCurrentCUDAStream(dev.index()).stream());
    TORCH_CHECK(err == cudaSuccess, "preempt_pods: launch failed: ", cudaGetErrorString(err));
    return {node, dv_out, evicted, fc_out, fm_out, info};
}

// DESIGN.md §2.15.  place_gangs' and preempt_pods' checks naming preempt_gangs, then the dtype and layout of
// gang_prio, run_gang and run_gang_min, their shapes, and their device; their values are the kernel's to check.
// Returns R.
int64_t check_running_gangs(const at::Tensor& free_core, int64_t J, int64_t H, const at::Tensor& gang_prio,
                            const at::Tensor& run_gang, const at::Tensor& run_gang_min) {
    constexpr const char* op = "preempt_gangs";
    check_int32_contiguous(op, gang_prio, "gang_prio");
    check_int32_contiguous(op, run_gang, "run_gang");
    check_int32_contiguous(op, run_gang_min, "run_gang_min");
    TORCH_CHECK_VALUE(gang_prio.dim() == 1 && gang_prio.size(0) == J, op, ": gang_prio must be [J] = [", J, "], got ",
                      gang_prio.sizes());
    TORCH_CHECK_VALUE(run_gang.dim() == 1 && run_gang.size(0) == H, op, ": run_gang must be [H] = [", H, "], got ",
                      run_gang.sizes());
    TORCH_CHECK_VALUE(run_gang_min.dim() == 1, op, ": run_gang_min must be [R], got ", run_gang_min.sizes());
    const int64_t R = run_gang_min.size(0);
    TORCH_CHECK_VALUE(R < std::numeric_limits<int32_t>::max(), op, ": R must be below 2^31 - 1, got ", R);
    for (const at::Tensor* t : {&gang_prio, &run_gang, &run_gang_min})
        TORCH_CHECK(t->is_cuda() && t->device() == free_core.device(), op,
                    ": every tensor must be on one CUDA device, got ", t->device(), " and ", free_core.device());
    return R;
}

std::tuple<at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor, at::Tensor> preempt_gangs(
    const at::Tensor& free_core, const at::Tensor& free_mem, const at::Tensor& d_valid, const at::Tensor& req_core,
    const at::Tensor& req_mem, const at::Tensor& pod_offsets, const at::Tensor& gang_offsets,
    const at::Tensor& gang_min, const at::Tensor& gang_prio, const at::Tensor& run_core, const at::Tensor& run_mem,
    const at::Tensor& run_dev, const at::Tensor& run_offsets, const at::Tensor& run_prio,
    const at::Tensor& node_offsets, const at::Tensor& run_gang, const at::Tensor& run_gang_min) {
    constexpr const char* op = "preempt_gangs";
    const auto [N, D, P] = check_inputs(op, free_core, free_mem, d_valid, req_core, req_mem);
    const int64_t G = check_pod_offsets(op, free_core, pod_offsets);
    const int64_t J = check_gangs(op, free_core, gang_offsets, gang_min);
    const auto [Q, H] = check_running(op, free_core, G, nullptr, run_core, run_mem, run_dev, run_offsets, run_prio,
                                      node_offsets);
    const int64_t R = check_running_gangs(free_core, J, H, gang_prio, run_gang, run_gang_min);
    const at::Device dev = free_core.device();
    const c10::cuda::CUDAGuard guard(dev);
    at::Tensor node = at::empty({G}, free_core.options());
    at::Tensor dv_out = at::empty({P}, free_core.options().dtype(at::kChar));
    at::Tensor placed = at::empty({J}, free_core.options());
    at::Tensor evicted = at::empty({H}, free_core.options());
    at::Tensor fc_out = at::empty({N, D}, free_core.options());
    at::Tensor fm_out = at::empty({N, D}, free_core.options());
    at::Tensor info = at::empty({3}, free_core.options());
    if (N == 0 || P == 0) {  // nothing to place, or nowhere to place it
        node.fill_(-1);
        dv_out.fill_(-1);
        placed.zero_();
        evicted.fill_(-1);
        fc_out.copy_(free_core);
        fm_out.copy_(free_mem);
        info.zero_();
        return {node, dv_out, placed, evicted, fc_out, fm_out, info};
    }
    at::Tensor scratch = at::empty({static_cast<int64_t>(egpu::preempt_gangs_scratch_bytes(
                                       static_cast<int>(N), static_cast<int>(G), static_cast<int>(J), static_cast<int>(R)))},
                                   free_core.options().dtype(at::kByte));
    const cudaError_t err = egpu::preempt_gangs_launch(
        free_core.data_ptr<int32_t>(), free_mem.data_ptr<int32_t>(), d_valid.data_ptr<int32_t>(), static_cast<int>(N),
        static_cast<int>(D), req_core.data_ptr<int32_t>(), req_mem.data_ptr<int32_t>(), static_cast<int>(P),
        pod_offsets.data_ptr<int32_t>(), static_cast<int>(G), gang_offsets.data_ptr<int32_t>(),
        gang_min.data_ptr<int32_t>(), gang_prio.data_ptr<int32_t>(), static_cast<int>(J), run_core.data_ptr<int32_t>(),
        run_mem.data_ptr<int32_t>(), run_dev.data_ptr<int8_t>(), static_cast<int>(Q), run_offsets.data_ptr<int32_t>(),
        run_prio.data_ptr<int32_t>(), static_cast<int>(H), node_offsets.data_ptr<int32_t>(), run_gang.data_ptr<int32_t>(),
        run_gang_min.data_ptr<int32_t>(), static_cast<int>(R), node.data_ptr<int32_t>(), dv_out.data_ptr<int8_t>(),
        placed.data_ptr<int32_t>(), evicted.data_ptr<int32_t>(), fc_out.data_ptr<int32_t>(), fm_out.data_ptr<int32_t>(),
        info.data_ptr<int32_t>(), scratch.data_ptr(), dev.index(), c10::cuda::getCurrentCUDAStream(dev.index()).stream());
    TORCH_CHECK(err == cudaSuccess, "preempt_gangs: launch failed: ", cudaGetErrorString(err));
    return {node, dv_out, placed, evicted, fc_out, fm_out, info};
}

}  // namespace

TORCH_LIBRARY(egpu, m) {
    m.def("bestfit_tables(Tensor free_core, Tensor free_mem, Tensor d_valid, Tensor req_core, Tensor req_mem) -> "
          "(Tensor, Tensor)");
    m.def("place_tables(Tensor free_core, Tensor free_mem, Tensor d_valid, Tensor req_core, Tensor req_mem) -> "
          "(Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("place_pods(Tensor free_core, Tensor free_mem, Tensor d_valid, Tensor req_core, Tensor req_mem, "
          "Tensor pod_offsets) -> (Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("place_gangs(Tensor free_core, Tensor free_mem, Tensor d_valid, Tensor req_core, Tensor req_mem, "
          "Tensor pod_offsets, Tensor gang_offsets, Tensor gang_min) -> (Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("preempt_pods(Tensor free_core, Tensor free_mem, Tensor d_valid, Tensor req_core, Tensor req_mem, "
          "Tensor pod_offsets, Tensor pod_prio, Tensor run_core, Tensor run_mem, Tensor run_dev, Tensor run_offsets, "
          "Tensor run_prio, Tensor node_offsets) -> (Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)");
    m.def("preempt_gangs(Tensor free_core, Tensor free_mem, Tensor d_valid, Tensor req_core, Tensor req_mem, "
          "Tensor pod_offsets, Tensor gang_offsets, Tensor gang_min, Tensor gang_prio, Tensor run_core, Tensor run_mem, "
          "Tensor run_dev, Tensor run_offsets, Tensor run_prio, Tensor node_offsets, Tensor run_gang, "
          "Tensor run_gang_min) -> (Tensor, Tensor, Tensor, Tensor, Tensor, Tensor, Tensor)");
}

// The CPU registration only refuses (the device check above): a CPU caller gets the same messages as a CUDA one.
TORCH_LIBRARY_IMPL(egpu, CUDA, m) {
    m.impl("bestfit_tables", &bestfit_tables);
    m.impl("place_tables", &place_tables);
    m.impl("place_pods", &place_pods);
    m.impl("place_gangs", &place_gangs);
    m.impl("preempt_pods", &preempt_pods);
    m.impl("preempt_gangs", &preempt_gangs);
}
TORCH_LIBRARY_IMPL(egpu, CPU, m) {
    m.impl("bestfit_tables", &bestfit_tables);
    m.impl("place_tables", &place_tables);
    m.impl("place_pods", &place_pods);
    m.impl("place_gangs", &place_gangs);
    m.impl("preempt_pods", &preempt_pods);
    m.impl("preempt_gangs", &preempt_gangs);
}

// egpu_tables.h — launcher of the multi-table best-fit scan (egpu_tables.cu), called by the
// PyTorch operator egpu::bestfit_tables (egpu_tables_op.cc).  Not part of the C ABI of include/.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace egpu {

// Scores P requests against N tables (DESIGN.md §2.10).  free_core / free_mem: int32[N][D], row-major;
// d_valid: int32[N]; req_core / req_mem: int32[P]; out_idx: int8[N][P]; out_key: int32[N][P].  All device
// pointers of `device`; 1 <= D <= 64, N >= 1, P >= 1 (the caller has checked the shapes).  Asynchronous
// on `stream`; returns the launch's error.
cudaError_t tables_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                          const int32_t* req_core, const int32_t* req_mem, int P, int8_t* out_idx, int32_t* out_key,
                          int device, cudaStream_t stream);

}  // namespace egpu

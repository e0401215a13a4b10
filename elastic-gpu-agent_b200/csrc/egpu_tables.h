// egpu_tables.h — launchers of the multi-table best-fit scan and placements (egpu_tables.cu), called by the
// PyTorch operators egpu::bestfit_tables, egpu::place_tables, egpu::place_pods, egpu::place_gangs,
// egpu::preempt_pods and egpu::preempt_gangs (egpu_tables_op.cc).  Not part of the C ABI of include/.
#pragma once
#include <cstddef>
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

// Bytes of device scratch place_launch needs for P requests (16-byte aligned, from the caller's allocator).
size_t place_scratch_bytes(int P);

// Places P requests on N tables by best-fit rounds to the fixed point (DESIGN.md §2.11) in one cooperative
// launch.  Inputs as tables_launch; out_node: int32[P]; out_dev: int8[P]; free_core_out / free_mem_out:
// int32[N][D]; info: int32[2].  scratch: place_scratch_bytes(P) bytes; its head is zeroed here on `stream`.
// N >= 1, P >= 1.  Asynchronous on `stream`; returns the first error of the memset or the launch.
cudaError_t place_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                         const int32_t* req_core, const int32_t* req_mem, int P, int32_t* out_node, int8_t* out_dev,
                         int32_t* free_core_out, int32_t* free_mem_out, int32_t* info, void* scratch, int device,
                         cudaStream_t stream);

// Bytes of device scratch pods_launch needs for G pods (16-byte aligned, from the caller's allocator).
size_t pods_scratch_bytes(int G);

// Places G pods of P containers on N tables, every container of a pod on one node, by best-fit rounds to the fixed
// point (DESIGN.md §2.12) in one cooperative launch.  Tables and containers as place_launch; pod_offsets:
// int32[G + 1], checked by the kernel before any container is read through it; out_node: int32[G]; out_dev:
// int8[P]; free_core_out / free_mem_out: int32[N][D]; info: int32[3].  scratch: pods_scratch_bytes(G) bytes; its
// head is zeroed here on `stream`.  N >= 1, P >= 1, G >= 0.  Asynchronous on `stream`; returns the first error of
// the memset or the launch.
cudaError_t pods_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                        const int32_t* req_core, const int32_t* req_mem, int P, const int32_t* pod_offsets, int G,
                        int32_t* out_node, int8_t* out_dev, int32_t* free_core_out, int32_t* free_mem_out, int32_t* info,
                        void* scratch, int device, cudaStream_t stream);

// Bytes of device scratch gangs_launch needs for G pods in J gangs (16-byte aligned, from the caller's allocator).
size_t gangs_scratch_bytes(int G, int J);

// Places J gangs of G pods of P containers on N tables, in gang order, each gang kept when at least gang_min of its pods
// are placed and rolled back otherwise (DESIGN.md §2.13), in one cooperative launch.  Tables, containers and
// pod_offsets as pods_launch; gang_offsets: int32[J + 1]; gang_min: int32[J]; the kernel checks all three index
// tensors before it reads anything through them.  out_node: int32[G]; out_dev: int8[P]; out_placed: int32[J];
// free_core_out / free_mem_out: int32[N][D]; info: int32[3].  scratch: gangs_scratch_bytes(G, J) bytes; its head is
// zeroed here on `stream`.  N >= 1, P >= 1, G >= 0, J >= 0.  Asynchronous on `stream`; returns the first error of the
// memset or the launch.
cudaError_t gangs_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                         const int32_t* req_core, const int32_t* req_mem, int P, const int32_t* pod_offsets, int G,
                         const int32_t* gang_offsets, const int32_t* gang_min, int J, int32_t* out_node, int8_t* out_dev,
                         int32_t* out_placed, int32_t* free_core_out, int32_t* free_mem_out, int32_t* info, void* scratch,
                         int device, cudaStream_t stream);

// Bytes of device scratch preempt_launch needs for G pods on N tables (16-byte aligned, from the caller's allocator).
size_t preempt_scratch_bytes(int N, int G);

// Places G pods of P containers on N tables as pods_launch, evicting lower-priority running pods where a pod fits no
// table as it is (DESIGN.md §2.14), in one cooperative launch.  Tables, containers and pod_offsets as pods_launch;
// pod_prio: int32[G]; running containers run_core / run_mem: int32[Q], run_dev: int8[Q]; run_offsets: int32[H + 1];
// run_prio: int32[H]; node_offsets: int32[N + 1].  The kernel checks the three offset tensors before it reads anything
// through them.  out_node: int32[G]; out_dev: int8[P]; out_evicted: int32[H]; free_core_out / free_mem_out:
// int32[N][D]; info: int32[3].  scratch: preempt_scratch_bytes(N, G) bytes; its head is zeroed here on `stream`.
// N >= 1, P >= 1, G >= 0, Q >= 0, H >= 0.  Asynchronous on `stream`; returns the first error of the memset or the
// launch.
cudaError_t preempt_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                           const int32_t* req_core, const int32_t* req_mem, int P, const int32_t* pod_offsets,
                           const int32_t* pod_prio, int G, const int32_t* run_core, const int32_t* run_mem,
                           const int8_t* run_dev, int Q, const int32_t* run_offsets, const int32_t* run_prio, int H,
                           const int32_t* node_offsets, int32_t* out_node, int8_t* out_dev, int32_t* out_evicted,
                           int32_t* free_core_out, int32_t* free_mem_out, int32_t* info, void* scratch, int device,
                           cudaStream_t stream);

// Bytes of device scratch preempt_gangs_launch needs for G pods in J gangs on N tables with R running jobs (16-byte
// aligned, from the caller's allocator).
size_t preempt_gangs_scratch_bytes(int N, int G, int J, int R);

// Places J gangs of G pods of P containers on N tables in gang order as gangs_launch, each gang's pods by
// preempt_launch's rounds at the gang's priority, never evicting a running job below its minAvailable (DESIGN.md
// §2.15), in one cooperative launch.  Tables, containers, pod_offsets, gang_offsets and gang_min as gangs_launch;
// gang_prio: int32[J]; running pods as preempt_launch; run_gang: int32[H] in [-1, R); run_gang_min: int32[R] >= 0.
// The kernel checks the five index tensors and run_gang_min before it reads anything through them.  out_node:
// int32[G]; out_dev: int8[P]; out_placed: int32[J]; out_evicted: int32[H]; free_core_out / free_mem_out: int32[N][D];
// info: int32[3].  scratch: preempt_gangs_scratch_bytes(N, G, J, R) bytes; its head is zeroed here on `stream`.
// N >= 1, P >= 1, G, J, Q, H, R >= 0.  Asynchronous on `stream`; returns the first error of the memset or the launch.
cudaError_t preempt_gangs_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N,
                                 int D, const int32_t* req_core, const int32_t* req_mem, int P,
                                 const int32_t* pod_offsets, int G, const int32_t* gang_offsets, const int32_t* gang_min,
                                 const int32_t* gang_prio, int J, const int32_t* run_core, const int32_t* run_mem,
                                 const int8_t* run_dev, int Q, const int32_t* run_offsets, const int32_t* run_prio,
                                 int H, const int32_t* node_offsets, const int32_t* run_gang,
                                 const int32_t* run_gang_min, int R, int32_t* out_node, int8_t* out_dev,
                                 int32_t* out_placed, int32_t* out_evicted, int32_t* free_core_out,
                                 int32_t* free_mem_out, int32_t* info, void* scratch, int device, cudaStream_t stream);

}  // namespace egpu

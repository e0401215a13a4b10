// How fast can one batch of the int32 ABI cross PCIe?  12 bytes per request: 8 in, 4 out.
// The library's scan reads pinned host memory in place (zero-copy), in and out concurrently; a
// copy-engine pipeline measured slower when it was tried inside the library (DESIGN.md 7.2).  This probe isolates the transport:
//   A  zero-copy kernel (ld.global.nc.v4 from mapped host memory, st.v4 to mapped host memory),
//      grid x rows-per-thread sweep: how many loads must be in flight to fill the link?
//   B  copy engines only: H2D of both arrays, D2H of the result, 1/2/4/8/16 chunks on three
//      streams (in / compute stand-in / out) with events - the best a staged pipeline can do
//   C  mixed: copy engine in, zero-copy stores out (the link is full duplex)
// Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o pcie_e2e_probe pcie_e2e_probe.cu
// Prints microseconds per 1 M-request batch for each variant (median of 20).
#include <algorithm>
#include <cstdio>
#include <vector>

#include <cuda_runtime.h>

#define CK(x)                                                                      \
    do {                                                                           \
        cudaError_t e_ = (x);                                                      \
        if (e_ != cudaSuccess) {                                                   \
            std::printf("%s: %s\n", #x, cudaGetErrorString(e_));                   \
            return 1;                                                              \
        }                                                                          \
    } while (0)

__device__ __forceinline__ int4 ldnc(const int* p) {
    int4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.s32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
    return v;
}

// stand-in for the scan: one cheap op per request so that the transport is what is measured
template <int UNROLL>
__global__ void touch(const int* __restrict__ a, const int* __restrict__ b, int* __restrict__ out, long long nvec) {
    const long long stride = static_cast<long long>(gridDim.x) * blockDim.x;
    long long v = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    for (; v + (UNROLL - 1) * stride < nvec; v += UNROLL * stride) {
        int4 x[UNROLL], y[UNROLL];
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            x[u] = ldnc(a + 4 * (v + u * stride));
            y[u] = ldnc(b + 4 * (v + u * stride));
        }
#pragma unroll
        for (int u = 0; u < UNROLL; ++u) {
            int4 r = make_int4(x[u].x ^ y[u].x, x[u].y ^ y[u].y, x[u].z ^ y[u].z, x[u].w ^ y[u].w);
            *reinterpret_cast<int4*>(out + 4 * (v + u * stride)) = r;
        }
    }
    for (; v < nvec; v += stride) {
        const int4 x = ldnc(a + 4 * v), y = ldnc(b + 4 * v);
        *reinterpret_cast<int4*>(out + 4 * v) = make_int4(x.x ^ y.x, x.y ^ y.y, x.z ^ y.z, x.w ^ y.w);
    }
}

static float median(std::vector<float>& v) {
    std::sort(v.begin(), v.end());
    return v[v.size() / 2];
}

int main() {
    const long long R = 1 << 20, nvec = R / 4;
    int *ha, *hb, *ho, *da, *db, *dout;
    CK(cudaHostAlloc(&ha, 4 * R, cudaHostAllocMapped));
    CK(cudaHostAlloc(&hb, 4 * R, cudaHostAllocMapped));
    CK(cudaHostAlloc(&ho, 4 * R, cudaHostAllocMapped));
    CK(cudaMalloc(&da, 4 * R));
    CK(cudaMalloc(&db, 4 * R));
    CK(cudaMalloc(&dout, 4 * R));
    for (long long i = 0; i < R; ++i) ha[i] = static_cast<int>(i), hb[i] = static_cast<int>(3 * i);
    int *za, *zb, *zo;
    CK(cudaHostGetDevicePointer(&za, ha, 0));
    CK(cudaHostGetDevicePointer(&zb, hb, 0));
    CK(cudaHostGetDevicePointer(&zo, ho, 0));
    cudaStream_t s_in, s_k, s_out;
    CK(cudaStreamCreateWithFlags(&s_in, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&s_k, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&s_out, cudaStreamNonBlocking));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    const int reps = 20;

    // ---- A: zero-copy kernel, grid x unroll
    for (int grid : {33, 66, 132, 264}) {
        for (int unroll : {1, 2, 4}) {
            std::vector<float> t;
            for (int r = 0; r < reps + 3; ++r) {
                CK(cudaEventRecord(e0, s_k));
                if (unroll == 1) touch<1><<<grid, 256, 0, s_k>>>(za, zb, zo, nvec);
                else if (unroll == 2) touch<2><<<grid, 256, 0, s_k>>>(za, zb, zo, nvec);
                else touch<4><<<grid, 256, 0, s_k>>>(za, zb, zo, nvec);
                CK(cudaEventRecord(e1, s_k));
                CK(cudaEventSynchronize(e1));
                float ms;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                if (r >= 3) t.push_back(ms * 1e3f);
            }
            std::printf("A zero-copy  grid %3d x 256, %d vector pairs in flight per thread: %7.1f us  (in %.1f GB/s)\n", grid, unroll,
                        median(t), 8.0 * R / median(t) * 1e-3);
        }
    }
    // ---- B: copy engines, chunked three-stage pipeline
    for (int chunks : {1, 2, 4, 8, 16}) {
        std::vector<cudaEvent_t> in_done(chunks), k_done(chunks);
        for (int c = 0; c < chunks; ++c) {
            CK(cudaEventCreateWithFlags(&in_done[c], cudaEventDisableTiming));
            CK(cudaEventCreateWithFlags(&k_done[c], cudaEventDisableTiming));
        }
        const long long per = R / chunks;
        std::vector<float> t;
        for (int r = 0; r < reps + 3; ++r) {
            CK(cudaDeviceSynchronize());
            CK(cudaEventRecord(e0, s_in));
            CK(cudaStreamWaitEvent(s_k, e0, 0));
            CK(cudaStreamWaitEvent(s_out, e0, 0));
            for (int c = 0; c < chunks; ++c) {
                const long long o = c * per;
                CK(cudaMemcpyAsync(da + o, ha + o, 4 * per, cudaMemcpyHostToDevice, s_in));
                CK(cudaMemcpyAsync(db + o, hb + o, 4 * per, cudaMemcpyHostToDevice, s_in));
                CK(cudaEventRecord(in_done[c], s_in));
                CK(cudaStreamWaitEvent(s_k, in_done[c], 0));
                touch<2><<<132, 256, 0, s_k>>>(da + o, db + o, dout + o, per / 4);
                CK(cudaEventRecord(k_done[c], s_k));
                CK(cudaStreamWaitEvent(s_out, k_done[c], 0));
                CK(cudaMemcpyAsync(ho + o, dout + o, 4 * per, cudaMemcpyDeviceToHost, s_out));
            }
            CK(cudaEventRecord(e1, s_out));
            CK(cudaEventSynchronize(e1));
            float ms;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (r >= 3) t.push_back(ms * 1e3f);
        }
        std::printf("B copy engines, %2d chunk(s): %7.1f us\n", chunks, median(t));
    }
    // ---- C: copy engine in, zero-copy stores out
    for (int chunks : {1, 4, 8, 16}) {
        std::vector<cudaEvent_t> in_done(chunks);
        for (int c = 0; c < chunks; ++c) CK(cudaEventCreateWithFlags(&in_done[c], cudaEventDisableTiming));
        const long long per = R / chunks;
        std::vector<float> t;
        for (int r = 0; r < reps + 3; ++r) {
            CK(cudaDeviceSynchronize());
            CK(cudaEventRecord(e0, s_in));
            CK(cudaStreamWaitEvent(s_k, e0, 0));
            for (int c = 0; c < chunks; ++c) {
                const long long o = c * per;
                CK(cudaMemcpyAsync(da + o, ha + o, 4 * per, cudaMemcpyHostToDevice, s_in));
                CK(cudaMemcpyAsync(db + o, hb + o, 4 * per, cudaMemcpyHostToDevice, s_in));
                CK(cudaEventRecord(in_done[c], s_in));
                CK(cudaStreamWaitEvent(s_k, in_done[c], 0));
                touch<2><<<62, 256, 0, s_k>>>(da + o, db + o, zo + o, per / 4);
            }
            CK(cudaEventRecord(e1, s_k));
            CK(cudaEventSynchronize(e1));
            float ms;
            CK(cudaEventElapsedTime(&ms, e0, e1));
            if (r >= 3) t.push_back(ms * 1e3f);
        }
        std::printf("C copy engine in + zero-copy out, %2d chunk(s): %7.1f us\n", chunks, median(t));
    }
    return 0;
}

// egpu_tables.cu — best fit of P requests against N capacity tables in one launch (sm_90a), the kernel
// of the PyTorch operator egpu::bestfit_tables (DESIGN.md §2.10, §4.5).
//
// The request cancels out of the best-fit order (§4.1), so a table's answer to every request is the
// first feasible row of that table sorted by (fc, fm, d).  One CTA takes a tile of kTabWarps tables
// and a chunk of the request vector.  Warp w sorts table w of the tile in shared memory (rank sort,
// as resort_table_cta), keeps its packed compare words in registers and streams the chunk: each lane
// scores four consecutive requests per step with first_feasible, so a warp writes 128 contiguous
// index bytes and 512 contiguous key bytes per step.  The 8 bytes per request are read once per tile
// (the 8 warps of a CTA share them through L1); the 5 bytes per pair written are what the launch moves.
// No barrier wider than a warp: every warp owns its table.
#include "egpu_kernels.cuh"
#include "egpu_tables.h"

namespace egpu {

constexpr int kTabWarps = 8;  // tables per CTA
constexpr int kTabThreads = kTabWarps * 32;
constexpr int kTabStep = 4 * 32;       // requests one warp scores per step
constexpr uint32_t kNoKey = 0x7fffffffu;  // the key of "no feasible device"

template <int DT, bool VEC>
__global__ void __launch_bounds__(kTabThreads)
bestfit_tables_kernel(const int32_t* __restrict__ free_core, const int32_t* __restrict__ free_mem,
                      const int32_t* __restrict__ d_valid, int N, int D, const int32_t* __restrict__ req_core,
                      const int32_t* __restrict__ req_mem, int P, int chunk, int8_t* __restrict__ out_idx,
                      int32_t* __restrict__ out_key, uint32_t gx, uint32_t gm) {
    // sK: packed compare words by sorted position (kPadWord past the table).  sBase: (fc << 24 | fm << 6 | d) by
    // sorted position, kNoKey at every position that is no row, including "none" (32 for DT <= 32, 64 for DT = 64):
    // the chosen position's base minus (core << 24 | mem << 6) is the key, and its low six bits are the device.
    __shared__ __align__(16) uint32_t sK[kTabWarps][DT];
    __shared__ uint32_t sBase[kTabWarps][kMaxD + 1];
    __shared__ uint32_t sRank[kTabWarps][kMaxD];
    const int lane = threadIdx.x & 31;
    const int warp = threadIdx.x >> 5;
    const int n = blockIdx.x * kTabWarps + warp;
    if (n >= N) return;  // ragged last tile: nothing below waits for the other warps

    // A table outside §2.1's domain (d_valid not in [1, D], or a row value out of range) answers -1 everywhere.
    // The operator's Python interface refuses such tables before the launch; this keeps the kernel defined
    // for callers of the raw operator, whose checks cannot read device data.
    const int dv = d_valid[n];
    bool ok = dv >= 1 && dv <= D;
    const int32_t* fc_row = free_core + static_cast<size_t>(n) * D;
    const int32_t* fm_row = free_mem + static_cast<size_t>(n) * D;
    for (int j = lane; j < DT; j += 32) {
        uint32_t rank = 0xffffffffu;
        if (ok && j < dv) {
            const int32_t c = fc_row[j], m = fm_row[j];
            if (c < 0 || c > kCoreMax || m < 0 || m > kMemMax) ok = false;
            rank = (static_cast<uint32_t>(c) << 24) | (static_cast<uint32_t>(m) << 6) | static_cast<uint32_t>(j);
        }
        sRank[warp][j] = rank;
        sK[warp][j] = kPadWord;
    }
    for (int j = lane; j <= kMaxD; j += 32) sBase[warp][j] = kNoKey;
    const int rows = __all_sync(0xffffffffu, ok) ? dv : 0;
    __syncwarp();
    for (int j = lane; j < rows; j += 32) {
        const uint32_t mine = sRank[warp][j];
        int pos = 0;
        for (int k = 0; k < rows; ++k) pos += sRank[warp][k] < mine;
        sK[warp][pos] = pack_table_word(static_cast<int32_t>(mine >> 24), static_cast<int32_t>((mine >> 6) & 0x3FFFFu)) |
                        (static_cast<uint32_t>(pos) & 31u);
        sBase[warp][pos] = mine;
    }
    __syncwarp();
    uint32_t K[DT];
#pragma unroll
    for (int j = 0; j < DT; j += 4) {
        const uint4 k4 = *reinterpret_cast<const uint4*>(&sK[warp][j]);
        K[j] = k4.x; K[j + 1] = k4.y; K[j + 2] = k4.z; K[j + 3] = k4.w;
    }
    const uint32_t* base_of = sBase[warp];

    auto decide = [&](int32_t core, int32_t mem, int32_t& key) -> int32_t {
        const uint32_t base = base_of[first_feasible<DT>(K, pack_request_word(core, mem), gx, gm)];
        const bool none = base == kNoKey;
        // feasible: 0 <= core <= fc and 0 <= mem <= fm, so the fields subtract without a borrow
        key = static_cast<int32_t>(none ? kNoKey : base - ((static_cast<uint32_t>(core) << 24) | (static_cast<uint32_t>(mem) << 6)));
        return none ? -1 : static_cast<int32_t>(base & 63u);
    };

    const int p_lo = blockIdx.y * chunk;
    const int p_hi = min(P, p_lo + chunk);
    const size_t row = static_cast<size_t>(n) * static_cast<size_t>(P);
    if constexpr (VEC) {  // P % 4 == 0 and 16-byte aligned requests: chunk bounds are multiples of 4
        const int4* vc = reinterpret_cast<const int4*>(req_core);
        const int4* vm = reinterpret_cast<const int4*>(req_mem);
        uint32_t* vo = reinterpret_cast<uint32_t*>(out_idx + row);
        int32_t* ko = out_key + row;
        for (int v = (p_lo >> 2) + lane; v < (p_hi >> 2); v += 32) {
            const int4 c = __ldg(vc + v), m = __ldg(vm + v);
            int4 k;
            const int32_t i0 = decide(c.x, m.x, k.x), i1 = decide(c.y, m.y, k.y);
            const int32_t i2 = decide(c.z, m.z, k.z), i3 = decide(c.w, m.w, k.w);
            st_stream_u32(vo + v, (static_cast<uint32_t>(i0) & 0xffu) | ((static_cast<uint32_t>(i1) & 0xffu) << 8) |
                                      ((static_cast<uint32_t>(i2) & 0xffu) << 16) | (static_cast<uint32_t>(i3) << 24));
            st_stream_v4(ko + 4 * static_cast<size_t>(v), k);
        }
    } else {
        for (int p = p_lo + lane; p < p_hi; p += 32) {
            int32_t k;
            const int32_t i = decide(__ldg(req_core + p), __ldg(req_mem + p), k);
            out_idx[row + p] = static_cast<int8_t>(i);
            out_key[row + p] = k;
        }
    }
}

template <int DT>
cudaError_t launch_bucket(bool vec, dim3 grid, cudaStream_t stream, const int32_t* fc, const int32_t* fm, const int32_t* dv,
                          int N, int D, const int32_t* rc, const int32_t* rm, int P, int chunk, int8_t* idx, int32_t* key) {
    if (vec)
        bestfit_tables_kernel<DT, true><<<grid, kTabThreads, 0, stream>>>(fc, fm, dv, N, D, rc, rm, P, chunk, idx, key, kGuards,
                                                                          kCandMask);
    else
        bestfit_tables_kernel<DT, false><<<grid, kTabThreads, 0, stream>>>(fc, fm, dv, N, D, rc, rm, P, chunk, idx, key, kGuards,
                                                                           kCandMask);
    return cudaGetLastError();
}

cudaError_t tables_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                          const int32_t* req_core, const int32_t* req_mem, int P, int8_t* out_idx, int32_t* out_key,
                          int device, cudaStream_t stream) {
    int sms = 0;
    cudaError_t err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err != cudaSuccess) return err;
    // Grid: one column of CTAs per tile of tables; the request vector is cut into as many chunks as it takes to
    // give the launch about four CTAs per SM (at N = 5 000 the tiles alone do; at N = 512 eight chunks of 1 024).
    // A chunk is a whole number of warp steps, so only the last chunk of a row is ragged.
    const int tiles = (N + kTabWarps - 1) / kTabWarps;
    const int steps = (P + kTabStep - 1) / kTabStep;
    const int want = (4 * sms + tiles - 1) / tiles;
    const int chunks_wanted = want < 1 ? 1 : (want > steps ? steps : want);
    const int chunk = ((steps + chunks_wanted - 1) / chunks_wanted) * kTabStep;
    const dim3 grid(static_cast<unsigned>(tiles), static_cast<unsigned>((P + chunk - 1) / chunk));
    const bool vec = (P % 4) == 0 && (reinterpret_cast<uintptr_t>(req_core) % 16) == 0 &&
                     (reinterpret_cast<uintptr_t>(req_mem) % 16) == 0 && (reinterpret_cast<uintptr_t>(out_idx) % 4) == 0 &&
                     (reinterpret_cast<uintptr_t>(out_key) % 16) == 0;
    if (D <= 8) return launch_bucket<8>(vec, grid, stream, free_core, free_mem, d_valid, N, D, req_core, req_mem, P, chunk, out_idx, out_key);
    if (D <= 16) return launch_bucket<16>(vec, grid, stream, free_core, free_mem, d_valid, N, D, req_core, req_mem, P, chunk, out_idx, out_key);
    if (D <= 32) return launch_bucket<32>(vec, grid, stream, free_core, free_mem, d_valid, N, D, req_core, req_mem, P, chunk, out_idx, out_key);
    return launch_bucket<64>(vec, grid, stream, free_core, free_mem, d_valid, N, D, req_core, req_mem, P, chunk, out_idx, out_key);
}

}  // namespace egpu

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

#include <algorithm>
#include <atomic>
#include <climits>

namespace egpu {

constexpr int kTabWarps = 8;  // tables per CTA
constexpr int kTabThreads = kTabWarps * 32;
constexpr int kTabStep = 4 * 32;       // requests one warp scores per step
constexpr uint32_t kNoKey = 0x7fffffffu;  // the key of "no feasible device"

// Warp-level rank sort of one table's first dv rows by (fc, fm, d), as resort_table_cta sorts a context's table.
// sK[pos] = the packed compare word (kPadWord past the rows); sBase[pos] = fc << 24 | fm << 6 | d, and kNoKey at
// every position that is no row, including "none" (32 for DT <= 32, 64 for DT = 64).  A table outside §2.1's
// domain (dv not in [1, D], or a row value out of range) gets no rows; dv is not read past D.  COHERENT: the table
// may have been written earlier in the same launch by another CTA, so it is read from L2.  Returns the rows.
template <int DT, bool COHERENT>
__device__ __forceinline__ int sort_table_warp(const int32_t* fc_row, const int32_t* fm_row, int dv, int D, uint32_t* sK,
                                               uint32_t* sBase, uint32_t* sRank) {
    const int lane = threadIdx.x & 31;
    bool ok = dv >= 1 && dv <= D;
    for (int j = lane; j < DT; j += 32) {
        uint32_t rank = 0xffffffffu;
        if (ok && j < dv) {
            const int32_t c = COHERENT ? __ldcg(fc_row + j) : fc_row[j], m = COHERENT ? __ldcg(fm_row + j) : fm_row[j];
            if (c < 0 || c > kCoreMax || m < 0 || m > kMemMax) ok = false;
            rank = (static_cast<uint32_t>(c) << 24) | (static_cast<uint32_t>(m) << 6) | static_cast<uint32_t>(j);
        }
        sRank[j] = rank;
        sK[j] = kPadWord;
    }
    for (int j = lane; j <= kMaxD; j += 32) sBase[j] = kNoKey;
    const int rows = __all_sync(0xffffffffu, ok) ? dv : 0;
    __syncwarp();
    for (int j = lane; j < rows; j += 32) {
        const uint32_t mine = sRank[j];
        int pos = 0;
        for (int k = 0; k < rows; ++k) pos += sRank[k] < mine;
        sK[pos] = pack_table_word(static_cast<int32_t>(mine >> 24), static_cast<int32_t>((mine >> 6) & 0x3FFFFu)) |
                  (static_cast<uint32_t>(pos) & 31u);
        sBase[pos] = mine;
    }
    __syncwarp();
    return rows;
}

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
    sort_table_warp<DT, false>(free_core + static_cast<size_t>(n) * D, free_mem + static_cast<size_t>(n) * D, d_valid[n], D,
                               sK[warp], sBase[warp], sRank[warp]);
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

// ---- egpu::place_tables (DESIGN.md §2.11, §4.6): best-fit rounds to the fixed point over N tables ---------------
//
// One cooperative launch of resident CTAs (256 threads, 8 warps, a warp per table as above) runs every round.
// A round is three phases separated by grid barriers:
//   1. choose: work items are (row chunk of kPlaceChunk pending rows, tile of 8 tables), cut into contiguous
//      ranges per CTA.  Each warp sorts its table from the current free_*_out and scores the chunk; the CTA
//      keeps each row's best word over its warps and over every tile it scores for that chunk in registers,
//      then does one atomicMax per row (the words are stored inverted, so 0 is "no choice yet");
//   2. commit: the CTA of a table tile streams the pending rows' words in row order, once, for its 8 warps (up to
//      kPlaceStage rows are staged in shared memory once per round for every tile the CTA takes); the warp of
//      table n walks the rows that chose n and commits each row while the running demand of the rows that chose
//      its device fits (§2.5 per device; rows of one 32-row step that share a device are summed in order with
//      __match_any_sync), then writes its table's new values;
//   3. compact: deferred rows go, in row order, into the other pending set (per-tile counts from phase 2,
//      exclusive offsets summed by every CTA), and their words are reset; rows that chose nothing become -1.
// Round 1 reads the caller's tables and requests directly and copies every table to free_*_out.  Everything a
// phase reads that another CTA wrote in this launch is read from L2 (__ldcg).
constexpr int kPlaceChunk = 1024;           // pending rows per choose work item
constexpr int kPlaceBlock = kTabThreads;    // rows per compaction tile
constexpr int kPlaceStage = kTabWarps * kPlaceBlock;  // pending rows the commit phase stages at once
constexpr int kPlaceDevices = 64;           // CUDA devices whose occupancy answer is cached

struct PlaceCtl {
    RoundsCtl bar;                // grid-barrier words
    unsigned long long timeouts;  // grid_barrier's count of waits that gave up (info[1] says whether one did)
    unsigned int in_domain;       // some request is in the domain
    unsigned int pad_[3];
};

struct PlaceArgs {
    const int32_t* fc;               // the caller's tables [N][D], d_valid [N] and requests [P]
    const int32_t* fm;
    const int32_t* dv;
    const int32_t* rc;
    const int32_t* rm;
    int N, D;
    long long P;
    int32_t* node;                   // outputs: placement [P], tables after every commit [N][D], info [2]
    int8_t* dev;
    int32_t* fc_out;
    int32_t* fm_out;
    int32_t* info;
    unsigned long long* best;        // [P]: each pending row's choice, inverted (0 = none yet)
    int32_t* set[2];                 // [P] each: the pending rows of a round, in row order
    unsigned int* count[2];          // [P / 256] each, by round parity: deferred rows per compaction tile
    PlaceCtl* ctl;
    uint32_t gx, gm;                 // kGuards, kCandMask (in registers: see DevState::cand_xor)
};

// The compaction's offsets, summed by the whole CTA from the per-tile deferred counts (read from L2: every CTA's
// commit wrote them): `before`, the rows deferred in the tiles before `lo`, and `total`, those of all `tiles`.
__device__ __forceinline__ void deferred_prefix(const unsigned int* count, long long tiles, long long lo,
                                                unsigned int& before, unsigned int& total,
                                                unsigned int (*red)[kTabWarps]) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    before = 0;
    total = 0;
    for (long long t = tid; t < tiles; t += kTabThreads) {
        const unsigned int c = __ldcg(count + t);
        total += c;
        before += t < lo ? c : 0u;
    }
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        before += __shfl_xor_sync(0xffffffffu, before, o);
        total += __shfl_xor_sync(0xffffffffu, total, o);
    }
    if (lane == 0) {
        red[0][warp] = before;
        red[1][warp] = total;
    }
    __syncthreads();
    before = 0;
    total = 0;
#pragma unroll
    for (int w = 0; w < kTabWarps; ++w) {
        before += red[0][w];
        total += red[1][w];
    }
    __syncthreads();
}

// One compaction tile, every thread of the CTA with its row: the rows that defer go to next[before ...] in row order,
// and `before` moves past them.
__device__ __forceinline__ void append_deferred(bool defer, int32_t row, int32_t* next, unsigned int& before,
                                                unsigned int* red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const unsigned int bal = __ballot_sync(0xffffffffu, defer);
    if (lane == 0) red[warp] = __popc(bal);
    __syncthreads();
    unsigned int at = before, in_tile = 0;
#pragma unroll
    for (int w = 0; w < kTabWarps; ++w) {
        at += w < warp ? red[w] : 0u;
        in_tile += red[w];
    }
    if (defer) next[at + __popc(bal & ((1u << lane) - 1u))] = row;
    before += in_tile;
    __syncthreads();
}

template <int DT, bool VEC>
__global__ void __launch_bounds__(kTabThreads, 2)
place_tables_kernel(const __grid_constant__ PlaceArgs a) {
    __shared__ __align__(16) uint32_t sK[kTabWarps][DT];
    __shared__ uint32_t sBase[kTabWarps][kMaxD + 1];
    __shared__ uint32_t sRank[kTabWarps][kMaxD];
    __shared__ unsigned long long sW[kTabWarps][kPlaceBlock];  // choose: each warp's (inverted) words for a block of rows
    __shared__ int32_t sFc[kTabWarps][kMaxD], sFm[kTabWarps][kMaxD];    // commit: the table as the round found it
    __shared__ int32_t sAccC[kTabWarps][kMaxD], sAccM[kTabWarps][kMaxD];  // ... demand committed per device
    __shared__ int32_t sClosed[kTabWarps][kMaxD];                          // ... a row did not fit: later rows cannot
    __shared__ int32_t sRow[kPlaceStage];  // commit: the staged rows (their words are staged in sW)
    __shared__ unsigned int sRed[2][kTabWarps];
    __shared__ int sOk;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int b = blockIdx.x, G = gridDim.x;
    const int N = a.N, D = a.D, T = (N + kTabWarps - 1) / kTabWarps;
    unsigned int gen = 0;

    // every row undecided; note whether any row is in the domain (info[0] counts rounds only then)
    bool in_domain = false;
    for (long long p = static_cast<long long>(b) * kTabThreads + tid; p < a.P; p += static_cast<long long>(G) * kTabThreads) {
        const int32_t c = __ldg(a.rc + p), m = __ldg(a.rm + p);
        in_domain |= c >= 0 && c <= kCoreMax && m >= 0 && m <= kMemMax;
        a.node[p] = -2;
        a.dev[p] = -2;
    }
    if (__syncthreads_or(in_domain) && tid == 0) a.ctl->in_domain = 1u;

    const int32_t* cur = nullptr;  // pending rows in row order; round 1: every row (position = row)
    long long n = a.P;
    int which = 0, round = 0;
    bool done = false;
    while (!done) {
        ++round;
        const int32_t* tab_c = round == 1 ? a.fc : a.fc_out;
        const int32_t* tab_m = round == 1 ? a.fm : a.fm_out;

        // ---- 1. choose
        {
            const long long chunks = (n + kPlaceChunk - 1) / kPlaceChunk, items = chunks * T;
            const long long lo = items * b / G, hi = items * (b + 1) / G;
            unsigned long long mine[kPlaceChunk / kPlaceBlock];
            long long held = -1;  // the chunk `mine` belongs to
            for (long long it = lo; it <= hi; ++it) {
                const long long chunk = it < hi ? it / T : -1;
                if (held >= 0 && chunk != held) {  // the CTA's last tile of a chunk: one atomic per row
#pragma unroll
                    for (int s = 0; s < kPlaceChunk / kPlaceBlock; ++s) {
                        const long long i = held * kPlaceChunk + s * kPlaceBlock + tid;
                        if (i < n && mine[s]) atomicMax(a.best + (cur ? __ldcg(cur + i) : i), mine[s]);
                    }
                }
                if (it == hi) break;
                if (chunk != held) {
                    held = chunk;
#pragma unroll
                    for (int s = 0; s < kPlaceChunk / kPlaceBlock; ++s) mine[s] = 0;
                }
                const int tile = static_cast<int>(it - chunk * T);
                const int tn = tile * kTabWarps + warp;
                const size_t off = static_cast<size_t>(tn) * D;
                sort_table_warp<DT, true>(tab_c + off, tab_m + off, tn < N ? __ldg(a.dv + tn) : 0, D, sK[warp], sBase[warp],
                                          sRank[warp]);
                if (round == 1 && chunk == 0 && tn < N)
                    for (int j = lane; j < D; j += 32) {
                        a.fc_out[off + j] = a.fc[off + j];
                        a.fm_out[off + j] = a.fm[off + j];
                    }
                uint32_t K[DT];
#pragma unroll
                for (int j = 0; j < DT; j += 4) {
                    const uint4 k4 = *reinterpret_cast<const uint4*>(&sK[warp][j]);
                    K[j] = k4.x; K[j + 1] = k4.y; K[j + 2] = k4.z; K[j + 3] = k4.w;
                }
                const uint32_t* base_of = sBase[warp];
                // ~((lc << 18 | lm) << 38 | n << 6 | d): the unsigned order of the word is (lc, lm, n, d)
                auto choose = [&](int32_t core, int32_t mem) -> unsigned long long {
                    const uint32_t base = base_of[first_feasible<DT>(K, pack_request_word(core, mem), a.gx, a.gm)];
                    if (base == kNoKey) return 0ull;
                    const uint32_t key = base - ((static_cast<uint32_t>(core) << 24) | (static_cast<uint32_t>(mem) << 6));
                    return ~((static_cast<unsigned long long>(key >> 6) << 38) | (static_cast<unsigned long long>(tn) << 6) |
                             (key & 63u));
                };
#pragma unroll
                for (int s = 0; s < kPlaceChunk / kPlaceBlock; ++s) {
                    const long long i0 = chunk * kPlaceChunk + s * kPlaceBlock;
                    if (i0 >= n) break;
                    if (VEC && round == 1) {  // P % 4 == 0 and 16-byte aligned requests: 4 consecutive rows per lane
#pragma unroll
                        for (int h = 0; h < kPlaceBlock / 128; ++h) {
                            const int j = h * 128 + 4 * lane;
                            unsigned long long w0 = 0, w1 = 0, w2 = 0, w3 = 0;
                            if (i0 + j < n) {
                                const int4 c = __ldg(reinterpret_cast<const int4*>(a.rc + i0 + j));
                                const int4 m = __ldg(reinterpret_cast<const int4*>(a.rm + i0 + j));
                                w0 = choose(c.x, m.x); w1 = choose(c.y, m.y); w2 = choose(c.z, m.z); w3 = choose(c.w, m.w);
                            }
                            sW[warp][j] = w0; sW[warp][j + 1] = w1; sW[warp][j + 2] = w2; sW[warp][j + 3] = w3;
                        }
                    } else {
#pragma unroll 4
                        for (int j = lane; j < kPlaceBlock; j += 32) {
                            const long long i = i0 + j;
                            unsigned long long w = 0;
                            if (i < n) {
                                const long long row = cur ? __ldcg(cur + i) : i;
                                w = choose(__ldg(a.rc + row), __ldg(a.rm + row));
                            }
                            sW[warp][j] = w;
                        }
                    }
                    __syncthreads();
                    unsigned long long m = sW[0][tid];
#pragma unroll
                    for (int w = 1; w < kTabWarps; ++w) m = max(m, sW[w][tid]);
                    mine[s] = max(mine[s], m);
                    __syncthreads();
                }
            }
        }
        if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) break;

        // ---- 2. commit
        unsigned int* const count = a.count[(round - 1) & 1];
        unsigned long long* const sStage = &sW[0][0];  // kPlaceStage words: the choose phase is over
        long long staged = -1;                         // the first pending row staged in sStage / sRow
        for (int tile = static_cast<int>(b); tile < T; tile += static_cast<int>(G)) {
            const int tn = tile * kTabWarps + warp;
            const int dv = tn < N ? __ldg(a.dv + tn) : 0;
            const bool live = dv >= 1 && dv <= D;  // a table outside the domain is never chosen: it keeps its copy
            const size_t off = static_cast<size_t>(tn) * D;
            for (int j = lane; j < kMaxD; j += 32) {
                sAccC[warp][j] = 0;
                sAccM[warp][j] = 0;
                sClosed[warp][j] = 0;
                if (live && j < dv) {
                    sFc[warp][j] = __ldcg(tab_c + off + j);
                    sFm[warp][j] = __ldcg(tab_m + off + j);
                }
            }
            __syncwarp();
            bool dirty = false;
            for (long long i0 = 0; i0 < n; i0 += kPlaceStage) {
                if (i0 != staged) {  // at most kPlaceStage pending rows are staged once per round for every tile
                    __syncthreads();  // every warp is done with the rows staged before
#pragma unroll
                    for (int k = tid; k < kPlaceStage; k += kTabThreads) {
                        const long long i = i0 + k;
                        unsigned long long w = ~0ull;  // names no table
                        if (i < n) {
                            const int32_t row = cur ? __ldcg(cur + i) : static_cast<int32_t>(i);
                            sRow[k] = row;
                            w = ~__ldcg(a.best + row);
                        }
                        sStage[k] = w;
                    }
                    __syncthreads();
                    staged = i0;
                }
                if (!live) continue;
                const int len = static_cast<int>(min(static_cast<long long>(kPlaceStage), n - i0));
                for (int j0 = 0; j0 < len; j0 += kPlaceBlock) {  // one compaction tile
                    unsigned int deferred = 0;
                    for (int j = j0 + lane; j < j0 + kPlaceBlock; j += 32) {
                        const unsigned long long w = sStage[j];
                        const bool matched = static_cast<int>((w >> 6) & 0x7fffffffu) == tn;
                        const unsigned int mb = __ballot_sync(0xffffffffu, matched);
                        if (mb == 0u) continue;
                        const int d = static_cast<int>(w & 63u);
                        const int32_t row = sRow[j];
                        const int32_t core = matched ? __ldg(a.rc + row) : 0, mem = matched ? __ldg(a.rm + row) : 0;
                        // in-order demand of the rows of this step that chose the same device, up to and including this one
                        const unsigned int peers = __match_any_sync(0xffffffffu, matched ? d : kMaxD);
                        int32_t pc = 0, pm = 0;
                        for (unsigned int r = mb; r; r &= r - 1u) {
                            const int src = __ffs(r) - 1;
                            const int32_t vc = __shfl_sync(0xffffffffu, core, src), vm = __shfl_sync(0xffffffffu, mem, src);
                            if (((peers >> src) & 1u) && src <= lane) {
                                pc += vc;
                                pm += vm;
                            }
                        }
                        int32_t acc_c = 0, acc_m = 0;
                        bool fits = false;
                        if (matched) {
                            acc_c = sAccC[warp][d] + pc;
                            acc_m = sAccM[warp][d] + pm;
                            fits = !sClosed[warp][d] && acc_c <= sFc[warp][d] && acc_m <= sFm[warp][d];
                        }
                        const unsigned int fb = __ballot_sync(0xffffffffu, fits);
                        __syncwarp();
                        if (fits) {
                            a.node[row] = tn;
                            a.dev[row] = static_cast<int8_t>(d);
                            if (lane == 31 - __clz(peers & fb)) {  // the last row of the device that fits
                                sAccC[warp][d] = acc_c;
                                sAccM[warp][d] = acc_m;
                            }
                        } else if (matched && lane == 31 - __clz(peers & ~fb)) {
                            sClosed[warp][d] = 1;  // demand only grows: every later row of this device is deferred
                        }
                        __syncwarp();
                        dirty |= fb != 0u;
                        deferred += __popc(mb & ~fb);
                    }
                    if (lane == 0 && deferred) atomicAdd(count + (i0 + j0) / kPlaceBlock, deferred);
                }
            }
            __syncwarp();
            if (dirty)
                for (int j = lane; j < dv; j += 32) {
                    a.fc_out[off + j] = sFc[warp][j] - sAccC[warp][j];
                    a.fm_out[off + j] = sFm[warp][j] - sAccM[warp][j];
                }
        }
        if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) break;

        // ---- 3. compact
        {
            const long long tiles = (n + kPlaceBlock - 1) / kPlaceBlock;
            unsigned int* const next_count = a.count[round & 1];  // last read in the previous round's phase 3
            for (long long t = static_cast<long long>(b) * kTabThreads + tid; t < tiles; t += static_cast<long long>(G) * kTabThreads)
                next_count[t] = 0u;
            const long long lo = tiles * b / G, hi = tiles * (b + 1) / G;
            unsigned int before, total;
            deferred_prefix(count, tiles, lo, before, total, sRed);
            int32_t* const next = a.set[which];
            for (long long t = lo; t < hi; ++t) {
                const long long i = t * kPlaceBlock + tid;
                bool defer = false;
                int32_t row = 0;
                if (i < n) {
                    row = cur ? __ldcg(cur + i) : static_cast<int32_t>(i);
                    if (__ldcg(a.best + row) == 0ull) {
                        a.node[row] = -1;
                        a.dev[row] = -1;
                    } else if (__ldcg(a.node + row) == -2) {
                        defer = true;
                        a.best[row] = 0ull;
                    }
                }
                append_deferred(defer, row, next, before, sRed[0]);
            }
            if (total == 0u) {
                done = true;
            } else {
                cur = next;
                n = total;
                which ^= 1;
            }
        }
        if (!done && !grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) break;
    }
    if (b == 0 && tid == 0) {
        a.info[0] = *reinterpret_cast<volatile unsigned int*>(&a.ctl->in_domain) ? round : 0;
        a.info[1] = done ? 0 : 1;
    }
}

// The cooperative launch of every round kernel: one resident wave of kTabThreads-thread CTAs on `device`, at most
// `cap` of them (the caller's count of work items: the barriers cost per CTA) and at least one.  The resident CTAs
// per SM are asked once per kernel and device: each instantiation has its own cache.
template <auto kernel, class Args>
cudaError_t coop_launch(const Args& a, long long cap, int device, cudaStream_t stream) {
    static std::atomic<int> per_sm_cache[kPlaceDevices];
    int per_sm = device >= 0 && device < kPlaceDevices ? per_sm_cache[device].load(std::memory_order_relaxed) : 0;
    if (per_sm == 0) {
        cudaError_t err = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, kTabThreads, 0);
        if (err != cudaSuccess) return err;
        if (per_sm < 1) return cudaErrorCooperativeLaunchTooLarge;
        if (device >= 0 && device < kPlaceDevices) per_sm_cache[device].store(per_sm, std::memory_order_relaxed);
    }
    int sms = 0;
    cudaError_t err = cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device);
    if (err != cudaSuccess) return err;
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(static_cast<unsigned>(std::max(1ll, std::min(static_cast<long long>(sms) * per_sm, cap))));
    cfg.blockDim = dim3(kTabThreads);
    cfg.dynamicSmemBytes = 0;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeCooperative;
    attr[0].val.cooperative = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, kernel, a);
}

template <int DT>
cudaError_t place_bucket(bool vec, int device, cudaStream_t stream, const PlaceArgs& a) {
    // Grid: no more CTAs than round 1 has work items of any phase.
    const long long tiles = (a.N + kTabWarps - 1) / kTabWarps;
    const long long items = tiles * ((a.P + kPlaceChunk - 1) / kPlaceChunk);
    const long long blocks = (a.P + kPlaceBlock - 1) / kPlaceBlock;
    return vec ? coop_launch<place_tables_kernel<DT, true>>(a, std::max(items, blocks), device, stream)
               : coop_launch<place_tables_kernel<DT, false>>(a, std::max(items, blocks), device, stream);
}

// place_tables' scratch, byte offsets: best uint64[P] | barrier words | deferred counts 2 x uint32[P / 256] |
// (16-aligned) two pending sets int32[P]; everything before the pending sets (`zeroed` bytes) starts at zero.
struct PlaceScratch {
    size_t blocks, ctl, count, zeroed, set, total;
    explicit PlaceScratch(int P) {
        blocks = (static_cast<size_t>(P) + kPlaceBlock - 1) / kPlaceBlock;
        ctl = 8 * static_cast<size_t>(P);
        count = ctl + sizeof(PlaceCtl);
        zeroed = count + 2 * 4 * blocks;
        set = (zeroed + 15) & ~size_t(15);
        total = set + 2 * 4 * static_cast<size_t>(P);
    }
};

size_t place_scratch_bytes(int P) { return PlaceScratch(P).total; }

cudaError_t place_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                         const int32_t* req_core, const int32_t* req_mem, int P, int32_t* out_node, int8_t* out_dev,
                         int32_t* free_core_out, int32_t* free_mem_out, int32_t* info, void* scratch, int device,
                         cudaStream_t stream) {
    const PlaceScratch L(P);
    char* s = static_cast<char*>(scratch);
    PlaceArgs a{};
    a.fc = free_core; a.fm = free_mem; a.dv = d_valid; a.rc = req_core; a.rm = req_mem;
    a.N = N; a.D = D; a.P = P;
    a.node = out_node; a.dev = out_dev; a.fc_out = free_core_out; a.fm_out = free_mem_out; a.info = info;
    a.best = reinterpret_cast<unsigned long long*>(s);
    a.ctl = reinterpret_cast<PlaceCtl*>(s + L.ctl);
    a.count[0] = reinterpret_cast<unsigned int*>(s + L.count);
    a.count[1] = a.count[0] + L.blocks;
    a.set[0] = reinterpret_cast<int32_t*>(s + L.set);
    a.set[1] = a.set[0] + P;
    a.gx = kGuards;
    a.gm = kCandMask;
    cudaError_t err = cudaMemsetAsync(scratch, 0, L.zeroed, stream);
    if (err != cudaSuccess) return err;
    const bool vec = (P % 4) == 0 && (reinterpret_cast<uintptr_t>(req_core) % 16) == 0 &&
                     (reinterpret_cast<uintptr_t>(req_mem) % 16) == 0;
    if (D <= 8) return place_bucket<8>(vec, device, stream, a);
    if (D <= 16) return place_bucket<16>(vec, device, stream, a);
    if (D <= 32) return place_bucket<32>(vec, device, stream, a);
    return place_bucket<64>(vec, device, stream, a);
}

// ---- egpu::place_pods (DESIGN.md §2.12, §4.7): whole pods, best-fit rounds to the fixed point over N tables -------
//
// One cooperative launch, the round structure of place_tables_kernel with a pod in place of a row:
//   0. the grid checks pod_offsets (first 0, last P, every step in [1, kMaxPod]) before any container is read
//      through them and copies the tables to free_*_out (every round reads them there); if an offset is bad
//      nothing is placed and info[2] = 1;
//   1. choose (pods_choose): work items are (block of 256 pending pods, tile of 8 tables).  A warp stages its table's
//      valid devices in shared memory and each lane replays one pod on it (pod_replay); the CTA keeps each pod's
//      best word over warps and tiles and does one atomicMax per pod (words inverted, 0 = no node yet);
//   2. commit (pods_commit): the warp of table n walks the pending pods that chose n in pod order.  The lanes replay
//      their pods again against the round's table to recover the containers' devices, then, one pod after another,
//      a pod commits when none of its devices is closed and the demand committed so far on each of them, plus its
//      own, fits; otherwise it closes all of them;
//   3. compact (deferred_prefix, pods_compact): deferred pods go, in pod order, into the other pending set; pods that
//      chose nothing become -1.
// The pods' devices are not kept between phases: the replay is deterministic, so commit recomputes them.
constexpr int kMaxPod = 8;                 // containers per pod
constexpr int kPodBlock = kTabThreads;     // pods per choose work item and per compaction tile
constexpr int kPodStage = kTabWarps * kPodBlock;  // pending pods the commit phase stages at once

struct PodsCtl {
    RoundsCtl bar;                // grid-barrier words
    unsigned long long timeouts;  // grid_barrier's count of waits that gave up (info[1] says whether one did)
    unsigned int in_domain;       // some pod is in the domain (place_pods)
    unsigned int bad_index;       // an index tensor failed the check (info[2])
    unsigned int pad_[2];
};

struct PodsArgs {
    const int32_t* fc;               // the caller's tables [N][D], d_valid [N], containers [P], pod_offsets [G + 1]
    const int32_t* fm;
    const int32_t* dv;
    const int32_t* rc;
    const int32_t* rm;
    const int32_t* off;
    int N, D;
    long long P, G;
    int32_t* node;                   // outputs: node per pod [G], device per container [P], tables [N][D], info [3]
    int8_t* dev;
    int32_t* fc_out;
    int32_t* fm_out;
    int32_t* info;
    unsigned long long* best;        // [G]: each pending pod's choice, inverted (0 = none yet)
    int32_t* set[2];                 // [G] each: the pending pods of a round, in pod order
    unsigned int* count[2];          // [G / 256] each, by round parity: deferred pods per compaction tile
    PodsCtl* ctl;
};

// What a pod's in-node replay leaves: the devices its containers touched (at most one per container), with the
// free values the pod left on them, and each container's device in 6 bits.
struct PodFit {
    int nt;                  // devices touched
    int td[kMaxPod];         // ... their indices
    int32_t tc[kMaxPod];     // ... free core and memory after the pod
    int32_t tm[kMaxPod];
    unsigned long long cdev; // container k's device in bits 6k .. 6k + 5
    uint32_t slc, slm;       // sums of the containers' leftovers at the moment each was placed
};

// §2.12's in-node replay: containers [c0, c0 + len) placed one after another on a table whose first `rows`
// devices are sc / sm (shared memory), each by §2.3's best fit, the smallest (lc, lm, d), against what the earlier
// containers left.  Untouched devices are read at the table's values; the touched ones are kept in registers (the
// slots are indexed by compile-time constants only).  Returns false when a container is outside §2.1's domain or
// finds no device.
__device__ __forceinline__ bool pod_replay(const int32_t* sc, const int32_t* sm, int rows, const int32_t* __restrict__ rc,
                                           const int32_t* __restrict__ rm, long long c0, int len, PodFit& f) {
    f.nt = 0;
    f.cdev = 0;
    f.slc = 0;
    f.slm = 0;
    unsigned long long touched = 0;
#pragma unroll
    for (int s = 0; s < kMaxPod; ++s) {
        f.td[s] = 0;
        f.tc[s] = 0;
        f.tm[s] = 0;
    }
    for (int k = 0; k < len; ++k) {
        const int32_t core = __ldg(rc + c0 + k), mem = __ldg(rm + c0 + k);
        if (core < 0 || core > kCoreMax || mem < 0 || mem > kMemMax) return false;
        uint32_t key = kNoKey;  // (lc << 24 | lm << 6 | d): its unsigned order is best fit's
#pragma unroll 4
        for (int d = 0; d < rows; ++d) {
            if ((touched >> d) & 1ull) continue;
            const int32_t lc = sc[d] - core, lm = sm[d] - mem;
            if ((lc | lm) >= 0)
                key = min(key, (static_cast<uint32_t>(lc) << 24) | (static_cast<uint32_t>(lm) << 6) | static_cast<uint32_t>(d));
        }
#pragma unroll
        for (int s = 0; s < kMaxPod; ++s) {
            const int32_t lc = f.tc[s] - core, lm = f.tm[s] - mem;
            if (s < f.nt && (lc | lm) >= 0)
                key = min(key, (static_cast<uint32_t>(lc) << 24) | (static_cast<uint32_t>(lm) << 6) |
                                   static_cast<uint32_t>(f.td[s]));
        }
        if (key == kNoKey) return false;
        const int d = static_cast<int>(key & 63u);
        f.slc += key >> 24;
        f.slm += (key >> 6) & 0x3FFFFu;
        f.cdev |= static_cast<unsigned long long>(d) << (6 * k);
        if ((touched >> d) & 1ull) {
#pragma unroll
            for (int s = 0; s < kMaxPod; ++s)
                if (s < f.nt && f.td[s] == d) {
                    f.tc[s] -= core;
                    f.tm[s] -= mem;
                }
        } else {
#pragma unroll
            for (int s = 0; s < kMaxPod; ++s)
                if (s == f.nt) {
                    f.td[s] = d;
                    f.tc[s] = sc[d] - core;
                    f.tm[s] = sm[d] - mem;
                }
            ++f.nt;
            touched |= 1ull << d;
        }
    }
    return true;
}

// Stages table tn's first D devices into sc / sm (the warp's rows of shared memory) and returns the number of
// devices it offers: d_valid, or 0 for a table outside §2.1's domain or past N.  COHERENT: read from L2.
__device__ __forceinline__ int stage_table_warp(const int32_t* fc_row, const int32_t* fm_row, int dv, int D, int32_t* sc,
                                                int32_t* sm) {
    const int lane = threadIdx.x & 31;
    bool ok = dv >= 1 && dv <= D;
    for (int j = lane; ok && j < dv; j += 32) {
        const int32_t c = __ldcg(fc_row + j), m = __ldcg(fm_row + j);
        ok = c >= 0 && c <= kCoreMax && m >= 0 && m <= kMemMax;
        sc[j] = c;
        sm[j] = m;
    }
    const int rows = __all_sync(0xffffffffu, ok) ? dv : 0;
    __syncwarp();
    return rows;
}

// One position of the check of a CSR offset array off [n + 1] over `total` entries: the first offset is 0, the last
// is total, and every step off[i + 1] - off[i] is in [lo, hi].  True when position i (0 <= i <= n) fails it.
__device__ __forceinline__ bool csr_bad(const int32_t* off, long long i, long long n, long long total, long long lo,
                                        long long hi) {
    const int32_t o = __ldg(off + i);
    const bool bad = i == 0 && o != 0;
    if (i == n) return bad || o != total;
    const long long step = static_cast<long long>(__ldg(off + i + 1)) - o;
    return bad || step < lo || step > hi;
}

// The shared memory of place_pods_kernel and place_gangs_kernel, the grid barrier's word apart.
struct PodsSmem {
    unsigned long long W[kTabWarps][kPodBlock];  // choose: each warp's (inverted) words for a block of pods
    int32_t Fc[kTabWarps][kMaxD], Fm[kTabWarps][kMaxD];      // the table as the round found it
    int32_t AccC[kTabWarps][kMaxD], AccM[kTabWarps][kMaxD];  // commit: demand committed per device
    int32_t Closed[kTabWarps][kMaxD];                        // ... a pod did not commit: later pods cannot
    int32_t Pod[kPodStage];  // commit: the staged pods (their words are staged in W)
    unsigned int Red[2][kTabWarps];
};

// The phases of place_pods_kernel and place_gangs_kernel.  The pending set of a round is positions [0, m): position i
// is pod cur[i], or pod pos0 + i when cur is null (round 1 of place_pods, pos0 = 0, and of a gang, pos0 = its first
// pod).  Every thread of the CTA calls them.

// ---- 1. choose
__device__ __forceinline__ void pods_choose(const PodsArgs& a, const int32_t* cur, long long pos0, long long m,
                                            PodsSmem& s) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int b = blockIdx.x, G = gridDim.x;
    const int N = a.N, D = a.D, T = (N + kTabWarps - 1) / kTabWarps;
    const long long blocks = (m + kPodBlock - 1) / kPodBlock, items = blocks * T;
    const long long lo = items * b / G, hi = items * (b + 1) / G;
    unsigned long long mine = 0;
    long long held = -1;  // the block of pods `mine` belongs to
    for (long long it = lo; it <= hi; ++it) {
        const long long blk = it < hi ? it / T : -1;
        if (held >= 0 && blk != held) {  // the CTA's last tile of a block: one atomic per pod
            const long long i = held * kPodBlock + tid;
            if (i < m && mine) atomicMax(a.best + (cur ? __ldcg(cur + i) : pos0 + i), mine);
            mine = 0;
        }
        if (it == hi) break;
        held = blk;
        const int tn = static_cast<int>(it - blk * T) * kTabWarps + warp;
        const size_t off = static_cast<size_t>(tn) * D;
        const int rows = stage_table_warp(a.fc_out + off, a.fm_out + off, tn < N ? __ldg(a.dv + tn) : 0, D, s.Fc[warp],
                                          s.Fm[warp]);
        for (int j = lane; j < kPodBlock; j += 32) {
            const long long i = blk * kPodBlock + j;
            unsigned long long w = 0;
            if (i < m && rows) {
                const long long g = cur ? __ldcg(cur + i) : pos0 + i;
                const int32_t c0 = __ldg(a.off + g);
                PodFit f;
                // ~(sum lc << 52 | sum lm << 31 | n): the unsigned order of the word is (sum lc, sum lm, n)
                if (pod_replay(s.Fc[warp], s.Fm[warp], rows, a.rc, a.rm, c0, __ldg(a.off + g + 1) - c0, f))
                    w = ~((static_cast<unsigned long long>(f.slc) << 52) |
                          (static_cast<unsigned long long>(f.slm) << 31) | static_cast<unsigned long long>(tn));
            }
            s.W[warp][j] = w;
        }
        __syncthreads();
#pragma unroll
        for (int w = 0; w < kTabWarps; ++w) mine = max(mine, s.W[w][tid]);
        __syncthreads();
    }
}

// ---- 2. commit: adds each compaction tile's deferred pods to count[tile]; returns the warp's committed pods.
__device__ __forceinline__ unsigned int pods_commit(const PodsArgs& a, unsigned int* count, const int32_t* cur,
                                                    long long pos0, long long m, PodsSmem& s) {
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int b = blockIdx.x, G = gridDim.x;
    const int N = a.N, D = a.D, T = (N + kTabWarps - 1) / kTabWarps;
    unsigned long long* const sStage = &s.W[0][0];  // kPodStage words: the choose phase is over
    long long staged = -1;                          // the first pending position staged in sStage / s.Pod
    unsigned int committed = 0;                     // this warp's committed pods
    for (int tile = static_cast<int>(b); tile < T; tile += static_cast<int>(G)) {
        const int tn = tile * kTabWarps + warp;
        const size_t off = static_cast<size_t>(tn) * D;
        // a table outside the domain offers no device, so no pod chose it: it keeps its copy
        const int rows = stage_table_warp(a.fc_out + off, a.fm_out + off, tn < N ? __ldg(a.dv + tn) : 0, D, s.Fc[warp],
                                          s.Fm[warp]);
        for (int j = lane; j < kMaxD; j += 32) {
            s.AccC[warp][j] = 0;
            s.AccM[warp][j] = 0;
            s.Closed[warp][j] = 0;
        }
        __syncwarp();
        bool dirty = false;
        for (long long i0 = 0; i0 < m; i0 += kPodStage) {
            if (i0 != staged) {  // at most kPodStage pending pods are staged once per round for every tile
                __syncthreads();  // every warp is done with the pods staged before
                for (int k = tid; k < kPodStage; k += kTabThreads) {
                    const long long i = i0 + k;
                    unsigned long long w = ~0ull;  // names no table
                    if (i < m) {
                        const int32_t g = cur ? __ldcg(cur + i) : static_cast<int32_t>(pos0 + i);
                        s.Pod[k] = g;
                        w = ~__ldcg(a.best + g);
                    }
                    sStage[k] = w;
                }
                __syncthreads();
                staged = i0;
            }
            if (!rows) continue;
            const int len = static_cast<int>(min(static_cast<long long>(kPodStage), m - i0));
            for (int j0 = 0; j0 < len; j0 += kPodBlock) {  // one compaction tile
                unsigned int deferred = 0;
                for (int j = j0 + lane; j < j0 + kPodBlock; j += 32) {
                    const unsigned long long w = sStage[j];
                    const bool matched = static_cast<int>(w & 0x7fffffffu) == tn;
                    const unsigned int mb = __ballot_sync(0xffffffffu, matched);
                    if (mb == 0u) continue;
                    PodFit f;
                    int32_t g = 0, c0 = 0, c1 = 0;
                    if (matched) {  // the choose phase's replay, again: it fitted then, so it fits now
                        g = s.Pod[j];
                        c0 = __ldg(a.off + g);
                        c1 = __ldg(a.off + g + 1);
                        pod_replay(s.Fc[warp], s.Fm[warp], rows, a.rc, a.rm, c0, c1 - c0, f);
                    }
                    // one pod after another, in pod order (lane order)
                    bool fits = false;
                    for (unsigned int r = mb; r; r &= r - 1u) {
                        if (lane == __ffs(r) - 1) {
                            bool ok = true;
#pragma unroll
                            for (int k = 0; k < kMaxPod; ++k)
                                if (k < f.nt) {  // committed + the pod's demand <= free  <=>  committed <= what the pod leaves
                                    const int d = f.td[k];
                                    ok &= !s.Closed[warp][d] && s.AccC[warp][d] <= f.tc[k] && s.AccM[warp][d] <= f.tm[k];
                                }
#pragma unroll
                            for (int k = 0; k < kMaxPod; ++k)
                                if (k < f.nt) {
                                    const int d = f.td[k];
                                    if (ok) {
                                        s.AccC[warp][d] += s.Fc[warp][d] - f.tc[k];
                                        s.AccM[warp][d] += s.Fm[warp][d] - f.tm[k];
                                    } else {
                                        s.Closed[warp][d] = 1;
                                    }
                                }
                            fits = ok;
                        }
                        __syncwarp();
                    }
                    if (fits) {
                        a.node[g] = tn;
                        for (int32_t c = c0; c < c1; ++c)
                            a.dev[c] = static_cast<int8_t>((f.cdev >> (6 * (c - c0))) & 63u);
                    }
                    const unsigned int fb = __ballot_sync(0xffffffffu, fits);
                    dirty |= fb != 0u;
                    committed += __popc(fb);
                    deferred += __popc(mb & ~fb);
                }
                if (lane == 0 && deferred) atomicAdd(count + (i0 + j0) / kPodBlock, deferred);
            }
        }
        __syncwarp();
        if (dirty)
            for (int j = lane; j < rows; j += 32) {
                a.fc_out[off + j] = s.Fc[warp][j] - s.AccC[warp][j];
                a.fm_out[off + j] = s.Fm[warp][j] - s.AccM[warp][j];
            }
    }
    return committed;
}

// ---- 3. compact the CTA's compaction tiles [lo, hi), `before` the deferred pods of the tiles before lo
__device__ __forceinline__ void pods_compact(const PodsArgs& a, const int32_t* cur, long long pos0, long long m,
                                             long long lo, long long hi, int32_t* next, unsigned int before,
                                             PodsSmem& s) {
    const int tid = threadIdx.x;
    for (long long t = lo; t < hi; ++t) {
        const long long i = t * kPodBlock + tid;
        bool defer = false;
        int32_t g = 0;
        if (i < m) {
            g = cur ? __ldcg(cur + i) : static_cast<int32_t>(pos0 + i);
            if (__ldcg(a.best + g) == 0ull) {
                a.node[g] = -1;
                for (int32_t c = __ldg(a.off + g), c1 = __ldg(a.off + g + 1); c < c1; ++c) a.dev[c] = -1;
            } else if (__ldcg(a.node + g) == -2) {
                defer = true;
                a.best[g] = 0ull;
            }
        }
        append_deferred(defer, g, next, before, s.Red[0]);
    }
}

__global__ void __launch_bounds__(kTabThreads, 2)
place_pods_kernel(const __grid_constant__ PodsArgs a) {
    __shared__ PodsSmem s;
    __shared__ int sOk;
    const int tid = threadIdx.x;
    const unsigned int b = blockIdx.x, G = gridDim.x;
    const int N = a.N, D = a.D;
    const long long stride = static_cast<long long>(G) * kTabThreads, first = static_cast<long long>(b) * kTabThreads + tid;
    unsigned int gen = 0;
    int round = 0;
    bool done = false;

    // ---- 0. every pod and container undecided, the tables copied; the offsets checked before a container is read
    // through them
    {
        bool bad = false;
        for (long long g = first; g <= a.G; g += stride) {
            bad |= csr_bad(a.off, g, a.G, a.P, 1, kMaxPod);
            if (g < a.G) a.node[g] = -2;
        }
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -2;
        for (long long j = first; j < static_cast<long long>(N) * D; j += stride) {
            a.fc_out[j] = a.fc[j];
            a.fm_out[j] = a.fm[j];
        }
        if (__syncthreads_or(bad) && tid == 0) atomicExch(&a.ctl->bad_index, 1u);
    }
    if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
    if (*reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index)) {  // nothing is placed
        for (long long g = first; g < a.G; g += stride) a.node[g] = -1;
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -1;
        done = true;
        goto finish;
    }
    {  // note whether any pod is in the domain (info[0] counts rounds only then)
        bool in_domain = false;
        for (long long g = first; g < a.G; g += stride) {
            const int32_t c0 = __ldg(a.off + g), c1 = __ldg(a.off + g + 1);
            bool ok = true;
            for (int32_t c = c0; c < c1; ++c) {
                const int32_t core = __ldg(a.rc + c), mem = __ldg(a.rm + c);
                ok &= core >= 0 && core <= kCoreMax && mem >= 0 && mem <= kMemMax;
            }
            in_domain |= ok;
        }
        if (__syncthreads_or(in_domain) && tid == 0) a.ctl->in_domain = 1u;
    }

    {
        const int32_t* cur = nullptr;  // pending pods in pod order; round 1: every pod (position = pod)
        long long n = a.G;
        int which = 0;
        while (!done) {
            ++round;
            pods_choose(a, cur, 0, n, s);
            if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) break;
            unsigned int* const count = a.count[(round - 1) & 1];
            pods_commit(a, count, cur, 0, n, s);
            if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) break;

            // ---- 3. compact
            {
                const long long tiles = (n + kPodBlock - 1) / kPodBlock;
                unsigned int* const next_count = a.count[round & 1];  // last read in the previous round's phase 3
                for (long long t = first; t < tiles; t += stride) next_count[t] = 0u;
                const long long lo = tiles * b / G, hi = tiles * (b + 1) / G;
                unsigned int before, total;
                deferred_prefix(count, tiles, lo, before, total, s.Red);
                pods_compact(a, cur, 0, n, lo, hi, a.set[which], before, s);
                if (total == 0u) {
                    done = true;
                } else {
                    cur = a.set[which];
                    n = total;
                    which ^= 1;
                }
            }
            if (!done && !grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) break;
        }
    }
finish:
    if (b == 0 && tid == 0) {
        const bool bad = *reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index) != 0u;
        a.info[0] = !bad && *reinterpret_cast<volatile unsigned int*>(&a.ctl->in_domain) ? round : 0;
        a.info[1] = done ? 0 : 1;
        a.info[2] = bad ? 1 : 0;
    }
}

// place_pods' and place_gangs' scratch (place_pods: J = 0), byte offsets: best uint64[G] | barrier words | deferred
// counts 2 x uint32[G / 256] | pods in the domain uint32[J] | committed pods uint32[J] | (16-aligned) two pending
// sets int32[G]; everything before the pending sets (`zeroed` bytes) starts at zero.
struct PodsScratch {
    size_t blocks, ctl, count, in_domain, committed, zeroed, set, total;
    PodsScratch(int G, int J) {
        blocks = (static_cast<size_t>(G) + kPodBlock - 1) / kPodBlock;
        ctl = 8 * static_cast<size_t>(G);
        count = ctl + sizeof(PodsCtl);
        in_domain = count + 2 * 4 * blocks;
        committed = in_domain + 4 * static_cast<size_t>(J);
        zeroed = committed + 4 * static_cast<size_t>(J);
        set = (zeroed + 15) & ~size_t(15);
        total = set + 2 * 4 * static_cast<size_t>(G);
    }
};

// Points a's scratch arrays into `scratch` as L lays them out (a.G set) and zeroes its head on `stream`.
static cudaError_t pods_scratch(PodsArgs& a, void* scratch, const PodsScratch& L, cudaStream_t stream) {
    char* s = static_cast<char*>(scratch);
    a.best = reinterpret_cast<unsigned long long*>(s);
    a.ctl = reinterpret_cast<PodsCtl*>(s + L.ctl);
    a.count[0] = reinterpret_cast<unsigned int*>(s + L.count);
    a.count[1] = a.count[0] + L.blocks;
    a.set[0] = reinterpret_cast<int32_t*>(s + L.set);
    a.set[1] = a.set[0] + a.G;
    return cudaMemsetAsync(scratch, 0, L.zeroed, stream);
}

size_t pods_scratch_bytes(int G) { return PodsScratch(G, 0).total; }

cudaError_t pods_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                        const int32_t* req_core, const int32_t* req_mem, int P, const int32_t* pod_offsets, int G,
                        int32_t* out_node, int8_t* out_dev, int32_t* free_core_out, int32_t* free_mem_out, int32_t* info,
                        void* scratch, int device, cudaStream_t stream) {
    const PodsScratch L(G, 0);
    PodsArgs a{};
    a.fc = free_core; a.fm = free_mem; a.dv = d_valid; a.rc = req_core; a.rm = req_mem; a.off = pod_offsets;
    a.N = N; a.D = D; a.P = P; a.G = G;
    a.node = out_node; a.dev = out_dev; a.fc_out = free_core_out; a.fm_out = free_mem_out; a.info = info;
    const cudaError_t err = pods_scratch(a, scratch, L, stream);
    if (err != cudaSuccess) return err;
    // Grid: no more CTAs than round 1 has choose work items; at least one, which finds G = 0's offsets bad.
    const long long tiles = (static_cast<long long>(N) + kTabWarps - 1) / kTabWarps;
    return coop_launch<place_pods_kernel>(a, tiles * static_cast<long long>(L.blocks), device, stream);
}

// ---- egpu::place_gangs (DESIGN.md §2.13, §4.8): gangs of pods, each kept or given back, in order, in one launch ---
//
// One cooperative launch with an outer loop over gangs; inside it, place_pods_kernel's rounds over the current gang's
// pending pods only:
//   0. the grid checks pod_offsets, gang_offsets and gang_min, marks every pod and container -2, every gang's placed
//      count 0, and copies the tables to free_*_out (every round reads them there).  After a barrier: if an index is
//      bad nothing is placed and info[2] = 1; otherwise each pod in the domain is counted into its gang
//      (count_into_gang), and a second barrier follows;
//   per gang j, while it has pending pods and placed + pending >= gang_min[j] (round 1's pending pods are the gang's
//   pods in the domain, its contiguous range holds them):
//   1. choose and 2. commit as §4.7 (pods_choose, pods_commit); the commit also counts the gang's committed pods;
//   3. compact: every CTA first reads the round's committed and deferred counts.  If nothing is deferred, or
//      committed + deferred < gang_min, the gang ends with this round.  A gang that ends with fewer than gang_min pods
//      committed is rolled back instead of compacted (give_back_pods): its committed containers' demand goes back to
//      free_*_out by integer atomics and all its pods become -1; one barrier follows before the next gang's choose
//      reads the tables.  A kept gang ends without a barrier: the next gang's choose reads nothing this phase writes.
// Deferred counts are indexed by the launch's round number over all gangs, so their zeroing follows §4.7's parity.
struct GangsArgs {
    PodsArgs p;                      // tables, containers, pod_offsets, the outputs node, dev, tables and info, and the
                                     // scratch best, set, count, ctl (p.ctl->in_domain unused)
    const int32_t* goff;             // gang_offsets [J + 1], gang_min [J]
    const int32_t* gmin;
    long long J;
    int32_t* placed;                 // output: placed pods per gang [J]
    unsigned int* in_domain;         // [J]: each gang's pods in the domain
    unsigned int* committed;         // [J]: each gang's committed pods
};

// Counts pod g, when ok, into in_domain[j] of its gang j, the last gang whose first pod is at or before g (a binary
// search of gang_offsets [J + 1]).  Every lane of the warp calls it.
__device__ __forceinline__ void count_into_gang(const int32_t* goff, long long J, long long g, bool ok,
                                                unsigned int* in_domain) {
    long long j = 0;
    if (ok) {
        long long lo = 0, hi = J - 1;
        while (lo < hi) {
            const long long mid = (lo + hi + 1) >> 1;
            if (__ldg(goff + mid) <= g) lo = mid;
            else hi = mid - 1;
        }
        j = lo;
    }
    // the pods of a warp are consecutive, so most share a gang: one atomic per gang and warp
    const unsigned int peers = __match_any_sync(0xffffffffu, ok ? j : -1ll);
    if (ok && (threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(in_domain + j, static_cast<unsigned int>(__popc(peers)));
}

// Gives the pods [g_lo, g_hi) back, grid-stride from `first`: a placed pod's containers' demand returns to free_*_out
// by integer atomics (the tables hold other pods' commits too), and every pod and container becomes -1.
template <class Args>
__device__ __forceinline__ void give_back_pods(const Args& a, long long g_lo, long long g_hi, long long first,
                                               long long stride) {
    for (long long g = g_lo + first; g < g_hi; g += stride) {
        const int32_t nd = __ldcg(a.node + g);
        for (int32_t c = __ldg(a.off + g), c1 = __ldg(a.off + g + 1); c < c1; ++c) {
            if (nd >= 0) {
                const size_t at = static_cast<size_t>(nd) * a.D + __ldcg(a.dev + c);
                atomicAdd(a.fc_out + at, __ldg(a.rc + c));
                atomicAdd(a.fm_out + at, __ldg(a.rm + c));
            }
            a.dev[c] = -1;
        }
        a.node[g] = -1;
    }
}

__global__ void __launch_bounds__(kTabThreads, 2)
place_gangs_kernel(const __grid_constant__ GangsArgs ga) {
    __shared__ PodsSmem s;
    __shared__ int sOk;
    const PodsArgs& a = ga.p;
    const int tid = threadIdx.x, lane = tid & 31;
    const unsigned int b = blockIdx.x, G = gridDim.x;
    const int N = a.N, D = a.D;
    const long long stride = static_cast<long long>(G) * kTabThreads, first = static_cast<long long>(b) * kTabThreads + tid;
    unsigned int gen = 0;
    int round = 0;  // rounds run by every gang so far: info[0], and the parity of the deferred counts
    bool done = false;

    // ---- 0. the three index tensors checked before anything is read through them; outputs marked, tables copied
    {
        bool bad = false;
        for (long long g = first; g <= a.G; g += stride) {
            bad |= csr_bad(a.off, g, a.G, a.P, 1, kMaxPod);
            if (g < a.G) a.node[g] = -2;
        }
        for (long long j = first; j <= ga.J; j += stride) {
            bad |= csr_bad(ga.goff, j, ga.J, a.G, 1, LLONG_MAX);
            if (j < ga.J) {
                const int32_t m = __ldg(ga.gmin + j);
                bad |= m < 1 || m > static_cast<long long>(__ldg(ga.goff + j + 1)) - __ldg(ga.goff + j);
                ga.placed[j] = 0;
            }
        }
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -2;
        for (long long j = first; j < static_cast<long long>(N) * D; j += stride) {
            a.fc_out[j] = a.fc[j];
            a.fm_out[j] = a.fm[j];
        }
        if (__syncthreads_or(bad) && tid == 0) atomicExch(&a.ctl->bad_index, 1u);
    }
    if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
    if (*reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index)) {  // nothing is placed
        for (long long g = first; g < a.G; g += stride) a.node[g] = -1;
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -1;
        done = true;
        goto finish;
    }
    // each gang's pods in the domain: round 1's pending pods
    for (long long g0 = static_cast<long long>(b) * kTabThreads; g0 < a.G; g0 += stride) {
        const long long g = g0 + tid;
        bool ok = g < a.G;
        if (ok)
            for (int32_t c = __ldg(a.off + g), c1 = __ldg(a.off + g + 1); c < c1; ++c) {
                const int32_t core = __ldg(a.rc + c), mem = __ldg(a.rm + c);
                ok &= core >= 0 && core <= kCoreMax && mem >= 0 && mem <= kMemMax;
            }
        count_into_gang(ga.goff, ga.J, g, ok, ga.in_domain);
    }
    if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;

    for (long long gang = 0; gang < ga.J; ++gang) {
        const int32_t g_lo = __ldg(ga.goff + gang), g_hi = __ldg(ga.goff + gang + 1), need = __ldg(ga.gmin + gang);
        const int32_t* cur = nullptr;  // pending pods in pod order; round 1: the gang's range (position = pod - g_lo)
        long long n = __ldcg(ga.in_domain + gang);  // pending pods
        long long m = g_hi - g_lo;                   // positions of the pending set
        int which = 0;
        bool gang_done = n < need;  // also n == 0: never rounds, nothing committed
        if (gang_done)
            for (long long g = g_lo + first; g < g_hi; g += stride) {
                a.node[g] = -1;
                for (int32_t c = __ldg(a.off + g), c1 = __ldg(a.off + g + 1); c < c1; ++c) a.dev[c] = -1;
            }
        while (!gang_done) {
            ++round;
            pods_choose(a, cur, g_lo, m, s);
            if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
            unsigned int* const count = a.count[(round - 1) & 1];
            {
                const unsigned int committed = pods_commit(a, count, cur, g_lo, m, s);
                if (lane == 0 && committed) atomicAdd(ga.committed + gang, committed);
            }
            if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;

            // ---- 3. compact, or end the gang: keep it, or give it back
            {
                const long long tiles = (m + kPodBlock - 1) / kPodBlock;
                unsigned int* const next_count = a.count[round & 1];  // last read in the previous round's phase 3
                // the next round may be the next gang's first, over up to G positions
                for (long long t = first; t < (a.G + kPodBlock - 1) / kPodBlock; t += stride) next_count[t] = 0u;
                const long long lo = tiles * b / G, hi = tiles * (b + 1) / G;
                unsigned int before, total;
                deferred_prefix(count, tiles, lo, before, total, s.Red);
                const long long placed = __ldcg(ga.committed + gang);
                gang_done = total == 0u || placed + total < need;
                if (gang_done && placed < need) {  // roll back: every pod of the gang -1, its demand given back
                    give_back_pods(a, g_lo, g_hi, first, stride);
                    if (gang + 1 < ga.J && !grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
                } else {
                    if (gang_done && b == 0 && tid == 0) ga.placed[gang] = static_cast<int32_t>(placed);
                    pods_compact(a, cur, g_lo, m, lo, hi, a.set[which], before, s);
                    if (!gang_done) {
                        cur = a.set[which];
                        m = n = total;
                        which ^= 1;
                        if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
                    }
                }
            }
        }
    }
    done = true;
finish:
    if (b == 0 && tid == 0) {
        const bool bad = *reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index) != 0u;
        a.info[0] = bad ? 0 : round;
        a.info[1] = done ? 0 : 1;
        a.info[2] = bad ? 1 : 0;
    }
}

size_t gangs_scratch_bytes(int G, int J) { return PodsScratch(G, J).total; }

cudaError_t gangs_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                         const int32_t* req_core, const int32_t* req_mem, int P, const int32_t* pod_offsets, int G,
                         const int32_t* gang_offsets, const int32_t* gang_min, int J, int32_t* out_node, int8_t* out_dev,
                         int32_t* out_placed, int32_t* free_core_out, int32_t* free_mem_out, int32_t* info, void* scratch,
                         int device, cudaStream_t stream) {
    const PodsScratch L(G, J);
    GangsArgs ga{};
    PodsArgs& a = ga.p;
    a.fc = free_core; a.fm = free_mem; a.dv = d_valid; a.rc = req_core; a.rm = req_mem; a.off = pod_offsets;
    a.N = N; a.D = D; a.P = P; a.G = G;
    a.node = out_node; a.dev = out_dev; a.fc_out = free_core_out; a.fm_out = free_mem_out; a.info = info;
    ga.goff = gang_offsets; ga.gmin = gang_min; ga.J = J;
    ga.placed = out_placed;
    ga.in_domain = reinterpret_cast<unsigned int*>(static_cast<char*>(scratch) + L.in_domain);
    ga.committed = reinterpret_cast<unsigned int*>(static_cast<char*>(scratch) + L.committed);
    const cudaError_t err = pods_scratch(a, scratch, L, stream);
    if (err != cudaSuccess) return err;
    // Grid: as pods_launch, from N and G alone (the gang sizes are device data): no more CTAs than a round over all G
    // pods has choose work items; at least one, which finds G = 0's offsets bad.
    const long long tiles = (static_cast<long long>(N) + kTabWarps - 1) / kTabWarps;
    return coop_launch<place_gangs_kernel>(ga, tiles * static_cast<long long>(L.blocks), device, stream);
}

// ---- egpu::preempt_pods (DESIGN.md §2.14, §4.9): whole pods with priority preemption, rounds to the fixed point ----
//
// One cooperative launch.  Every (pod, node) question is answered by one warp holding the node's table in registers
// (lane l owns devices l and l + 32), so the in-node replay of a container is one __reduce_min_sync, and the reprieve
// chain of §2.14 step 3, serial per pair, runs a replay per step without touching shared memory:
//   0. the grid checks pod_offsets, run_offsets and node_offsets before anything is read through them, marks every
//      pod and container -2 and every running pod -1 (alive), and copies the tables to free_*_out (every round reads
//      them there).  After a barrier: if an index is bad nothing is placed and info[2] = 1; otherwise pods outside
//      the domain become -1, and each node is marked usable (pre_usable) when its table is in §2.1's domain and its
//      running data is consistent (an unusable node offers no candidate and is never written);
//   per round, over the pending pods (node = -2):
//   1a. choose, empty victim set: work items are (pod, chunk of nodes), chunk-major so that one pod's chunks spread
//       over CTAs.  Each warp replays the pod on its nodes of the chunk; the CTA reduces the warps' best keys and
//       writes one record per item (pre_record).  A pod that fits some node as it is is flagged;
//   1b. choose, with victims: the same items, for the pods no node took as it is: steps 2 and 3 of §2.14 per node
//       where the pod outranks an alive running pod (pre_victims: C, then the reprieve walk pre_walk); the records
//       are overwritten;
//   2.  reduce (pre_reduce): one thread per pending pod takes the smallest of its K records (§2.14's key is 142 bits,
//       so the records are three 64-bit words compared in order, not an atomic); a pod with none becomes -1;
//   3.  commit: the warp of node n walks the pending pods that chose n in pod order, §2.14's commit rule (pre_fits
//       for a pod that evicts nothing).  The replay and the chain are deterministic and nothing changed node n since
//       the choose phases, so the warp recomputes a pod's devices, and a committing preemptor's victims, instead of
//       storing them;
//   then every CTA reads the round's deferred count: zero ends the launch.
constexpr int kMaxRun = 128;     // running pods per node
constexpr int kPreChunks = 32;   // node chunks per pending pod in the choose phases

struct PreemptCtl {
    RoundsCtl bar;                // grid-barrier words
    unsigned long long timeouts;  // grid_barrier's count of waits that gave up (info[1] says whether one did)
    unsigned int bad_index;       // an index tensor (or run_gang_min) failed the check (info[2])
    unsigned int in_domain;       // some pod is in the domain (preempt_pods)
    unsigned int deferred[2];     // pods deferred by a round's commit, by round parity
    unsigned int budget[2];       // a round recorded a preemptor with a victim in a running job, by round parity
                                  // (preempt_gangs)
};

struct PreemptArgs {
    const int32_t* fc;     // the caller's tables [N][D], d_valid [N], containers [P], pod_offsets [G + 1], pod_prio [G]
    const int32_t* fm;
    const int32_t* dv;
    const int32_t* rc;
    const int32_t* rm;
    const int32_t* off;
    const int32_t* prio;
    const int32_t* qc;     // running containers [Q], run_offsets [H + 1], run_prio [H], node_offsets [N + 1]
    const int32_t* qm;
    const int8_t* qd;
    const int32_t* roff;
    const int32_t* rprio;
    const int32_t* noff;
    int N, D, K;           // K: node chunks per pod in the choose phases
    long long P, G, Q, H;
    int32_t* node;         // outputs: node per pod [G], device per container [P], evictor per running pod [H],
    int8_t* dev;           // tables [N][D], info [3]
    int32_t* evicted;
    int32_t* fc_out;
    int32_t* fm_out;
    int32_t* info;
    unsigned long long* rec;     // [G][K][3]: each (pod, chunk)'s smallest key
    unsigned long long* choice;  // [G]: the chosen node, bit 32 set when the victim set is not empty; ~0 = none
    unsigned int* has_empty;     // [G]: some node takes the pod as it is (phase 1a -> 1b)
    unsigned int* usable;        // [N]: table in the domain and running data consistent
    PreemptCtl* ctl;
};

// A node's table as one warp holds it: lane l's devices l and l + 32.
struct WarpTab {
    int32_t c[2], m[2];
};

// §2.14's choice key (highest victim priority, sum of victim priorities, victims, sum lc, sum lm, n) as three
// words compared in order: a = 0 for no victim, else (highest prio + 2^31) + 1; b = sum (prio + 2^31) << 8 | |V|;
// c = (sum lc << 21 | sum lm) << 31 | n.  All ones: no candidate.
struct PreKey {
    unsigned long long a, b, c;
};

__device__ __forceinline__ bool pre_less(const PreKey& x, const PreKey& y) {
    return x.a != y.a ? x.a < y.a : x.b != y.b ? x.b < y.b : x.c < y.c;
}

// §2.12's in-node replay by one warp on the table t (its first `rows` devices), updated to what the pod leaves.
// Each container takes the device with the smallest (lc, lm, d), one __reduce_min_sync over the lanes' keys.
// used: the lane's devices some container chose (bit 0: lane, bit 1: lane + 32).  Returns false when a container is
// outside §2.1's domain or finds no device.
__device__ __forceinline__ bool warp_replay(WarpTab& t, int rows, const int32_t* __restrict__ rc,
                                            const int32_t* __restrict__ rm, long long c0, int len, uint32_t& slc,
                                            uint32_t& slm, unsigned long long& cdev, unsigned int& used) {
    const int lane = threadIdx.x & 31;
    slc = 0;
    slm = 0;
    cdev = 0;
    used = 0;
    for (int k = 0; k < len; ++k) {
        const int32_t core = __ldg(rc + c0 + k), mem = __ldg(rm + c0 + k);
        if (core < 0 || core > kCoreMax || mem < 0 || mem > kMemMax) return false;
        uint32_t key = kNoKey;
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            const int d = lane + 32 * i;
            const int32_t lc = t.c[i] - core, lm = t.m[i] - mem;
            if (d < rows && (lc | lm) >= 0)
                key = min(key, (static_cast<uint32_t>(lc) << 24) | (static_cast<uint32_t>(lm) << 6) | static_cast<uint32_t>(d));
        }
        key = __reduce_min_sync(0xffffffffu, key);
        if (key == kNoKey) return false;
        const int d = static_cast<int>(key & 63u);
#pragma unroll
        for (int i = 0; i < 2; ++i)
            if (d == lane + 32 * i) {
                t.c[i] -= core;
                t.m[i] -= mem;
                used |= 1u << i;
            }
        slc += key >> 24;
        slm += (key >> 6) & 0x3FFFFu;
        cdev |= static_cast<unsigned long long>(d) << (6 * k);
    }
    return true;
}

// t += sign x the demand of running pod h (its containers' devices are in range: the node is usable).
__device__ __forceinline__ void add_running(const PreemptArgs& a, WarpTab& t, long long h, int sign) {
    const int lane = threadIdx.x & 31;
    for (int32_t c = __ldg(a.roff + h), c1 = __ldg(a.roff + h + 1); c < c1; ++c) {
        const int d = __ldg(a.qd + c);
        const int32_t core = sign * __ldg(a.qc + c), mem = sign * __ldg(a.qm + c);
#pragma unroll
        for (int i = 0; i < 2; ++i)
            if (d == lane + 32 * i) {
                t.c[i] += core;
                t.m[i] += mem;
            }
    }
}

// §2.14 step 3 for the pod of containers [c0, c0 + len) on node n, whose table as the round found it is t and whose
// running pods are [h0, h1) (at most kMaxRun: running pod h0 + lane + 32 i is slot i of the lane), from the victim
// candidates C, which is not empty: cand holds the lane's slots of C (bit i: slot lane + 32 i) and q[i] slot i's
// priority + 2^31 (its unsigned order is the priority's).  Returns false when n is not a candidate; otherwise t becomes
// the table plus the demand of V minus the pod's (what committing leaves), in_v holds V by slot, cdev the pod's devices
// and k the key.
__device__ __forceinline__ bool pre_walk(const PreemptArgs& a, WarpTab& t, int rows, unsigned int cand,
                                         const uint32_t (&q)[4], long long c0, int len, long long h0, int n,
                                         unsigned int& in_v, PreKey& k, unsigned long long& cdev) {
    const int lane = threadIdx.x & 31;
    WarpTab base = t;  // the table plus the demand of V
#pragma unroll
    for (int i = 0; i < 4; ++i)
        for (unsigned int m = __ballot_sync(0xffffffffu, (cand >> i) & 1u); m; m &= m - 1u)
            add_running(a, base, h0 + (__ffs(m) - 1) + 32 * i, 1);
    WarpTab w = base;
    uint32_t slc, slm;
    unsigned int used;
    if (!warp_replay(w, rows, a.rc, a.rm, c0, len, slc, slm, cdev, used)) return false;
    // walk C by (priority descending, h ascending): h is reprieved when the pod fits without evicting it
    in_v = cand;
    unsigned int left = cand;
    while (__any_sync(0xffffffffu, left != 0u)) {
        uint32_t bq = 0;
        int bi = 4;
#pragma unroll
        for (int i = 0; i < 4; ++i)
            if (((left >> i) & 1u) && (bi == 4 || q[i] > bq)) {
                bq = q[i];
                bi = i;
            }
        const uint32_t top = __reduce_max_sync(0xffffffffu, bi < 4 ? bq : 0u);
        const uint32_t at = __reduce_min_sync(0xffffffffu, bi < 4 && bq == top ? static_cast<uint32_t>(lane + 32 * bi) : ~0u);
        const int slot = static_cast<int>(at >> 5), owner = static_cast<int>(at & 31u);
        if (lane == owner) left &= ~(1u << slot);
        WarpTab trial = base;
        add_running(a, trial, h0 + at, -1);
        WarpTab tw = trial;
        uint32_t tlc, tlm;
        unsigned long long tdev;
        if (warp_replay(tw, rows, a.rc, a.rm, c0, len, tlc, tlm, tdev, used)) {
            base = trial;
            w = tw;
            slc = tlc;
            slm = tlm;
            cdev = tdev;
            if (lane == owner) in_v &= ~(1u << slot);
        }
    }
    uint32_t top = 0;
    unsigned long long sum = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
        if ((in_v >> i) & 1u) {
            top = max(top, q[i]);
            sum += q[i];
        }
    top = __reduce_max_sync(0xffffffffu, top);
    const unsigned int count = __reduce_add_sync(0xffffffffu, static_cast<unsigned int>(__popc(in_v)));
#pragma unroll
    for (int o = 16; o; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    k.a = static_cast<unsigned long long>(top) + 1ull;
    k.b = (sum << 8) | count;
    k.c = (((static_cast<unsigned long long>(slc) << 21) | slm) << 31) | static_cast<unsigned long long>(n);
    t = w;
    return true;
}

// §2.14 steps 2 and 3 for the pod of priority p: C is the alive running pods of lower priority, walked by pre_walk.
// The caller knows step 1 failed.
__device__ __forceinline__ bool pre_victims(const PreemptArgs& a, WarpTab& t, int rows, int32_t p, long long c0, int len,
                                            long long h0, long long h1, int n, unsigned int& in_v, PreKey& k,
                                            unsigned long long& cdev) {
    const int lane = threadIdx.x & 31;
    unsigned int cand = 0;  // C: alive running pods of lower priority
    uint32_t q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long h = h0 + lane + 32 * i;
        q[i] = 0;
        if (h < h1) {
            const int32_t r = __ldg(a.rprio + h);
            q[i] = static_cast<uint32_t>(r) ^ 0x80000000u;
            if (r < p && __ldcg(a.evicted + h) == -1) cand |= 1u << i;
        }
    }
    if (!__any_sync(0xffffffffu, cand != 0u)) return false;
    return pre_walk(a, t, rows, cand, q, c0, len, h0, n, in_v, k, cdev);
}

// pre_victims with C given: cand holds the lane's slots of C (bit i: slot lane + 32 i).
__device__ __forceinline__ bool pre_victims_capped(const PreemptArgs& a, WarpTab& t, int rows, unsigned int cand,
                                                   long long c0, int len, long long h0, long long h1, int n,
                                                   unsigned int& in_v, PreKey& k, unsigned long long& cdev) {
    const int lane = threadIdx.x & 31;
    if (!__any_sync(0xffffffffu, cand != 0u)) return false;
    uint32_t q[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const long long h = h0 + lane + 32 * i;
        q[i] = h < h1 ? static_cast<uint32_t>(__ldg(a.rprio + h)) ^ 0x80000000u : 0u;
    }
    return pre_walk(a, t, rows, cand, q, c0, len, h0, n, in_v, k, cdev);
}

// Node n's table from free_*_out into the warp's registers (the values past `rows` are not read).
__device__ __forceinline__ WarpTab load_tab(const PreemptArgs& a, int n, int rows) {
    const int lane = threadIdx.x & 31;
    WarpTab t;
    const size_t off = static_cast<size_t>(n) * a.D;
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const int d = lane + 32 * i;
        t.c[i] = d < rows ? __ldcg(a.fc_out + off + d) : 0;
        t.m[i] = d < rows ? __ldcg(a.fm_out + off + d) : 0;
    }
    return t;
}

// ---- 0. (end) usable[n], one warp per node: the table is in §2.1's domain and the running data consistent (every
// running container on a valid device and in the domain, and the free values plus the running demand within it).
// sSumC / sSumM: kTabWarps rows of kMaxD words of shared memory.
__device__ __forceinline__ void pre_usable(const PreemptArgs& a, int32_t (*sSumC)[kMaxD], int32_t (*sSumM)[kMaxD]) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int N = a.N, D = a.D;
    const long long wstride = static_cast<long long>(gridDim.x) * kTabWarps;
    for (long long n = static_cast<long long>(blockIdx.x) * kTabWarps + warp; n < N; n += wstride) {
        const int dv = __ldg(a.dv + n);
        bool ok = dv >= 1 && dv <= D;
        const size_t off = static_cast<size_t>(n) * D;
        for (int j = lane; j < kMaxD; j += 32) {
            const int32_t c = ok && j < dv ? __ldg(a.fc + off + j) : 0, m = ok && j < dv ? __ldg(a.fm + off + j) : 0;
            ok &= c >= 0 && c <= kCoreMax && m >= 0 && m <= kMemMax;
            sSumC[warp][j] = c;
            sSumM[warp][j] = m;
        }
        __syncwarp();
        const int32_t q0 = __ldg(a.roff + __ldg(a.noff + n)), q1 = __ldg(a.roff + __ldg(a.noff + n + 1));
        for (int32_t c = q0 + lane; ok && c < q1; c += 32) {
            const int d = __ldg(a.qd + c);
            const int32_t core = __ldg(a.qc + c), mem = __ldg(a.qm + c);
            ok = d >= 0 && d < dv && core >= 0 && core <= kCoreMax && mem >= 0 && mem <= kMemMax;
            if (ok) {
                atomicAdd(&sSumC[warp][d], core);
                atomicAdd(&sSumM[warp][d], mem);
            }
        }
        __syncwarp();
        for (int j = lane; ok && j < dv; j += 32) ok = sSumC[warp][j] <= kCoreMax && sSumM[warp][j] <= kMemMax;
        ok = __all_sync(0xffffffffu, ok);
        if (lane == 0) a.usable[n] = ok ? 1u : 0u;
        __syncwarp();
    }
}

// ---- 1. (end of a choose item (g, k)) the smallest of the CTA's warps' keys is the item's record; in pass 0, a pod
// that some node takes as it is is flagged.  Every thread of the CTA calls it with its warp's key.
__device__ __forceinline__ void pre_record(const PreemptArgs& a, PreKey best, long long g, long long k, int pass,
                                           PreKey* sKey) {
    const int tid = threadIdx.x;
    if ((tid & 31) == 0) sKey[tid >> 5] = best;
    __syncthreads();
    if (tid == 0) {
        for (int w = 1; w < kTabWarps; ++w)
            if (pre_less(sKey[w], best)) best = sKey[w];
        unsigned long long* r = a.rec + 3 * (g * a.K + k);
        r[0] = best.a;
        r[1] = best.b;
        r[2] = best.c;
        if (pass == 0 && best.a == 0ull) a.has_empty[g] = 1u;
    }
    __syncthreads();
}

// ---- 2. reduce: each pending pod of [g_lo, g_hi) takes the smallest of its records
__device__ __forceinline__ void pre_reduce(const PreemptArgs& a, long long g_lo, long long g_hi) {
    const long long stride = static_cast<long long>(gridDim.x) * kTabThreads;
    const PreKey none{~0ull, ~0ull, ~0ull};
    for (long long g = g_lo + static_cast<long long>(blockIdx.x) * kTabThreads + threadIdx.x; g < g_hi; g += stride) {
        if (__ldcg(a.node + g) != -2) continue;
        PreKey best = none;
        for (int k = 0; k < a.K; ++k) {
            const unsigned long long* r = a.rec + 3 * (g * a.K + k);
            const PreKey key{__ldcg(r), __ldcg(r + 1), __ldcg(r + 2)};
            if (pre_less(key, best)) best = key;
        }
        a.has_empty[g] = 0u;
        if (best.a == ~0ull) {  // fits no node when scored: -1 for good
            a.choice[g] = ~0ull;
            a.node[g] = -1;
            for (int32_t c = __ldg(a.off + g), c1 = __ldg(a.off + g + 1); c < c1; ++c) a.dev[c] = -1;
        } else {
            a.choice[g] = (best.a != 0ull ? 1ull << 32 : 0ull) | (best.c & 0x7fffffffull);
        }
    }
}

// ---- 3. (a pod that evicts nothing) §2.12 on node table t, in registers: w = t becomes what the pod leaves and cdev
// holds its devices.  The pod commits when none of its devices is closed and the demand committed before (acc_*)
// fits on top of its own; then its demand joins acc_*, otherwise its devices close.  Returns whether it commits.
__device__ __forceinline__ bool pre_fits(const PreemptArgs& a, const WarpTab& t, WarpTab& w, int rows, long long c0,
                                         int len, int32_t (&acc_c)[2], int32_t (&acc_m)[2], unsigned int& closed,
                                         unsigned long long& cdev) {
    uint32_t slc, slm;
    unsigned int used;
    warp_replay(w, rows, a.rc, a.rm, c0, len, slc, slm, cdev, used);
    bool ok = true;
#pragma unroll
    for (int i = 0; i < 2; ++i)
        if ((used >> i) & 1u) ok &= !((closed >> i) & 1u) && acc_c[i] <= w.c[i] && acc_m[i] <= w.m[i];
    const bool commit = __all_sync(0xffffffffu, ok);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        if (commit) {
            acc_c[i] += t.c[i] - w.c[i];
            acc_m[i] += t.m[i] - w.m[i];
        } else {
            closed |= used;
        }
    }
    return commit;
}

__global__ void __launch_bounds__(kTabThreads, 2)
preempt_pods_kernel(const __grid_constant__ PreemptArgs a) {
    __shared__ int32_t sSumC[kTabWarps][kMaxD], sSumM[kTabWarps][kMaxD];  // phase 0: free + running demand per device
    __shared__ PreKey sKey[kTabWarps];
    __shared__ int sOk;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int b = blockIdx.x, G = gridDim.x;
    const int N = a.N, D = a.D, K = a.K;
    const long long stride = static_cast<long long>(G) * kTabThreads, first = static_cast<long long>(b) * kTabThreads + tid;
    const long long wstride = static_cast<long long>(G) * kTabWarps, wfirst = static_cast<long long>(b) * kTabWarps + warp;
    const PreKey none{~0ull, ~0ull, ~0ull};
    unsigned int gen = 0;
    int round = 0;
    bool done = false;

    // ---- 0. the three index tensors checked before anything is read through them; outputs marked, tables copied
    {
        bool bad = false;
        for (long long g = first; g <= a.G; g += stride) {
            bad |= csr_bad(a.off, g, a.G, a.P, 1, kMaxPod);
            if (g < a.G) a.node[g] = -2;
        }
        for (long long h = first; h <= a.H; h += stride) {
            bad |= csr_bad(a.roff, h, a.H, a.Q, 1, kMaxPod);
            if (h < a.H) a.evicted[h] = -1;
        }
        for (long long n = first; n <= N; n += stride) bad |= csr_bad(a.noff, n, N, a.H, 0, kMaxRun);
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -2;
        for (long long j = first; j < static_cast<long long>(N) * D; j += stride) {
            a.fc_out[j] = a.fc[j];
            a.fm_out[j] = a.fm[j];
        }
        if (__syncthreads_or(bad) && tid == 0) atomicExch(&a.ctl->bad_index, 1u);
    }
    if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
    if (*reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index)) {  // nothing is placed or evicted
        for (long long g = first; g < a.G; g += stride) a.node[g] = -1;
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -1;
        done = true;
        goto finish;
    }
    {  // pods outside the domain are -1; the nodes a pod may use
        bool in_domain = false;
        for (long long g = first; g < a.G; g += stride) {
            const int32_t c0 = __ldg(a.off + g), c1 = __ldg(a.off + g + 1);
            bool ok = true;
            for (int32_t c = c0; c < c1; ++c) {
                const int32_t core = __ldg(a.rc + c), mem = __ldg(a.rm + c);
                ok &= core >= 0 && core <= kCoreMax && mem >= 0 && mem <= kMemMax;
            }
            if (!ok) {
                a.node[g] = -1;
                for (int32_t c = c0; c < c1; ++c) a.dev[c] = -1;
            }
            in_domain |= ok;
        }
        if (__syncthreads_or(in_domain) && tid == 0) a.ctl->in_domain = 1u;
        pre_usable(a, sSumC, sSumM);
    }
    if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
    done = *reinterpret_cast<volatile unsigned int*>(&a.ctl->in_domain) == 0u;

    while (!done) {
        ++round;
        // ---- 1a. / 1b. choose: (pod, chunk) items, chunk-major
        for (int pass = 0; pass < 2; ++pass) {
            // this round's count was round - 2's, which every CTA read before the barriers of round - 1
            if (pass == 1 && b == 0 && tid == 0) a.ctl->deferred[round & 1] = 0u;
            const long long items = static_cast<long long>(K) * a.G;
            for (long long it = items * b / G, hi = items * (b + 1) / G; it < hi; ++it) {
                const long long g = it % a.G, k = it / a.G;
                if (__ldcg(a.node + g) != -2) continue;
                if (pass == 1 && __ldcg(a.has_empty + g)) continue;
                const int32_t c0 = __ldg(a.off + g), len = __ldg(a.off + g + 1) - c0, p = __ldg(a.prio + g);
                PreKey best = none;
                for (long long n = N * k / K + warp, n1 = N * (k + 1) / K; n < n1; n += kTabWarps) {
                    const int rows = __ldcg(a.usable + n) ? __ldg(a.dv + n) : 0;
                    if (!rows) continue;
                    WarpTab t = load_tab(a, static_cast<int>(n), rows);
                    uint32_t slc, slm;
                    unsigned long long cdev;
                    unsigned int used;
                    PreKey key = none;
                    if (pass == 0) {
                        if (warp_replay(t, rows, a.rc, a.rm, c0, len, slc, slm, cdev, used))
                            key = PreKey{0ull, 0ull,
                                         (((static_cast<unsigned long long>(slc) << 21) | slm) << 31) |
                                             static_cast<unsigned long long>(n)};
                    } else {
                        unsigned int in_v;
                        pre_victims(a, t, rows, p, c0, len, __ldg(a.noff + n), __ldg(a.noff + n + 1),
                                    static_cast<int>(n), in_v, key, cdev);
                    }
                    if (pre_less(key, best)) best = key;
                }
                pre_record(a, best, g, k, pass, sKey);
            }
            if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
        }

        pre_reduce(a, 0, a.G);
        if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;

        // ---- 3. commit: per node, the pods that chose it in pod order
        for (long long n = wfirst; n < N; n += wstride) {
            const int rows = __ldcg(a.usable + n) ? __ldg(a.dv + n) : 0;
            if (!rows) continue;  // no pod chose it: it keeps its copy
            WarpTab t = load_tab(a, static_cast<int>(n), rows);
            int32_t acc_c[2] = {0, 0}, acc_m[2] = {0, 0};
            unsigned int closed = 0;  // the lane's devices a pod that did not commit chose
            bool node_closed = false, chosen = false, dirty = false;
            unsigned int deferred = 0;
            const long long h0 = __ldg(a.noff + n), h1 = __ldg(a.noff + n + 1);
            for (long long g0 = 0; g0 < a.G; g0 += 32) {
                const long long gl = g0 + lane;
                unsigned long long ch = ~0ull;
                if (gl < a.G && __ldcg(a.node + gl) == -2) ch = __ldcg(a.choice + gl);
                for (unsigned int mb = __ballot_sync(0xffffffffu, (ch & 0xffffffffull) == static_cast<unsigned long long>(n));
                     mb; mb &= mb - 1u) {
                    const int j = __ffs(mb) - 1;
                    const long long g = g0 + j;
                    const bool evicts = (__shfl_sync(0xffffffffu, ch, j) >> 32) != 0ull;
                    if (node_closed || (evicts && chosen)) {
                        chosen = true;
                        node_closed |= evicts;
                        ++deferred;
                        continue;
                    }
                    chosen = true;
                    const int32_t c0 = __ldg(a.off + g), len = __ldg(a.off + g + 1) - c0;
                    WarpTab w = t;
                    unsigned long long cdev;
                    bool commit = true;
                    if (!evicts) {
                        commit = pre_fits(a, t, w, rows, c0, len, acc_c, acc_m, closed, cdev);
                    } else {  // the first pod of the round on n: evict V, then take the pod's demand
                        unsigned int in_v;
                        PreKey key;
                        pre_victims(a, w, rows, __ldg(a.prio + g), c0, len, h0, h1, static_cast<int>(n), in_v, key, cdev);
#pragma unroll
                        for (int i = 0; i < 4; ++i)
                            if ((in_v >> i) & 1u) a.evicted[h0 + lane + 32 * i] = static_cast<int32_t>(g);
                        t = w;
                        node_closed = true;
                    }
                    if (commit) {
                        if (lane == 0) a.node[g] = static_cast<int32_t>(n);
                        if (lane < len) a.dev[c0 + lane] = static_cast<int8_t>((cdev >> (6 * lane)) & 63u);
                        dirty = true;
                    } else {
                        ++deferred;
                    }
                }
            }
            if (dirty) {
                const size_t off = static_cast<size_t>(n) * D;
#pragma unroll
                for (int i = 0; i < 2; ++i)
                    if (lane + 32 * i < rows) {
                        a.fc_out[off + lane + 32 * i] = t.c[i] - acc_c[i];
                        a.fm_out[off + lane + 32 * i] = t.m[i] - acc_m[i];
                    }
            }
            if (lane == 0 && deferred) atomicAdd(&a.ctl->deferred[round & 1], deferred);
        }
        if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
        done = *reinterpret_cast<volatile unsigned int*>(&a.ctl->deferred[round & 1]) == 0u;
    }
finish:
    if (b == 0 && tid == 0) {
        const bool bad = *reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index) != 0u;
        a.info[0] = !bad && *reinterpret_cast<volatile unsigned int*>(&a.ctl->in_domain) ? round : 0;
        a.info[1] = done ? 0 : 1;
        a.info[2] = bad ? 1 : 0;
    }
}

static int preempt_chunks(int N) { return std::max(1, std::min(kPreChunks, (N + kTabWarps - 1) / kTabWarps)); }

// preempt_pods' and preempt_gangs' scratch (preempt_pods: J = R = 0, and it leaves pre, vdev, vmask and cap alone),
// byte offsets: barrier words | has_empty uint32[G] | pre uint32[G] | in_domain uint32[J] | committed uint32[J] |
// alive int32[R] | used int32[R] | (16-aligned) records uint64[G][K][3] | choice uint64[G] | vdev uint64[G] | vmask
// uint32[G][4] | cap uint32[N][4] | usable uint32[N]; everything before the records (`zeroed` bytes) starts at zero.
struct PreemptScratch {
    int K;
    size_t has_empty, pre, in_domain, committed, alive, used, zeroed, rec, choice, vdev, vmask, cap, usable, total;
    PreemptScratch(int N, int G, int J, int R) {
        K = preempt_chunks(N);
        has_empty = sizeof(PreemptCtl);
        pre = has_empty + 4 * static_cast<size_t>(G);
        in_domain = pre + 4 * static_cast<size_t>(G);
        committed = in_domain + 4 * static_cast<size_t>(J);
        alive = committed + 4 * static_cast<size_t>(J);
        used = alive + 4 * static_cast<size_t>(R);
        zeroed = used + 4 * static_cast<size_t>(R);
        rec = (zeroed + 15) & ~size_t(15);
        choice = rec + 24 * static_cast<size_t>(G) * K;
        vdev = choice + 8 * static_cast<size_t>(G);
        vmask = vdev + 8 * static_cast<size_t>(G);
        cap = vmask + 16 * static_cast<size_t>(G);
        usable = cap + 16 * static_cast<size_t>(N);
        total = usable + 4 * static_cast<size_t>(N);
    }
};

// Points a's scratch arrays into `scratch` as L lays them out and zeroes its head on `stream`.
static cudaError_t preempt_scratch(PreemptArgs& a, void* scratch, const PreemptScratch& L, cudaStream_t stream) {
    char* s = static_cast<char*>(scratch);
    a.K = L.K;
    a.ctl = reinterpret_cast<PreemptCtl*>(s);
    a.has_empty = reinterpret_cast<unsigned int*>(s + L.has_empty);
    a.rec = reinterpret_cast<unsigned long long*>(s + L.rec);
    a.choice = reinterpret_cast<unsigned long long*>(s + L.choice);
    a.usable = reinterpret_cast<unsigned int*>(s + L.usable);
    return cudaMemsetAsync(scratch, 0, L.zeroed, stream);
}

size_t preempt_scratch_bytes(int N, int G) { return PreemptScratch(N, G, 0, 0).total; }

cudaError_t preempt_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N, int D,
                           const int32_t* req_core, const int32_t* req_mem, int P, const int32_t* pod_offsets,
                           const int32_t* pod_prio, int G, const int32_t* run_core, const int32_t* run_mem,
                           const int8_t* run_dev, int Q, const int32_t* run_offsets, const int32_t* run_prio, int H,
                           const int32_t* node_offsets, int32_t* out_node, int8_t* out_dev, int32_t* out_evicted,
                           int32_t* free_core_out, int32_t* free_mem_out, int32_t* info, void* scratch, int device,
                           cudaStream_t stream) {
    const PreemptScratch L(N, G, 0, 0);
    PreemptArgs a{};
    a.fc = free_core; a.fm = free_mem; a.dv = d_valid; a.rc = req_core; a.rm = req_mem; a.off = pod_offsets;
    a.prio = pod_prio; a.qc = run_core; a.qm = run_mem; a.qd = run_dev; a.roff = run_offsets; a.rprio = run_prio;
    a.noff = node_offsets;
    a.N = N; a.D = D; a.P = P; a.G = G; a.Q = Q; a.H = H;
    a.node = out_node; a.dev = out_dev; a.evicted = out_evicted; a.fc_out = free_core_out; a.fm_out = free_mem_out;
    a.info = info;
    const cudaError_t err = preempt_scratch(a, scratch, L, stream);
    if (err != cudaSuccess) return err;
    // Grid: no more CTAs than round 1 has choose items; at least one, which finds G = 0's offsets bad.
    return coop_launch<preempt_pods_kernel>(a, static_cast<long long>(L.K) * G, device, stream);
}

// ---- egpu::preempt_gangs (DESIGN.md §2.15, §4.10): gangs with priority preemption, in gang order ----
//
// One cooperative launch.  The outer loop over gangs is place_gangs_kernel's; a gang's rounds are preempt_pods_kernel's
// phases over the gang's pending pods (node = -2 inside [gang_offsets[j], gang_offsets[j + 1])), with two changes:
//   0. as preempt_pods, plus gang_offsets, gang_min, run_gang and run_gang_min checked before anything is read through
//      them.  After the check's barrier, each gang's pods in the domain (count_into_gang) and each running job's alive
//      pods are counted;
//      a job's slack is max(0, alive - run_gang_min) wherever it is read, so evictions and their undoing only move
//      the alive count;
//   1a. before the choose items, one warp per usable node writes the capped C (§2.15 rule 1) as a 128-bit slot mask
//       from the round-start slacks; 1b's reprieve walk starts from that mask (pre_victims_capped);
//   3.  commit: as preempt_pods, except that a first-on-node preemptor with a victim in a running job only records
//       its victims and devices and flags the round.  In a flagged round one warp then walks the gang's recorded
//       preemptors in pod order and counts their victims per job (§2.15 rule 2; a pod passes when no atomicAdd of its
//       own victims finds the count at the job's slack), and after another barrier the passing ones are applied, one
//       warp per pod.  Unflagged rounds (every round when no running pod is in a job) skip both barriers;
//   end of a gang: placed + deferred < gang_min or nothing deferred ends it.  A gang given back is rolled back by
//   integer atomics: its pods' demand returns to the tables (give_back_pods), and every running pod it evicted is
//   alive again, its demand taken from the tables and its job's count restored; one barrier follows before the next
//   gang reads them.
struct PreGangsArgs {
    PreemptArgs p;               // tables, containers, pod_offsets, running pods, the outputs node, dev, evicted,
                                 // tables and info, and the scratch ctl, rec, choice, has_empty, usable (p.prio unused)
    const int32_t* goff;         // gang_offsets [J + 1], gang_min [J], gang_prio [J], run_gang [H], run_gang_min [R]
    const int32_t* gmin;
    const int32_t* gprio;
    const int32_t* rgang;
    const int32_t* rgmin;
    long long J, R;
    int32_t* placed;             // output: placed pods per gang [J]
    unsigned int* in_domain;     // [J]: each gang's pods in the domain
    unsigned int* committed;     // [J]: each gang's committed pods
    int32_t* alive;              // [R]: each running job's pods not evicted
    int32_t* used;               // [R]: the budget pass's victims per job, zeroed again by the apply phase
    unsigned int* pre;           // [G]: 1 a preemptor waiting for the budget, 2 it passed, 0 otherwise
    unsigned int* vmask;         // [G][4]: a waiting preemptor's victims by slot (bit lane of word i: slot lane + 32 i)
    unsigned long long* vdev;    // [G]: a waiting preemptor's devices
    unsigned int* cap;           // [N][4]: the round's capped C per node, by slot
};

__global__ void __launch_bounds__(kTabThreads, 2)
preempt_gangs_kernel(const __grid_constant__ PreGangsArgs ga) {
    __shared__ int32_t sSumC[kTabWarps][kMaxD], sSumM[kTabWarps][kMaxD];  // phase 0: free + running demand per device
    __shared__ PreKey sKey[kTabWarps];
    __shared__ int sOk;
    const PreemptArgs& a = ga.p;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const unsigned int b = blockIdx.x, G = gridDim.x;
    const int N = a.N, D = a.D, K = a.K;
    const long long stride = static_cast<long long>(G) * kTabThreads, first = static_cast<long long>(b) * kTabThreads + tid;
    const long long wstride = static_cast<long long>(G) * kTabWarps, wfirst = static_cast<long long>(b) * kTabWarps + warp;
    const PreKey none{~0ull, ~0ull, ~0ull};
    unsigned int gen = 0;
    int round = 0;  // rounds run by every gang so far: info[0], and the parity of the round counters
    bool done = false;

    // ---- 0. the five index tensors and run_gang_min checked before anything is read through them
    {
        bool bad = false;
        for (long long g = first; g <= a.G; g += stride) {
            bad |= csr_bad(a.off, g, a.G, a.P, 1, kMaxPod);
            if (g < a.G) a.node[g] = -2;
        }
        for (long long j = first; j <= ga.J; j += stride) {
            bad |= csr_bad(ga.goff, j, ga.J, a.G, 1, LLONG_MAX);
            if (j < ga.J) {
                const int32_t m = __ldg(ga.gmin + j);
                bad |= m < 1 || m > static_cast<long long>(__ldg(ga.goff + j + 1)) - __ldg(ga.goff + j);
                ga.placed[j] = 0;
            }
        }
        for (long long h = first; h <= a.H; h += stride) {
            bad |= csr_bad(a.roff, h, a.H, a.Q, 1, kMaxPod);
            if (h < a.H) {
                const int32_t r = __ldg(ga.rgang + h);
                bad |= r < -1 || r >= ga.R;
                a.evicted[h] = -1;
            }
        }
        for (long long n = first; n <= N; n += stride) bad |= csr_bad(a.noff, n, N, a.H, 0, kMaxRun);
        for (long long r = first; r < ga.R; r += stride) bad |= __ldg(ga.rgmin + r) < 0;
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -2;
        for (long long j = first; j < static_cast<long long>(N) * D; j += stride) {
            a.fc_out[j] = a.fc[j];
            a.fm_out[j] = a.fm[j];
        }
        if (__syncthreads_or(bad) && tid == 0) atomicExch(&a.ctl->bad_index, 1u);
    }
    if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
    if (*reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index)) {  // nothing is placed or evicted
        for (long long g = first; g < a.G; g += stride) a.node[g] = -1;
        for (long long c = first; c < a.P; c += stride) a.dev[c] = -1;
        done = true;
        goto finish;
    }
    {  // pods outside the domain are -1, the others counted into their gang; the usable nodes; the jobs' alive pods
        for (long long g0 = static_cast<long long>(b) * kTabThreads; g0 < a.G; g0 += stride) {
            const long long g = g0 + tid;
            bool ok = g < a.G;
            if (ok) {
                const int32_t c0 = __ldg(a.off + g), c1 = __ldg(a.off + g + 1);
                for (int32_t c = c0; c < c1; ++c) {
                    const int32_t core = __ldg(a.rc + c), mem = __ldg(a.rm + c);
                    ok &= core >= 0 && core <= kCoreMax && mem >= 0 && mem <= kMemMax;
                }
                if (!ok) {
                    a.node[g] = -1;
                    for (int32_t c = c0; c < c1; ++c) a.dev[c] = -1;
                }
            }
            count_into_gang(ga.goff, ga.J, g, ok, ga.in_domain);
        }
        for (long long h = first; h < a.H; h += stride) {
            const int32_t r = __ldg(ga.rgang + h);
            if (r >= 0) atomicAdd(ga.alive + r, 1);
        }
        pre_usable(a, sSumC, sSumM);
    }
    if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;

    for (long long gang = 0; gang < ga.J; ++gang) {
        const int32_t g_lo = __ldg(ga.goff + gang), g_hi = __ldg(ga.goff + gang + 1), need = __ldg(ga.gmin + gang);
        const int32_t p = __ldg(ga.gprio + gang);
        const long long size = g_hi - g_lo;
        bool gang_done = static_cast<long long>(__ldcg(ga.in_domain + gang)) < need;  // never rounds, nothing changes
        if (gang_done)
            for (long long g = g_lo + first; g < g_hi; g += stride) {
                a.node[g] = -1;
                for (int32_t c = __ldg(a.off + g), c1 = __ldg(a.off + g + 1); c < c1; ++c) a.dev[c] = -1;
            }
        while (!gang_done) {
            ++round;
            // ---- 1a. / 1b. choose: (pod, chunk) items over the gang's pods, chunk-major
            for (int pass = 0; pass < 2; ++pass) {
                if (pass == 0)  // the capped C of every usable node, from the round-start slacks
                    for (long long n = wfirst; n < N; n += wstride) {
                        if (!__ldcg(a.usable + n)) continue;
                        const long long h0 = __ldg(a.noff + n), h1 = __ldg(a.noff + n + 1);
                        bool in_c[4];
                        int32_t job[4];
                        uint32_t q[4];
                        int later[4];
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const long long h = h0 + lane + 32 * i;
                            in_c[i] = false;
                            job[i] = -1;
                            q[i] = 0;
                            later[i] = 0;
                            if (h < h1) {
                                const int32_t r = __ldg(a.rprio + h);
                                q[i] = static_cast<uint32_t>(r) ^ 0x80000000u;
                                in_c[i] = r < p && __ldcg(a.evicted + h) == -1;
                                job[i] = in_c[i] ? __ldg(ga.rgang + h) : -1;
                            }
                        }
                        if (__any_sync(0xffffffffu, job[0] >= 0 || job[1] >= 0 || job[2] >= 0 || job[3] >= 0))
                            // later[i]: the pods of C in slot i's job after it in the walk order (priority
                            // descending, h ascending)
                            for (int s = 0; s < static_cast<int>(h1 - h0); ++s) {
                                const int si = s >> 5, src = s & 31;
                                const int32_t js = __shfl_sync(0xffffffffu, si == 0 ? job[0] : si == 1 ? job[1] : si == 2 ? job[2] : job[3], src);
                                const uint32_t qs = __shfl_sync(0xffffffffu, si == 0 ? q[0] : si == 1 ? q[1] : si == 2 ? q[2] : q[3], src);
                                if (js < 0) continue;
#pragma unroll
                                for (int i = 0; i < 4; ++i)
                                    later[i] += job[i] == js && (qs < q[i] || (qs == q[i] && s > lane + 32 * i));
                            }
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            bool keep = in_c[i];
                            if (keep && job[i] >= 0)
                                keep = later[i] < __ldcg(ga.alive + job[i]) - __ldg(ga.rgmin + job[i]);
                            const unsigned int m = __ballot_sync(0xffffffffu, keep);
                            if (lane == 0) ga.cap[4 * n + i] = m;
                        }
                    }
                if (pass == 1 && b == 0 && tid == 0) {  // round - 2's counters, read before round - 1's barriers
                    a.ctl->deferred[round & 1] = 0u;
                    a.ctl->budget[round & 1] = 0u;
                }
                const long long items = static_cast<long long>(K) * size;
                for (long long it = items * b / G, hi = items * (b + 1) / G; it < hi; ++it) {
                    const long long g = g_lo + it % size, k = it / size;
                    if (__ldcg(a.node + g) != -2) continue;
                    if (pass == 1 && __ldcg(a.has_empty + g)) continue;
                    const int32_t c0 = __ldg(a.off + g), len = __ldg(a.off + g + 1) - c0;
                    PreKey best = none;
                    for (long long n = N * k / K + warp, n1 = N * (k + 1) / K; n < n1; n += kTabWarps) {
                        const int rows = __ldcg(a.usable + n) ? __ldg(a.dv + n) : 0;
                        if (!rows) continue;
                        WarpTab t = load_tab(a, static_cast<int>(n), rows);
                        uint32_t slc, slm;
                        unsigned long long cdev;
                        unsigned int used;
                        PreKey key = none;
                        if (pass == 0) {
                            if (warp_replay(t, rows, a.rc, a.rm, c0, len, slc, slm, cdev, used))
                                key = PreKey{0ull, 0ull,
                                             (((static_cast<unsigned long long>(slc) << 21) | slm) << 31) |
                                                 static_cast<unsigned long long>(n)};
                        } else {
                            unsigned int cand = 0, in_v;
#pragma unroll
                            for (int i = 0; i < 4; ++i) cand |= ((__ldcg(ga.cap + 4 * n + i) >> lane) & 1u) << i;
                            pre_victims_capped(a, t, rows, cand, c0, len, __ldg(a.noff + n), __ldg(a.noff + n + 1),
                                               static_cast<int>(n), in_v, key, cdev);
                        }
                        if (pre_less(key, best)) best = key;
                    }
                    pre_record(a, best, g, k, pass, sKey);
                }
                if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
            }

            pre_reduce(a, g_lo, g_hi);
            if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;

            // ---- 3. commit: per node, the gang's pods that chose it in pod order
            for (long long n = wfirst; n < N; n += wstride) {
                const int rows = __ldcg(a.usable + n) ? __ldg(a.dv + n) : 0;
                if (!rows) continue;  // no pod chose it: it keeps its copy
                WarpTab t = load_tab(a, static_cast<int>(n), rows);
                int32_t acc_c[2] = {0, 0}, acc_m[2] = {0, 0};
                unsigned int closed = 0;  // the lane's devices a pod that did not commit chose
                bool node_closed = false, chosen = false, dirty = false;
                unsigned int deferred = 0, committed = 0;
                const long long h0 = __ldg(a.noff + n), h1 = __ldg(a.noff + n + 1);
                for (long long g0 = g_lo; g0 < g_hi; g0 += 32) {
                    const long long gl = g0 + lane;
                    unsigned long long ch = ~0ull;
                    if (gl < g_hi && __ldcg(a.node + gl) == -2) ch = __ldcg(a.choice + gl);
                    for (unsigned int mb = __ballot_sync(0xffffffffu, (ch & 0xffffffffull) == static_cast<unsigned long long>(n));
                         mb; mb &= mb - 1u) {
                        const int j = __ffs(mb) - 1;
                        const long long g = g0 + j;
                        const bool evicts = (__shfl_sync(0xffffffffu, ch, j) >> 32) != 0ull;
                        if (node_closed || (evicts && chosen)) {
                            chosen = true;
                            node_closed |= evicts;
                            ++deferred;
                            continue;
                        }
                        chosen = true;
                        const int32_t c0 = __ldg(a.off + g), len = __ldg(a.off + g + 1) - c0;
                        WarpTab w = t;
                        unsigned long long cdev;
                        bool commit = true;
                        if (!evicts) {
                            commit = pre_fits(a, t, w, rows, c0, len, acc_c, acc_m, closed, cdev);
                            if (!commit) ++deferred;
                        } else {  // the first pod of the round on n: its victims from the same capped C
                            unsigned int cand = 0, in_v;
                            PreKey key;
#pragma unroll
                            for (int i = 0; i < 4; ++i) cand |= ((__ldcg(ga.cap + 4 * n + i) >> lane) & 1u) << i;
                            pre_victims_capped(a, w, rows, cand, c0, len, h0, h1, static_cast<int>(n), in_v, key, cdev);
                            bool in_job = false;
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                if ((in_v >> i) & 1u) in_job |= __ldg(ga.rgang + h0 + lane + 32 * i) >= 0;
                            node_closed = true;
                            if (__any_sync(0xffffffffu, in_job)) {  // the budget pass decides
#pragma unroll
                                for (int i = 0; i < 4; ++i) {
                                    const unsigned int m = __ballot_sync(0xffffffffu, (in_v >> i) & 1u);
                                    if (lane == 0) ga.vmask[4 * g + i] = m;
                                }
                                if (lane == 0) {
                                    ga.vdev[g] = cdev;
                                    ga.pre[g] = 1u;
                                    a.ctl->budget[round & 1] = 1u;
                                }
                                continue;
                            }
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                if ((in_v >> i) & 1u) a.evicted[h0 + lane + 32 * i] = static_cast<int32_t>(g);
                            t = w;
                        }
                        if (commit) {
                            if (lane == 0) a.node[g] = static_cast<int32_t>(n);
                            if (lane < len) a.dev[c0 + lane] = static_cast<int8_t>((cdev >> (6 * lane)) & 63u);
                            dirty = true;
                            ++committed;
                        }
                    }
                }
                if (dirty) {
                    const size_t off = static_cast<size_t>(n) * D;
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        if (lane + 32 * i < rows) {
                            a.fc_out[off + lane + 32 * i] = t.c[i] - acc_c[i];
                            a.fm_out[off + lane + 32 * i] = t.m[i] - acc_m[i];
                        }
                }
                if (lane == 0 && deferred) atomicAdd(&a.ctl->deferred[round & 1], deferred);
                if (lane == 0 && committed) atomicAdd(ga.committed + gang, committed);
            }
            if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;

            if (*reinterpret_cast<volatile unsigned int*>(&a.ctl->budget[round & 1])) {
                // ---- 3b. the round budget: the recorded preemptors in pod order, their victims counted per job
                if (b == 0 && warp == 0)
                    for (long long g0 = g_lo; g0 < g_hi; g0 += 32) {
                        const long long gl = g0 + lane;
                        const bool waiting = gl < g_hi && __ldcg(ga.pre + gl) == 1u;
                        for (unsigned int mb = __ballot_sync(0xffffffffu, waiting); mb; mb &= mb - 1u) {
                            const long long g = g0 + __ffs(mb) - 1;
                            const long long h0 = __ldg(a.noff + (__ldcg(a.choice + g) & 0x7fffffffull));
                            bool over = false;
#pragma unroll
                            for (int i = 0; i < 4; ++i)
                                if ((__ldcg(ga.vmask + 4 * g + i) >> lane) & 1u) {
                                    const int32_t r = __ldg(ga.rgang + h0 + lane + 32 * i);
                                    if (r >= 0)
                                        over |= atomicAdd(ga.used + r, 1) >= __ldcg(ga.alive + r) - __ldg(ga.rgmin + r);
                                }
                            if (!__any_sync(0xffffffffu, over) && lane == 0) ga.pre[g] = 2u;
                        }
                    }
                if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;

                // ---- 3c. apply the preemptors that passed, one warp per pod; the others are deferred
                unsigned int deferred = 0, committed = 0;
                for (long long g = g_lo + wfirst; g < g_hi; g += wstride) {
                    const unsigned int st = __ldcg(ga.pre + g);
                    if (st == 0u) continue;
                    const int n = static_cast<int>(__ldcg(a.choice + g) & 0x7fffffffull);
                    const long long h0 = __ldg(a.noff + n);
                    unsigned int in_v = 0;
#pragma unroll
                    for (int i = 0; i < 4; ++i) in_v |= ((__ldcg(ga.vmask + 4 * g + i) >> lane) & 1u) << i;
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        if ((in_v >> i) & 1u) {
                            const int32_t r = __ldg(ga.rgang + h0 + lane + 32 * i);
                            if (r >= 0) {
                                ga.used[r] = 0;
                                if (st == 2u) atomicSub(ga.alive + r, 1);
                            }
                            if (st == 2u) a.evicted[h0 + lane + 32 * i] = static_cast<int32_t>(g);
                        }
                    if (lane == 0) ga.pre[g] = 0u;
                    if (st != 2u) {
                        deferred += lane == 0;
                        continue;
                    }
                    const int rows = __ldg(a.dv + n);
                    WarpTab t = load_tab(a, n, rows);
#pragma unroll
                    for (int i = 0; i < 4; ++i)
                        for (unsigned int m = __ballot_sync(0xffffffffu, (in_v >> i) & 1u); m; m &= m - 1u)
                            add_running(a, t, h0 + (__ffs(m) - 1) + 32 * i, 1);
                    const int32_t c0 = __ldg(a.off + g), len = __ldg(a.off + g + 1) - c0;
                    const unsigned long long cdev = __ldcg(ga.vdev + g);
                    for (int k = 0; k < len; ++k) {
                        const int d = static_cast<int>((cdev >> (6 * k)) & 63u);
#pragma unroll
                        for (int i = 0; i < 2; ++i)
                            if (d == lane + 32 * i) {
                                t.c[i] -= __ldg(a.rc + c0 + k);
                                t.m[i] -= __ldg(a.rm + c0 + k);
                            }
                    }
                    const size_t off = static_cast<size_t>(n) * D;
#pragma unroll
                    for (int i = 0; i < 2; ++i)
                        if (lane + 32 * i < rows) {
                            a.fc_out[off + lane + 32 * i] = t.c[i];
                            a.fm_out[off + lane + 32 * i] = t.m[i];
                        }
                    if (lane == 0) a.node[g] = n;
                    if (lane < len) a.dev[c0 + lane] = static_cast<int8_t>((cdev >> (6 * lane)) & 63u);
                    committed += lane == 0;
                }
                if (deferred) atomicAdd(&a.ctl->deferred[round & 1], deferred);
                if (committed) atomicAdd(ga.committed + gang, committed);
                if (!grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
            }

            // ---- 4. end the gang, or run another round
            const unsigned int pending = *reinterpret_cast<volatile unsigned int*>(&a.ctl->deferred[round & 1]);
            const long long placed = __ldcg(ga.committed + gang);
            gang_done = pending == 0u || placed + pending < need;
            if (!gang_done) continue;
            if (placed >= need) {
                if (b == 0 && tid == 0) ga.placed[gang] = static_cast<int32_t>(placed);
                break;  // nothing is pending: the next gang reads only what the barriers before published
            }
            // give the gang back: its pods' demand, and every running pod it evicted
            give_back_pods(a, g_lo, g_hi, first, stride);
            for (long long n = wfirst; n < N; n += wstride)
                for (long long h = __ldg(a.noff + n) + lane, h1 = __ldg(a.noff + n + 1); h < h1; h += 32) {
                    const int32_t e = __ldcg(a.evicted + h);
                    if (e < g_lo || e >= g_hi) continue;
                    a.evicted[h] = -1;
                    for (int32_t c = __ldg(a.roff + h), c1 = __ldg(a.roff + h + 1); c < c1; ++c) {
                        const size_t at = static_cast<size_t>(n) * D + __ldg(a.qd + c);
                        atomicSub(a.fc_out + at, __ldg(a.qc + c));
                        atomicSub(a.fm_out + at, __ldg(a.qm + c));
                    }
                    const int32_t r = __ldg(ga.rgang + h);
                    if (r >= 0) atomicAdd(ga.alive + r, 1);
                }
            if (gang + 1 < ga.J && !grid_barrier(&a.ctl->bar, &a.ctl->timeouts, gen, &sOk)) goto finish;
        }
    }
    done = true;
finish:
    if (b == 0 && tid == 0) {
        const bool bad = *reinterpret_cast<volatile unsigned int*>(&a.ctl->bad_index) != 0u;
        a.info[0] = bad ? 0 : round;
        a.info[1] = done ? 0 : 1;
        a.info[2] = bad ? 1 : 0;
    }
}

size_t preempt_gangs_scratch_bytes(int N, int G, int J, int R) { return PreemptScratch(N, G, J, R).total; }

cudaError_t preempt_gangs_launch(const int32_t* free_core, const int32_t* free_mem, const int32_t* d_valid, int N,
                                 int D, const int32_t* req_core, const int32_t* req_mem, int P,
                                 const int32_t* pod_offsets, int G, const int32_t* gang_offsets, const int32_t* gang_min,
                                 const int32_t* gang_prio, int J, const int32_t* run_core, const int32_t* run_mem,
                                 const int8_t* run_dev, int Q, const int32_t* run_offsets, const int32_t* run_prio,
                                 int H, const int32_t* node_offsets, const int32_t* run_gang,
                                 const int32_t* run_gang_min, int R, int32_t* out_node, int8_t* out_dev,
                                 int32_t* out_placed, int32_t* out_evicted, int32_t* free_core_out,
                                 int32_t* free_mem_out, int32_t* info, void* scratch, int device, cudaStream_t stream) {
    const PreemptScratch L(N, G, J, R);
    char* s = static_cast<char*>(scratch);
    PreGangsArgs ga{};
    PreemptArgs& a = ga.p;
    a.fc = free_core; a.fm = free_mem; a.dv = d_valid; a.rc = req_core; a.rm = req_mem; a.off = pod_offsets;
    a.qc = run_core; a.qm = run_mem; a.qd = run_dev; a.roff = run_offsets; a.rprio = run_prio; a.noff = node_offsets;
    a.N = N; a.D = D; a.P = P; a.G = G; a.Q = Q; a.H = H;
    a.node = out_node; a.dev = out_dev; a.evicted = out_evicted; a.fc_out = free_core_out; a.fm_out = free_mem_out;
    a.info = info;
    ga.goff = gang_offsets; ga.gmin = gang_min; ga.gprio = gang_prio; ga.rgang = run_gang; ga.rgmin = run_gang_min;
    ga.J = J; ga.R = R;
    ga.placed = out_placed;
    ga.pre = reinterpret_cast<unsigned int*>(s + L.pre);
    ga.in_domain = reinterpret_cast<unsigned int*>(s + L.in_domain);
    ga.committed = reinterpret_cast<unsigned int*>(s + L.committed);
    ga.alive = reinterpret_cast<int32_t*>(s + L.alive);
    ga.used = reinterpret_cast<int32_t*>(s + L.used);
    ga.vdev = reinterpret_cast<unsigned long long*>(s + L.vdev);
    ga.vmask = reinterpret_cast<unsigned int*>(s + L.vmask);
    ga.cap = reinterpret_cast<unsigned int*>(s + L.cap);
    const cudaError_t err = preempt_scratch(a, scratch, L, stream);
    if (err != cudaSuccess) return err;
    // Grid: as preempt_launch, from N and G alone (the gang sizes are device data): no more CTAs than a round over
    // all G pods has choose items; at least one, which finds G = 0's offsets bad.
    return coop_launch<preempt_gangs_kernel>(ga, static_cast<long long>(L.K) * G, device, stream);
}

}  // namespace egpu

// egpu_prefalloc.cu — GetPreferredAllocation for every container request of a PreferredAllocationRequest
// in one call (egpu_preferred_allocation_batch, include/egpu_plugin.h), from flat ID buffers, with all ID
// work on the GPU.  The answers are those of egpu_preferred_allocation (egpu_plugin.cc) on the same
// strings, return codes and their precedence included.
//
//   parse    one thread per ID: its set (binary search in the set offsets), "%d-%02d" -> (gpu, unit)
//            (egpu_id_grammar.h, the host codec's grammar), the first bad available ID of every request
//            (atomicMin of position << 2 | code), per-(request, GPU) counts (warp-aggregated atomics),
//            must-include keys into the request's region of an open-addressing table
//   lookup   one thread per available ID: the first position of every must-include key (atomicMin)
//   must     one thread per must-include ID: the first failure, the first index of every pinned GPU and
//            the distinct must-include IDs per GPU
//   choose   one warp per request (lane = GPU, two per lane): the return-code precedence, the pins in
//            order, the best fit of spec 2.3 pick by pick, how many IDs every chosen GPU gives
//   sort     the identity pipeline's stable LSD radix sort, first on (gpu << 50 | unit) - must-include
//            IDs keep key 0, i.e. their order - then on the set index: every available list ends up in
//            (gpu, unit, position) order inside its own range
//   flag, scan, emit   which sorted entries are given, their rank inside their (request, GPU) run, and
//            one thread per entry writes its position (or -1 for a request that failed)
// The host reads only the 2 n_req + 1 set offsets, the sizes and the buffer length; the n_ids-long
// arrays go to the copy engine.
#include <algorithm>
#include <cstring>
#include <vector>

#include "../../include/egpu_plugin.h"
#include "egpu_ctx.h"
#include "egpu_id_grammar.h"

namespace egpu {

constexpr int kUnitBits = 50;                        // 15 decimal digits < 2^50
constexpr int kKeyDigits = (kUnitBits + 6 + 3) / 4;  // 4-bit digits of gpu << 50 | unit (gpu < 64)
constexpr int kSetDigits = 5;                        // set index < 2 * EGPU_PREFALLOC_MAX_REQUESTS + 1 <= 16^5
static_assert(2ll * EGPU_PREFALLOC_MAX_REQUESTS + 1 <= (1ll << (4 * kSetDigits)), "set digits");
constexpr unsigned long long kNoKey = ~0ull;
constexpr uint32_t kNone = 0xffffffffu;
constexpr int32_t kSlotMalformed = -2;  // slot_of of a malformed must-include ID (-1: not in the table)

struct PaReq {
    long long a0, m0;          // first available / must-include ID (global index)
    long long out_off;         // first answer slot on the device
    long long hash_off;        // the request's region of the must-include table
    uint32_t hash_mask;        // region size - 1 (0: no must-include IDs)
    int32_t n_av, n_must, size;
    int32_t w;                 // answer slots on the device: size when 0 <= size <= n_av, else 0
};

__device__ __forceinline__ unsigned long long mix64(unsigned long long x) {
    x ^= x >> 33;
    x *= 0xff51afd7ed558ccdull;
    x ^= x >> 33;
    x *= 0xc4ceb9fe1a85ec53ull;
    x ^= x >> 33;
    return x;
}

__device__ __forceinline__ long long find_slot(const unsigned long long* skey, const PaReq& r, unsigned long long k) {
    uint32_t h = static_cast<uint32_t>(mix64(k)) & r.hash_mask;
    for (;;) {  // the region is at most half full: the probe ends
        const unsigned long long v = skey[r.hash_off + h];
        if (v == k) return r.hash_off + h;
        if (v == kNoKey) return -1;
        h = (h + 1) & r.hash_mask;
    }
}

__global__ void __launch_bounds__(256)
pa_parse_kernel(const char* __restrict__ flat, long long flat_bytes, const long long* __restrict__ id_off, long long n,
                const long long* __restrict__ set_off, long long n_sets, const PaReq* __restrict__ req,
                unsigned long long* __restrict__ gu, uint32_t* __restrict__ set_of, int32_t* __restrict__ slot_of,
                unsigned long long* __restrict__ key, uint32_t* __restrict__ val, unsigned long long* __restrict__ first_bad,
                uint32_t* __restrict__ cnt, unsigned long long* __restrict__ skey, uint32_t* __restrict__ smk) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    uint32_t count_at = kNone;  // (request, GPU) cell this ID counts in
    if (i < n) {
        long long lo = 0, hi = n_sets;  // the last s with set_off[s] <= i (empty sets share their offset)
        while (hi - lo > 1) {
            const long long mid = (lo + hi) >> 1;
            if (set_off[mid] <= i) lo = mid; else hi = mid;
        }
        const uint32_t s = static_cast<uint32_t>(lo);
        const PaReq r = req[s >> 1];
        const long long b = id_off[i], e = id_off[i + 1];
        int32_t g = 0;
        int64_t u = 0;
        const bool ok = b >= 0 && b <= e && e <= flat_bytes && egpu_id_grammar(flat + b, e - b, &g, &u) == 0;
        const unsigned long long k = ok && g < kMaxD ? (static_cast<unsigned long long>(g) << kUnitBits) | static_cast<unsigned long long>(u)
                                                     : kNoKey;
        gu[i] = k;
        set_of[i] = s;
        val[i] = static_cast<uint32_t>(i);
        if (!(s & 1)) {
            key[i] = k == kNoKey ? 0ull : k;
            if (k == kNoKey)
                atomicMin(&first_bad[s >> 1], (static_cast<unsigned long long>(i - r.a0) << 2) | (ok ? 2ull : 1ull));
            else
                count_at = (s >> 1) * kMaxD + static_cast<uint32_t>(g);
        } else {
            key[i] = 0ull;  // must-include IDs keep their order through the sort
            int32_t slot = ok ? -1 : kSlotMalformed;
            if (k != kNoKey) {
                uint32_t h = static_cast<uint32_t>(mix64(k)) & r.hash_mask;
                for (;;) {
                    const unsigned long long prev = atomicCAS(&skey[r.hash_off + h], kNoKey, k);
                    if (prev == kNoKey || prev == k) break;
                    h = (h + 1) & r.hash_mask;
                }
                slot = static_cast<int32_t>(r.hash_off + h);
                atomicMin(&smk[slot], static_cast<uint32_t>(i - r.m0));
            }
            slot_of[i] = slot;
        }
    }
    // the IDs of one GPU usually sit together: one atomic per (request, GPU) per warp
    const unsigned peers = __match_any_sync(0xffffffffu, count_at);
    if (count_at != kNone && static_cast<int>(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&cnt[count_at], __popc(peers));
}

__global__ void __launch_bounds__(256)
pa_lookup_kernel(long long n, const uint32_t* __restrict__ set_of, const PaReq* __restrict__ req,
                 const unsigned long long* __restrict__ gu, const unsigned long long* __restrict__ skey,
                 uint32_t* __restrict__ sval, int32_t* __restrict__ slot_of) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = set_of[i];
    if (s & 1) return;
    const PaReq r = req[s >> 1];
    const unsigned long long k = gu[i];
    long long slot = -1;
    if (r.hash_mask && k != kNoKey) slot = find_slot(skey, r, k);
    if (slot >= 0) atomicMin(&sval[slot], static_cast<uint32_t>(i - r.a0));
    slot_of[i] = static_cast<int32_t>(slot);
}

__global__ void __launch_bounds__(256)
pa_must_kernel(long long n, const uint32_t* __restrict__ set_of, const PaReq* __restrict__ req,
               const unsigned long long* __restrict__ gu, const int32_t* __restrict__ slot_of,
               const uint32_t* __restrict__ sval, const uint32_t* __restrict__ smk, unsigned long long* __restrict__ must_bad,
               uint32_t* __restrict__ pin_first, uint32_t* __restrict__ mcnt) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = set_of[i];
    if (!(s & 1)) return;
    const uint32_t q = s >> 1;
    const uint32_t k = static_cast<uint32_t>(i - req[q].m0);
    const int32_t slot = slot_of[i];
    if (slot == kSlotMalformed) {
        atomicMin(&must_bad[q], (static_cast<unsigned long long>(k) << 2) | 1ull);  // PARSE
        return;
    }
    if (slot < 0 || sval[slot] == kNone) {
        atomicMin(&must_bad[q], (static_cast<unsigned long long>(k) << 2) | 2ull);  // not available: UNSAT
        return;
    }
    const uint32_t g = static_cast<uint32_t>(gu[i] >> kUnitBits);
    atomicMin(&pin_first[q * kMaxD + g], k);
    if (smk[slot] == k) atomicAdd(&mcnt[q * kMaxD + g], 1u);  // the first listing of this ID
}

constexpr int kChooseWarps = 4;

__global__ void __launch_bounds__(32 * kChooseWarps)
pa_choose_kernel(const PaReq* __restrict__ req, long long n_req, int resource, const unsigned long long* __restrict__ first_bad,
                 const unsigned long long* __restrict__ must_bad, const uint32_t* __restrict__ pin_first,
                 const uint32_t* __restrict__ cnt, const uint32_t* __restrict__ mcnt, int32_t* __restrict__ rc_out,
                 int32_t* __restrict__ gpu_out, uint32_t* __restrict__ e_cnt, uint32_t* __restrict__ e_base,
                 uint32_t* __restrict__ run_start) {
    __shared__ int pins[kChooseWarps][kMaxD];
    __shared__ int chosen[kChooseWarps][kMaxD];
    __shared__ uint32_t ecs[kChooseWarps][kMaxD], ebs[kChooseWarps][kMaxD];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long q = static_cast<long long>(blockIdx.x) * kChooseWarps + warp;
    if (q >= n_req) return;  // whole warps
    const unsigned full = 0xffffffffu;
    const PaReq r = req[q];
    const int d0 = lane, d1 = lane + 32;
    const uint32_t c0 = cnt[q * kMaxD + d0], c1 = cnt[q * kMaxD + d1];
    const uint32_t mc0 = mcnt[q * kMaxD + d0], mc1 = mcnt[q * kMaxD + d1];
    {   // start of every GPU's run in the sorted available list: exclusive prefix of the counts
        uint32_t x0 = c0, x1 = c1;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y0 = __shfl_up_sync(full, x0, o), y1 = __shfl_up_sync(full, x1, o);
            if (lane >= o) x0 += y0, x1 += y1;
        }
        const uint32_t total0 = __shfl_sync(full, x0, 31);
        run_start[q * kMaxD + d0] = x0 - c0;
        run_start[q * kMaxD + d1] = total0 + x1 - c1;
    }
    ecs[warp][d0] = ecs[warp][d1] = 0;
    ebs[warp][d0] = ebs[warp][d1] = 0;
    const bool core = resource == EGPU_RESOURCE_CORE;
    const bool whole = core && r.size > EGPU_CORE_MAX;
    const long long n_gpus = whole ? r.size / EGPU_CORE_MAX : 1;
    const unsigned long long fb = first_bad[q];
    int code = EGPU_OK;
    int n_chosen = 0;
    if (r.size < 0) {
        code = EGPU_ERR_INVALID;
    } else if (r.n_must > r.size) {
        code = EGPU_ERR_UNSAT;
    } else if (fb != kNoKey) {
        code = (fb & 3) == 1 ? EGPU_ERR_PARSE : EGPU_ERR_INVALID;
    } else if (r.n_av == 0) {
        code = r.size == 0 ? EGPU_OK : EGPU_ERR_UNSAT;
    } else if (whole && r.size % EGPU_CORE_MAX != 0) {
        code = EGPU_ERR_UNSAT;
    } else {
        // must-include: pins are the GPUs of the IDs before the first failure, in order of first listing
        const unsigned long long mb = must_bad[q];
        const uint32_t kb = mb == kNoKey ? kNone : static_cast<uint32_t>(mb >> 2);
        const uint32_t p0 = pin_first[q * kMaxD + d0], p1 = pin_first[q * kMaxD + d1];
        const bool in0 = p0 < kb, in1 = p1 < kb;
        const unsigned lo_pins = __ballot_sync(full, in0), hi_pins = __ballot_sync(full, in1);
        const int n_pins = __popc(lo_pins) + __popc(hi_pins);
        int rank0 = 0, rank1 = 0;
        for (int t = 0; t < 32; ++t) {
            const uint32_t x0 = __shfl_sync(full, p0, t), x1 = __shfl_sync(full, p1, t);
            const bool y0 = (lo_pins >> t) & 1, y1 = (hi_pins >> t) & 1;
            rank0 += (y0 && x0 < p0) + (y1 && x1 < p0);
            rank1 += (y0 && x0 < p1) + (y1 && x1 < p1);
        }
        if (in0) pins[warp][rank0] = d0;
        if (in1) pins[warp][rank1] = d1;
        __syncwarp();
        if (n_pins > n_gpus) {
            code = EGPU_ERR_UNSAT;  // spans more GPUs than the request takes
        } else if (mb != kNoKey) {
            code = (mb & 3) == 1 ? EGPU_ERR_PARSE : EGPU_ERR_UNSAT;
        } else {
            // the availability table of egpu_plugin.cc: usable rows, the other dimension at its cap,
            // request (size, 1) or (1, size); whole cards: one full card per pick, pinned cards first
            const unsigned lo_has = __ballot_sync(full, c0 > 0), hi_has = __ballot_sync(full, c1 > 0);
            const int D = hi_has ? 64 - __clz(hi_has) : 32 - __clz(lo_has);
            const unsigned long long pin_mask = (static_cast<unsigned long long>(hi_pins) << 32) | lo_pins;
            const int32_t cap = core ? EGPU_CORE_MAX : EGPU_MEM_MAX;
            const int32_t rq_core = core ? (whole ? EGPU_CORE_MAX : r.size) : 1;
            const int32_t rq_mem = core ? 1 : r.size;
            const bool in_domain = rq_core <= EGPU_CORE_MAX && rq_mem <= EGPU_MEM_MAX;  // spec 2.2
            unsigned long long taken = 0;
            for (long long pick = 0; pick < n_gpus; ++pick) {  // ends after at most D + 1 picks
                const int pin = pick < n_pins ? pins[warp][pick] : -1;
                uint32_t best = kNone;
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int d = h ? d1 : d0;
                    const int32_t c = static_cast<int32_t>(min(h ? c1 : c0, static_cast<uint32_t>(cap)));
                    const bool later_pin = pin < 0 && ((pin_mask >> d) & 1);
                    const bool usable = d < D && !((taken >> d) & 1) && !later_pin && (pin < 0 || d == pin);
                    const int32_t fc = core ? (usable ? c : 0) : (usable ? EGPU_CORE_MAX : 0);
                    const int32_t fm = core ? (usable ? EGPU_MEM_MAX : 0) : (usable ? c : 0);
                    if (in_domain && rq_core <= fc && rq_mem <= fm)
                        best = min(best, (static_cast<uint32_t>(fc - rq_core) << 24) | (static_cast<uint32_t>(fm - rq_mem) << 6) |
                                             static_cast<uint32_t>(d));
                }
                best = __reduce_min_sync(full, best);
                if (best == kNone) {
                    code = EGPU_ERR_UNSAT;
                    break;
                }
                const int g = static_cast<int>(best & 63u);
                taken |= 1ull << g;
                if (lane == 0) chosen[warp][n_chosen] = g;
                ++n_chosen;
            }
            __syncwarp();
            if (code == EGPU_OK) {
                // must-include IDs first, then every chosen GPU's lowest units: how many each gives
                uint32_t n_out = __reduce_add_sync(full, mc0 + mc1);
                if (lane == 0) {
                    const uint32_t want = whole ? EGPU_CORE_MAX : static_cast<uint32_t>(r.size);
                    for (int j = 0; j < n_chosen; ++j) {
                        const int g = chosen[warp][j];
                        const uint32_t have = mcnt[q * kMaxD + g];
                        const uint32_t cand = cnt[q * kMaxD + g] - have;
                        const uint32_t need = want > have ? want - have : 0u;
                        const uint32_t e = min(min(cand, need), static_cast<uint32_t>(r.size) - n_out);
                        ecs[warp][g] = e;
                        ebs[warp][g] = n_out;
                        n_out += e;
                    }
                }
                n_out = __shfl_sync(full, n_out, 0);
                if (n_out != static_cast<uint32_t>(r.size)) code = EGPU_ERR_UNSAT;
            }
        }
    }
    __syncwarp();
    const bool ok = code == EGPU_OK;
    e_cnt[q * kMaxD + d0] = ok ? ecs[warp][d0] : 0u;
    e_cnt[q * kMaxD + d1] = ok ? ecs[warp][d1] : 0u;
    e_base[q * kMaxD + d0] = ebs[warp][d0];
    e_base[q * kMaxD + d1] = ebs[warp][d1];
    if (lane == 0) {
        rc_out[q] = code;
        gpu_out[q] = ok && n_chosen > 0 ? chosen[warp][0] : -1;
    }
}

// between the two sorts: the key becomes the set index (the order of the first sort is kept inside a set)
__global__ void __launch_bounds__(256)
pa_rekey_kernel(long long n, const uint32_t* __restrict__ val, const uint32_t* __restrict__ set_of, unsigned long long* __restrict__ key) {
    const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j < n) key[j] = set_of[val[j]];
}

// sorted entry j is given: a must-include ID at its first listing, or an available ID that is not the
// first position of a must-include ID (requests that failed give nothing)
__global__ void __launch_bounds__(256)
pa_flag_kernel(long long n, const uint32_t* __restrict__ val, const uint32_t* __restrict__ set_of, const PaReq* __restrict__ req,
               const int32_t* __restrict__ rc, const int32_t* __restrict__ slot_of, const uint32_t* __restrict__ sval,
               const uint32_t* __restrict__ smk, uint32_t* __restrict__ flag) {
    const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t i = val[j], s = set_of[i];
    uint32_t f = 0;
    if (rc[s >> 1] == EGPU_OK) {
        const PaReq& r = req[s >> 1];
        const int32_t slot = slot_of[i];
        if (s & 1)
            f = slot >= 0 && smk[slot] == static_cast<uint32_t>(i - r.m0);
        else
            f = !(slot >= 0 && sval[slot] == static_cast<uint32_t>(i - r.a0));
    }
    flag[j] = f;
}

__global__ void __launch_bounds__(256)
pa_emit_kernel(long long n, const uint32_t* __restrict__ val, const uint32_t* __restrict__ set_of, const PaReq* __restrict__ req,
               const int32_t* __restrict__ rc, const unsigned long long* __restrict__ gu, const int32_t* __restrict__ slot_of,
               const uint32_t* __restrict__ sval, const uint32_t* __restrict__ flag, const unsigned long long* __restrict__ rank,
               const uint32_t* __restrict__ e_cnt, const uint32_t* __restrict__ e_base, const uint32_t* __restrict__ run_start,
               int32_t* __restrict__ out) {
    const long long j = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (j >= n) return;
    const uint32_t i = val[j], s = set_of[i], q = s >> 1;
    const PaReq& r = req[q];
    const bool ok = rc[q] == EGPU_OK;
    if (s & 1) {  // must-include IDs first, in their order, once each
        if (ok && flag[j]) out[r.out_off + static_cast<long long>(rank[j] - rank[r.m0])] = static_cast<int32_t>(sval[slot_of[i]]);
        return;
    }
    const long long p = static_cast<long long>(i) - r.a0;
    if (!ok) {
        if (p < r.w) out[r.out_off + p] = -1;
        return;
    }
    if (!flag[j]) return;
    const uint32_t cell = q * kMaxD + static_cast<uint32_t>(gu[i] >> kUnitBits);
    const unsigned long long k = rank[j] - rank[r.a0 + run_start[cell]];
    if (k < e_cnt[cell]) out[r.out_off + e_base[cell] + static_cast<long long>(k)] = static_cast<int32_t>(p);
}

}  // namespace egpu

using namespace egpu;

extern "C" int egpu_preferred_allocation_batch(egpu_ctx* ctx, int resource, const char* ids_flat, const int64_t* id_offsets,
                                               int64_t n_ids, const int64_t* set_offsets, int64_t n_req,
                                               const int32_t* allocation_size, int32_t* out_positions, int32_t* out_gpu,
                                               int32_t* out_rc) {
    if (!ctx || n_ids < 0 || n_req < 0 || n_ids > 0x7fffffffll || n_req > EGPU_PREFALLOC_MAX_REQUESTS) return EGPU_ERR_INVALID;
    if (resource != EGPU_RESOURCE_CORE && resource != EGPU_RESOURCE_MEM) return EGPU_ERR_INVALID;
    if (n_req == 0) return n_ids == 0 ? EGPU_OK : EGPU_ERR_INVALID;
    if (!set_offsets || !allocation_size || !out_rc || (n_ids > 0 && !id_offsets)) return EGPU_ERR_INVALID;
    const int64_t n_sets = 2 * n_req;
    if (set_offsets[0] != 0 || set_offsets[n_sets] != n_ids) return EGPU_ERR_INVALID;
    for (int64_t s = 0; s < n_sets; ++s)
        if (set_offsets[s + 1] < set_offsets[s]) return EGPU_ERR_INVALID;
    const int64_t flat_bytes = n_ids > 0 ? id_offsets[n_ids] : 0;
    if (flat_bytes < 0 || (flat_bytes > 0 && !ids_flat)) return EGPU_ERR_INVALID;

    // per-request layout: answer slots (caller's and device's) and the must-include table regions
    std::vector<PaReq> req(static_cast<size_t>(n_req));
    int64_t total_out = 0, dev_out = 0, hash_slots = 0;
    for (int64_t q = 0; q < n_req; ++q) {
        PaReq& r = req[static_cast<size_t>(q)];
        r.a0 = set_offsets[2 * q];
        r.m0 = set_offsets[2 * q + 1];
        r.n_av = static_cast<int32_t>(r.m0 - r.a0);
        r.n_must = static_cast<int32_t>(set_offsets[2 * q + 2] - r.m0);
        r.size = allocation_size[q];
        total_out += std::max<int32_t>(r.size, 0);
        r.w = r.size >= 0 && r.size <= r.n_av ? r.size : 0;
        r.out_off = dev_out;
        dev_out += r.w;
        r.hash_off = hash_slots;
        r.hash_mask = 0;
        if (r.n_must > 0) {
            int64_t h = 2;
            while (h < 2 * static_cast<int64_t>(r.n_must)) h <<= 1;
            r.hash_mask = static_cast<uint32_t>(h - 1);
            hash_slots += h;
        }
    }
    if (total_out > 0 && !out_positions) return EGPU_ERR_INVALID;

    std::lock_guard<std::mutex> lock(ctx->mu);
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    cudaStream_t s = ctx->stream;
    const size_t n = static_cast<size_t>(n_ids), nr = static_cast<size_t>(n_req), cells = nr * kMaxD;
    const size_t H = static_cast<size_t>(hash_slots > 0 ? hash_slots : 1);
    // scratch: the context's grow-only arena (shared with the identity pipeline), sized before any work
    void *flat = nullptr, *id_off = nullptr, *set_off = nullptr, *d_req = nullptr, *gu = nullptr, *set_of = nullptr,
         *slot_of = nullptr, *key_a = nullptr, *key_b = nullptr, *val_a = nullptr, *val_b = nullptr, *flag = nullptr,
         *rank = nullptr, *blk = nullptr, *hist = nullptr, *first_bad = nullptr, *must_bad = nullptr, *pin_first = nullptr,
         *cnt = nullptr, *mcnt = nullptr, *rc = nullptr, *gpu = nullptr, *e_cnt = nullptr, *e_base = nullptr,
         *run_start = nullptr, *skey = nullptr, *sval = nullptr, *smk = nullptr, *out = nullptr;
    const ArenaWant wants[] = {
        {&flat, static_cast<size_t>(flat_bytes)}, {&id_off, 8 * (n + 1)}, {&set_off, 8 * (static_cast<size_t>(n_sets) + 1)},
        {&d_req, sizeof(PaReq) * nr}, {&gu, 8 * n}, {&set_of, 4 * n}, {&slot_of, 4 * n}, {&key_a, 8 * n}, {&key_b, 8 * n},
        {&val_a, 4 * n}, {&val_b, 4 * n}, {&flag, 4 * n}, {&rank, 8 * (n + 1)}, {&blk, 8 * ((n + 1023) / 1024 + 1)},
        {&hist, 4 * radix_hist_words(n_ids)}, {&first_bad, 8 * nr}, {&must_bad, 8 * nr}, {&pin_first, 4 * cells},
        {&cnt, 4 * cells}, {&mcnt, 4 * cells}, {&rc, 4 * nr}, {&gpu, 4 * nr}, {&e_cnt, 4 * cells}, {&e_base, 4 * cells},
        {&run_start, 4 * cells}, {&skey, 8 * H}, {&sval, 4 * H}, {&smk, 4 * H}, {&out, 4 * static_cast<size_t>(dev_out)}};
    EGPU_CUDA(ctx, arena_carve(ctx, wants, sizeof wants / sizeof wants[0]));
    // the per-request state and the must-include table start empty: 0xff.. = "none" for the minima and keys
    EGPU_CUDA(ctx, cudaMemsetAsync(first_bad, 0xff, 8 * nr, s));
    EGPU_CUDA(ctx, cudaMemsetAsync(must_bad, 0xff, 8 * nr, s));
    EGPU_CUDA(ctx, cudaMemsetAsync(pin_first, 0xff, 4 * cells, s));
    EGPU_CUDA(ctx, cudaMemsetAsync(cnt, 0, 4 * cells, s));
    EGPU_CUDA(ctx, cudaMemsetAsync(mcnt, 0, 4 * cells, s));
    EGPU_CUDA(ctx, cudaMemsetAsync(skey, 0xff, 8 * H, s));
    EGPU_CUDA(ctx, cudaMemsetAsync(sval, 0xff, 4 * H, s));
    EGPU_CUDA(ctx, cudaMemsetAsync(smk, 0xff, 4 * H, s));
    if (flat_bytes) EGPU_CUDA(ctx, cudaMemcpyAsync(flat, ids_flat, static_cast<size_t>(flat_bytes), cudaMemcpyHostToDevice, s));
    if (n) EGPU_CUDA(ctx, cudaMemcpyAsync(id_off, id_offsets, 8 * (n + 1), cudaMemcpyHostToDevice, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(set_off, set_offsets, 8 * (static_cast<size_t>(n_sets) + 1), cudaMemcpyHostToDevice, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(d_req, req.data(), sizeof(PaReq) * nr, cudaMemcpyHostToDevice, s));

    const PaReq* R = static_cast<const PaReq*>(d_req);
    const unsigned nb = static_cast<unsigned>((n_ids + 255) / 256);
    auto u64 = [](void* p) { return static_cast<unsigned long long*>(p); };
    auto u32 = [](void* p) { return static_cast<uint32_t*>(p); };
    auto i32 = [](void* p) { return static_cast<int32_t*>(p); };
    if (n) {
        pa_parse_kernel<<<nb, 256, 0, s>>>(static_cast<const char*>(flat), flat_bytes, static_cast<const long long*>(id_off), n_ids,
                                          static_cast<const long long*>(set_off), n_sets, R, u64(gu), u32(set_of), i32(slot_of),
                                          u64(key_a), u32(val_a), u64(first_bad), u32(cnt), u64(skey), u32(smk));
        pa_lookup_kernel<<<nb, 256, 0, s>>>(n_ids, u32(set_of), R, u64(gu), u64(skey), u32(sval), i32(slot_of));
        pa_must_kernel<<<nb, 256, 0, s>>>(n_ids, u32(set_of), R, u64(gu), i32(slot_of), u32(sval), u32(smk), u64(must_bad),
                                         u32(pin_first), u32(mcnt));
        ctx->launches += 3;
    }
    pa_choose_kernel<<<static_cast<unsigned>((n_req + kChooseWarps - 1) / kChooseWarps), 32 * kChooseWarps, 0, s>>>(
        R, n_req, resource, u64(first_bad), u64(must_bad), u32(pin_first), u32(cnt), u32(mcnt), i32(rc), i32(gpu), u32(e_cnt),
        u32(e_base), u32(run_start));
    ctx->launches += 1;
    if (n) {
        unsigned long long *ka = u64(key_a), *kb = u64(key_b);
        uint32_t *va = u32(val_a), *vb = u32(val_b);
        ctx->launches += radix_sort_pairs(s, ka, va, kb, vb, n_ids, kKeyDigits, u32(hist));
        pa_rekey_kernel<<<nb, 256, 0, s>>>(n_ids, va, u32(set_of), ka);
        ctx->launches += 1;
        ctx->launches += radix_sort_pairs(s, ka, va, kb, vb, n_ids, kSetDigits, u32(hist));
        pa_flag_kernel<<<nb, 256, 0, s>>>(n_ids, va, u32(set_of), R, i32(rc), i32(slot_of), u32(sval), u32(smk), u32(flag));
        ctx->launches += 1;
        ctx->launches += exclusive_scan_u32(s, u32(flag), n_ids, u64(blk), u64(rank));
        pa_emit_kernel<<<nb, 256, 0, s>>>(n_ids, va, u32(set_of), R, i32(rc), u64(gu), i32(slot_of), u32(sval), u32(flag), u64(rank),
                                         u32(e_cnt), u32(e_base), u32(run_start), i32(out));
        ctx->launches += 1;
    }
    EGPU_CUDA(ctx, cudaGetLastError());
    std::vector<int32_t> h_gpu(nr);
    if (dev_out) EGPU_CUDA(ctx, cudaMemcpyAsync(out_positions, out, 4 * static_cast<size_t>(dev_out), cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(out_rc, rc, 4 * nr, cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(h_gpu.data(), gpu, 4 * nr, cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    ctx->prev_is_scan = false;
    if (out_gpu) std::memcpy(out_gpu, h_gpu.data(), 4 * nr);
    if (dev_out != total_out) {
        // requests larger than their available list have no device slots (they fail): move the answers to
        // the caller's layout, last request first (every answer only moves up), and fill those with -1
        int64_t off = total_out;
        for (int64_t q = n_req - 1; q >= 0; --q) {
            const PaReq& r = req[static_cast<size_t>(q)];
            const int32_t len = std::max<int32_t>(r.size, 0);
            off -= len;
            if (r.w == len)
                std::memmove(out_positions + off, out_positions + r.out_off, sizeof(int32_t) * static_cast<size_t>(len));
            else
                std::fill(out_positions + off, out_positions + off + len, -1);
        }
    }
    return EGPU_OK;
}

// egpu_plugin.cc — host logic between the kubelet device-plugin messages and the CUDA
// best-fit scan: ID codec ("%d-%02d", pkg/plugins/gpushare.go:28,163) and
// GetPreferredAllocation for one container (the stub at pkg/plugins/base.go:94-96).
// Plain C++; the device choice is delegated to egpu_bestfit_query (CUDA).
#include <algorithm>
#include <cstdio>
#include <cstring>
#include <string>
#include <unordered_map>
#include <utility>
#include <vector>

#include "../../include/egpu_plugin.h"
#include "egpu_id_grammar.h"

extern "C" {

int egpu_device_id_format(int32_t gpu, int64_t unit, char* out, int64_t cap) {
    if (!out || cap <= 0 || gpu < 0 || unit < 0) return EGPU_ERR_INVALID;
    const int n = std::snprintf(out, static_cast<size_t>(cap), "%d-%02lld", gpu, static_cast<long long>(unit));
    if (n < 0 || n >= cap) return EGPU_ERR_INVALID;
    return n;
}

int egpu_device_id_parse(const char* id, int32_t* gpu, int64_t* unit) {
    if (!id || !gpu || !unit) return EGPU_ERR_INVALID;
    // the grammar is shared with the device pipeline of egpu_preferred_allocation_batch
    return egpu_id_grammar(id, -1, gpu, unit) == 0 ? EGPU_OK : EGPU_ERR_PARSE;
}

int egpu_preferred_allocation(egpu_ctx* ctx, const char* const* available_ids, int64_t n_available,
                              const char* const* must_include_ids, int64_t n_must, int32_t allocation_size,
                              int resource, int32_t* out_positions, int32_t* out_gpu) {
    if (!ctx || n_available < 0 || n_must < 0 || allocation_size < 0) return EGPU_ERR_INVALID;
    if ((n_available > 0 && !available_ids) || (n_must > 0 && !must_include_ids)) return EGPU_ERR_INVALID;
    if (allocation_size > 0 && !out_positions) return EGPU_ERR_INVALID;
    if (resource != EGPU_RESOURCE_CORE && resource != EGPU_RESOURCE_MEM) return EGPU_ERR_INVALID;
    if (n_available > 0x7fffffffll) return EGPU_ERR_INVALID;
    if (n_must > allocation_size) return EGPU_ERR_UNSAT;

    // 1. IDs -> (gpu, unit); per-GPU availability = the free table of this request
    std::vector<int32_t> gpu_of(static_cast<size_t>(n_available));
    std::vector<int64_t> unit_of(static_cast<size_t>(n_available));
    int32_t D = 0;
    for (int64_t i = 0; i < n_available; ++i) {
        // the strings are wherever the caller's runtime put them: one cache miss each unless asked for early
        if (i + 16 < n_available) __builtin_prefetch(available_ids[i + 16]);
        const int rc = egpu_device_id_parse(available_ids[i], &gpu_of[i], &unit_of[i]);
        if (rc != EGPU_OK) return rc;
        if (gpu_of[i] >= EGPU_MAX_DEVICES) return EGPU_ERR_INVALID;
        D = std::max(D, gpu_of[i] + 1);
    }
    if (D == 0) return allocation_size == 0 ? EGPU_OK : EGPU_ERR_UNSAT;
    std::vector<int64_t> count(static_cast<size_t>(D), 0);
    for (int64_t i = 0; i < n_available; ++i) count[gpu_of[i]] += 1;

    // Whole-card requests (gpu-core only): more than 100 core units means allocation_size / 100 whole GPUs,
    // the reference's len/100 (pkg/plugins/gpushare.go:62-69); the size must then be a multiple of 100.
    const bool whole_cards = resource == EGPU_RESOURCE_CORE && allocation_size > EGPU_CORE_MAX;
    if (whole_cards && allocation_size % EGPU_CORE_MAX != 0) return EGPU_ERR_UNSAT;
    const int32_t n_gpus = whole_cards ? allocation_size / EGPU_CORE_MAX : 1;

    // 2. must-include IDs pin the GPU (whole-card requests: up to n_gpus GPUs)
    std::vector<int32_t> pinned;
    std::unordered_map<std::string, int32_t> pos_of;
    if (n_must > 0) {
        pos_of.reserve(static_cast<size_t>(n_available) * 2);
        for (int64_t i = 0; i < n_available; ++i) pos_of.emplace(available_ids[i], static_cast<int32_t>(i));
        for (int64_t k = 0; k < n_must; ++k) {
            int32_t g;
            int64_t u;
            const int rc = egpu_device_id_parse(must_include_ids[k], &g, &u);
            if (rc != EGPU_OK) return rc;
            if (pos_of.find(must_include_ids[k]) == pos_of.end()) return EGPU_ERR_UNSAT;  // kubelet promises must ⊆ available
            if (std::find(pinned.begin(), pinned.end(), g) == pinned.end()) pinned.push_back(g);
            if (static_cast<int32_t>(pinned.size()) > n_gpus) return EGPU_ERR_UNSAT;      // spans more GPUs than the request takes
        }
    }

    // 3. the choice: CUDA best-fit over the availability table.  One GPU per pick; a whole-card request
    //    makes n_gpus picks of a full card each, every pick against the table without the cards already
    //    taken (the sequential rule of the spec, DESIGN.md 2.6), pinned GPUs first.
    const int64_t cap_units = resource == EGPU_RESOURCE_CORE ? EGPU_CORE_MAX : EGPU_MEM_MAX;
    std::vector<int32_t> free_core(static_cast<size_t>(D)), free_mem(static_cast<size_t>(D));
    std::vector<int32_t> chosen;
    for (int32_t pick = 0; pick < n_gpus; ++pick) {
        const int32_t pin = pick < static_cast<int32_t>(pinned.size()) ? pinned[static_cast<size_t>(pick)] : -1;
        for (int32_t d = 0; d < D; ++d) {
            const int32_t c = static_cast<int32_t>(std::min<int64_t>(count[d], cap_units));
            const bool taken_card = std::find(chosen.begin(), chosen.end(), d) != chosen.end();
            // single-GPU requests: only the pinned GPU is usable; whole cards: this pick's pin, and never a later pick's pin
            const bool later_pin = pin < 0 && std::find(pinned.begin(), pinned.end(), d) != pinned.end();
            const bool usable = !taken_card && !later_pin && (pin < 0 || d == pin);
            free_core[d] = resource == EGPU_RESOURCE_CORE ? (usable ? c : 0) : (usable ? EGPU_CORE_MAX : 0);
            free_mem[d] = resource == EGPU_RESOURCE_MEM ? (usable ? c : 0) : (usable ? EGPU_MEM_MAX : 0);
        }
        // a request for 0 units of the constrained resource still needs 1 unit of the other
        // dimension on unusable GPUs to be excluded: unusable rows are (0, 0), request >= (0, 0)
        // would fit them, so ask for one unit of the unconstrained dimension
        int32_t req_core = resource == EGPU_RESOURCE_CORE ? (whole_cards ? EGPU_CORE_MAX : allocation_size) : 1;
        int32_t req_mem = resource == EGPU_RESOURCE_MEM ? allocation_size : 1;
        // stateless query against this request's availability table: the context's own table (the
        // node's committed placement, INTEGRATION.md) is neither read nor written, and the call
        // holds the context mutex from the table upload to the answer
        int32_t idx = -1;
        const int rc = egpu_bestfit_query(ctx, free_core.data(), free_mem.data(), D, &req_core, &req_mem, 1, &idx);
        if (rc != EGPU_OK) return rc;
        if (idx < 0) return EGPU_ERR_UNSAT;
        chosen.push_back(idx);
    }
    if (out_gpu) *out_gpu = chosen[0];

    // 4. IDs of the chosen GPU(s): must-include first, then pick by pick, ascending unit number
    std::vector<char> taken(static_cast<size_t>(n_available), 0);
    int32_t n_out = 0;
    for (int64_t k = 0; k < n_must; ++k) {
        const int32_t p = pos_of[must_include_ids[k]];
        if (!taken[p]) {
            taken[p] = 1;
            out_positions[n_out++] = p;
        }
    }
    for (int32_t g : chosen) {
        // candidates as (unit, position) pairs: their natural order is the selection rule (lowest unit first,
        // the earlier position among equal units) and the comparisons stay inside one contiguous array
        std::vector<std::pair<int64_t, int32_t>> cand;
        for (int64_t i = 0; i < n_available; ++i)
            if (gpu_of[i] == g && !taken[i]) cand.emplace_back(unit_of[i], static_cast<int32_t>(i));
        // a single-GPU request takes what it still needs; a whole card gives all 100 of its units
        const int32_t want = whole_cards ? EGPU_CORE_MAX : allocation_size;
        int32_t have = 0;
        for (int32_t i = 0; i < n_out; ++i) have += gpu_of[out_positions[i]] == g;
        // only the `want - have` lowest unit numbers are needed: select them, then order them (a gpu-memory
        // plugin offers one ID per MiB, 81 559 per H100 80GB: sorting them all is wasted work)
        const size_t need = static_cast<size_t>(want > have ? want - have : 0);
        if (need < cand.size()) {
            std::nth_element(cand.begin(), cand.begin() + static_cast<std::ptrdiff_t>(need), cand.end());
            cand.resize(need);
        }
        std::sort(cand.begin(), cand.end());
        for (size_t k = 0; k < cand.size() && have < want && n_out < allocation_size; ++k, ++have) out_positions[n_out++] = cand[k].second;
    }
    return n_out == allocation_size ? EGPU_OK : EGPU_ERR_UNSAT;
}

}  // extern "C"

/* release_oracle.c - scalar restatement of the release rule (DESIGN.md 2.8), for the tests only.
 * TEST INFRASTRUCTURE: nothing in the product includes or links this file.  tests/test_release_oracle.py
 * compiles it into tests/_build/ and checks it against tests/release_np.py and the known answers. */
#include <stdint.h>

#define CORE_MAX 100
#define MEM_MAX ((1 << 18) - 1)
#define REL_FLAGGED 1
#define REL_EXCEEDS 2

/* Row r holds (core[r], mem[r]) on device idx[r] iff 0 <= idx[r] < D and the request is in the domain.
 * u[2*D] receives the sums, table_out[3*D] free + u (refused: free) and the reason words.
 * Returns 1 when accepted, 0 when refused, -1 on a bad argument. */
int oracle_release(const int32_t* free_core, const int32_t* free_mem, const int32_t* oversub, int32_t D,
                   const int32_t* core, const int32_t* mem, const int32_t* idx, int64_t R, int64_t* u,
                   int32_t* table_out) {
    if (D < 1 || D > 64 || R < 0) return -1;
    for (int d = 0; d < 2 * D; ++d) u[d] = 0;
    for (int64_t r = 0; r < R; ++r) {
        if (idx[r] < 0 || idx[r] >= D) continue;
        if (core[r] < 0 || core[r] > CORE_MAX || mem[r] < 0 || mem[r] > MEM_MAX) continue;
        u[idx[r]] += core[r];
        u[D + idx[r]] += mem[r];
    }
    int refused = 0;
    for (int d = 0; d < D; ++d) {
        int32_t reason = 0;
        if (u[d] > 0 || u[D + d] > 0) {
            if (oversub[d]) reason = REL_FLAGGED;
            else if (free_core[d] + u[d] > CORE_MAX || free_mem[d] + u[D + d] > MEM_MAX) reason = REL_EXCEEDS;
        }
        table_out[2 * D + d] = reason;
        refused |= reason != 0;
    }
    for (int d = 0; d < D; ++d) {
        table_out[d] = refused ? free_core[d] : (int32_t)(free_core[d] + u[d]);
        table_out[D + d] = refused ? free_mem[d] : (int32_t)(free_mem[d] + u[D + d]);
    }
    return !refused;
}

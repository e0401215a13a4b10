// egpu_id_grammar.h — the device-ID grammar "%d-%02d" (pkg/plugins/gpushare.go:28,163), in one place
// for the host codec (egpu_plugin.cc, also built by plain g++ without CUDA headers) and the device
// pipeline of egpu_preferred_allocation_batch (egpu_prefalloc.cu).  Internal.
#pragma once
#include <stdint.h>

#ifdef __CUDACC__
#define EGPU_ID_HD __host__ __device__ __forceinline__
#else
#define EGPU_ID_HD inline
#endif

// Longest ID the grammar accepts: 9 GPU digits, '-', 15 unit digits.
#define EGPU_ID_MAX_BYTES 25

// Strict parse of one ID: decimal GPU without padding, '-', decimal unit of at least two digits, padded
// to exactly two digits at most; nothing else.  n < 0: the ID is NUL-terminated; n >= 0: it is exactly
// the n bytes at s (a NUL among them is a foreign character).  Never reads past the first byte that
// breaks the grammar.  Returns 0 and sets *gpu, *unit, or -1 for a malformed ID.
EGPU_ID_HD int egpu_id_grammar(const char* s, int64_t n, int32_t* gpu, int64_t* unit) {
    const int end = n < 0 ? 0 : -1;  // what at() returns after the last byte
    int64_t i = 0;
#define EGPU_ID_AT(k) (n < 0 || (k) < n ? static_cast<int>(static_cast<unsigned char>(s[k])) : -1)
    int c = EGPU_ID_AT(i);
    if (c < '0' || c > '9') return -1;
    const int g0 = c;
    int64_t g = 0;
    int digits = 0;
    while (c >= '0' && c <= '9') {
        g = g * 10 + (c - '0');
        if (++digits > 9) return -1;
        ++i;
        c = EGPU_ID_AT(i);
    }
    if (digits > 1 && g0 == '0') return -1;  // %d never pads the GPU index
    if (c != '-') return -1;
    ++i;
    c = EGPU_ID_AT(i);
    const int u0 = c;
    int64_t u = 0;
    digits = 0;
    while (c >= '0' && c <= '9') {
        u = u * 10 + (c - '0');
        if (++digits > 15) return -1;
        ++i;
        c = EGPU_ID_AT(i);
    }
#undef EGPU_ID_AT
    if (c != end || digits < 2) return -1;       // %02d: at least two digits
    if (digits > 2 && u0 == '0') return -1;      // padding only up to two digits
    *gpu = static_cast<int32_t>(g);
    *unit = u;
    return 0;
}

// egpu_devhash.cu — device-set identity on the GPU: types.NewDevice + hash + Equals of
// elastic-ai/elastic-gpu-agent (pkg/types/device.go:17-54), batched over many ID lists the
// way KubeletDeviceLocator.Locate needs them (pkg/kube/locator.go:62-90).
//
//   sort.Strings(ids); Hash = hex(sha256(strings.Join(ids, ":")))[0:8]
//
// Product path (no CPU fallback, nothing from oracle/).  Byte work, HBM/latency bound:
//   pack      one thread per ID: <= 16 chars of {'-','0'..'9'} -> 4 bits each in a u64,
//             first character in the top nibble, so u64 order == byte-wise string order
//   sort      LSD radix sort, 4-bit digits, on (set, key): only as many passes as the
//             longest ID has characters, plus ceil(log16(n_sets)) for the set index
//   render    exclusive scan of (len + 1) gives every ID its place in its set's message;
//             one thread per ID writes the characters and the ':' separator
//   sha256    one thread per set walks its message in 64-byte blocks (the chain is serial)
//   locate    candidate set == request set iff same size and all sorted keys equal
#include <algorithm>
#include <cstddef>
#include <cstdlib>
#include <cstring>
#include <new>
#include <vector>

#include "../../include/egpu_devhash.h"
#include "../../include/egpu_restore.h"
#include "egpu_ctx.h"

namespace egpu {

constexpr int kSortThreads = 256;
constexpr int kSortItems = 8;                          // items per thread (blocked arrangement)
constexpr int kSortTile = kSortThreads * kSortItems;   // items per CTA per pass

struct HashErr {
    int bad;      // != 0: some ID is empty, longer than 16 bytes, outside the byte buffer or has a foreign character
    int max_len;  // longest ID of the batch: the number of key digits the sort has to look at
};

__device__ __forceinline__ uint32_t char_code(unsigned char c) {
    if (c == '-') return 1u;
    if (c >= '0' && c <= '9') return 2u + (c - '0');
    return 0u;  // invalid
}
__device__ __forceinline__ char code_char(uint32_t n) { return n == 1u ? '-' : static_cast<char>('0' + (n - 2u)); }

// Also the validation of the caller's offsets (every ID 1..16 bytes, inside the byte buffer), the set
// index of every ID (binary search in the few set offsets) and the longest ID: the host never walks
// the n_ids-long arrays, it only hands them to the copy engine.
__global__ void pack_ids_kernel(const char* __restrict__ flat, long long flat_bytes, const long long* __restrict__ id_off,
                                long long n_ids, const long long* __restrict__ set_off, long long n_sets,
                                unsigned long long* __restrict__ key, uint32_t* __restrict__ set, uint32_t* __restrict__ len1,
                                HashErr* err) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    const bool live = i < n_ids;
    const long long b = live ? id_off[i] : 0, e = live ? id_off[i + 1] : 1;
    const long long l = e - b;
    const int my_len = live && l >= 1 && l <= 16 ? static_cast<int>(l) : 0;
    const int warp_max = __reduce_max_sync(0xffffffffu, my_len);
    if ((threadIdx.x & 31) == 0 && warp_max) atomicMax(&err->max_len, warp_max);
    if (!live) return;
    {   // set of ID i: the last q with set_off[q] <= i (empty sets share their offset with the next one)
        long long lo = 0, hi = n_sets;  // invariant: set_off[lo] <= i < set_off[hi]
        while (hi - lo > 1) {
            const long long mid = (lo + hi) >> 1;
            if (set_off[mid] <= i) lo = mid; else hi = mid;
        }
        set[i] = static_cast<uint32_t>(lo);
    }
    unsigned long long k = 0;
    bool ok = l >= 1 && l <= 16 && b >= 0 && e <= flat_bytes;
    for (int j = 0; j < 16; ++j) {
        uint32_t code = 0;
        if (j < l && ok) {
            code = char_code(static_cast<unsigned char>(flat[b + j]));
            ok = ok && code != 0u;
        }
        k = (k << 4) | code;
    }
    if (!ok) {
        err->bad = 1;
        k = 0;
    }
    key[i] = k;
    len1[i] = static_cast<uint32_t>(ok ? l : 0) + 1u;  // + ':' (the last one of a set is dropped later)
}

// ---- sort inside the sets, in shared memory -------------------------------------------
// The IDs of a set are contiguous in the input (set_off), so "(set, key) order" is every set's own
// range in key order.  When the largest set fits shared memory (<= 16 384 keys = 128 KB; a node-scale
// container has 4 K .. 16 K IDs) one CTA per set runs a bitonic network over its range, padded to a
// power of two with all-ones keys (no packed ID has a 0xF nibble): 105 barrier-separated steps at
// 16 K, against ten global radix passes of three kernels over the whole batch.  Equal keys are equal IDs, so the network's instability is invisible.
constexpr int kSortSmemMaxKeys = 16384;
__global__ void __launch_bounds__(1024)
sort_sets_smem_kernel(unsigned long long* __restrict__ key, const long long* __restrict__ set_off) {
    extern __shared__ unsigned long long sk[];
    const long long b = set_off[blockIdx.x];
    const int n = static_cast<int>(set_off[blockIdx.x + 1] - b);
    if (n <= 1) return;
    int np = 2;
    while (np < n) np <<= 1;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int i = tid; i < np; i += nt) sk[i] = i < n ? key[b + i] : ~0ull;
    __syncthreads();
    for (int k = 2; k <= np; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int t = tid; t < (np >> 1); t += nt) {
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));  // t with a 0 inserted at bit log2(j)
                const int p = i | j;
                const unsigned long long a = sk[i], c = sk[p];
                const bool ascending = (i & k) == 0;
                if ((a > c) == ascending) {
                    sk[i] = c;
                    sk[p] = a;
                }
            }
            __syncthreads();
        }
    }
    for (int i = tid; i < n; i += nt) key[b + i] = sk[i];
}

// ---- LSD radix sort, 4-bit digit, stable (sets too large for shared memory) ------------
// digit source: shift < 64 -> key nibble, else set-index nibble (shift - 64)
__device__ __forceinline__ uint32_t digit_of(unsigned long long k, uint32_t s, int shift) {
    return shift < 64 ? static_cast<uint32_t>(k >> shift) & 15u : (s >> (shift - 64)) & 15u;
}

__global__ void __launch_bounds__(kSortThreads)
radix_hist_kernel(const unsigned long long* __restrict__ key, const uint32_t* __restrict__ set, long long n, int shift,
                  uint32_t* __restrict__ hist /* [16][gridDim.x] */) {
    __shared__ uint32_t sh[16];
    if (threadIdx.x < 16) sh[threadIdx.x] = 0;
    __syncthreads();
    const long long base = static_cast<long long>(blockIdx.x) * kSortTile;
    uint32_t local[16];
#pragma unroll
    for (int b = 0; b < 16; ++b) local[b] = 0;
    for (int j = 0; j < kSortItems; ++j) {
        const long long i = base + threadIdx.x + static_cast<long long>(j) * kSortThreads;  // coalesced: order is irrelevant here
        if (i < n) {
            const uint32_t d = digit_of(key[i], set[i], shift);
#pragma unroll
            for (int b = 0; b < 16; ++b) local[b] += (d == static_cast<uint32_t>(b));
        }
    }
#pragma unroll
    for (int b = 0; b < 16; ++b) {
        const uint32_t w = __reduce_add_sync(0xffffffffu, local[b]);
        if ((threadIdx.x & 31) == 0 && w) atomicAdd(&sh[b], w);
    }
    __syncthreads();
    if (threadIdx.x < 16) hist[threadIdx.x * gridDim.x + blockIdx.x] = sh[threadIdx.x];
}

// exclusive scan of hist in (digit major, block minor) order; one CTA
__global__ void __launch_bounds__(1024) radix_scan_kernel(uint32_t* __restrict__ hist, int n) {
    __shared__ uint32_t carry;
    __shared__ uint32_t warp_sum[32];
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n; base += 1024) {
        const int i = base + threadIdx.x;
        const uint32_t v = i < n ? hist[i] : 0u;
        uint32_t x = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
            if ((threadIdx.x & 31) >= o) x += y;
        }
        if ((threadIdx.x & 31) == 31) warp_sum[threadIdx.x >> 5] = x;
        __syncthreads();
        if (threadIdx.x < 32) {
            uint32_t w = warp_sum[threadIdx.x];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t y = __shfl_up_sync(0xffffffffu, w, o);
                if (threadIdx.x >= o) w += y;
            }
            warp_sum[threadIdx.x] = w;  // inclusive over warps
        }
        __syncthreads();
        const uint32_t wprev = (threadIdx.x >> 5) ? warp_sum[(threadIdx.x >> 5) - 1] : 0u;
        const uint32_t incl = x + wprev + carry;
        if (i < n) hist[i] = incl - v;
        __syncthreads();
        if (threadIdx.x == 1023) carry = incl;
        __syncthreads();
    }
}

__global__ void __launch_bounds__(kSortThreads)
radix_scatter_kernel(const unsigned long long* __restrict__ key_in, const uint32_t* __restrict__ set_in, long long n, int shift,
                     const uint32_t* __restrict__ offs /* scanned hist */, unsigned long long* __restrict__ key_out,
                     uint32_t* __restrict__ set_out) {
    // blocked arrangement: thread t owns items [t*kSortItems, (t+1)*kSortItems) of the tile, so a
    // per-thread count followed by a scan over threads gives STABLE ranks
    __shared__ uint32_t cnt[16][kSortThreads + 1];
    const int t = threadIdx.x;
    const long long base = static_cast<long long>(blockIdx.x) * kSortTile + static_cast<long long>(t) * kSortItems;
    unsigned long long k[kSortItems];
    uint32_t s[kSortItems], d[kSortItems];
    uint32_t local[16];
#pragma unroll
    for (int b = 0; b < 16; ++b) local[b] = 0;
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        const long long i = base + j;
        d[j] = 16u;
        if (i < n) {
            k[j] = key_in[i];
            s[j] = set_in[i];
            d[j] = digit_of(k[j], s[j], shift);
#pragma unroll
            for (int b = 0; b < 16; ++b) local[b] += (d[j] == static_cast<uint32_t>(b));
        }
    }
#pragma unroll
    for (int b = 0; b < 16; ++b) cnt[b][t] = local[b];
    __syncthreads();
    // exclusive scan of each digit row over the threads: warp w scans rows w, w+8
    {
        const int warp = t >> 5, lane = t & 31;
        for (int row = warp; row < 16; row += kSortThreads / 32) {
            uint32_t run = 0;
            for (int c0 = 0; c0 < kSortThreads; c0 += 32) {
                const uint32_t v = cnt[row][c0 + lane];
                uint32_t x = v;
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) {
                    const uint32_t y = __shfl_up_sync(0xffffffffu, x, o);
                    if (lane >= o) x += y;
                }
                cnt[row][c0 + lane] = run + x - v;
                run += __shfl_sync(0xffffffffu, x, 31);
            }
        }
    }
    __syncthreads();
    uint32_t pos[16];
#pragma unroll
    for (int b = 0; b < 16; ++b) pos[b] = offs[b * gridDim.x + blockIdx.x] + cnt[b][t];
#pragma unroll
    for (int j = 0; j < kSortItems; ++j) {
        if (d[j] < 16u) {
            uint32_t dst = 0;
#pragma unroll
            for (int b = 0; b < 16; ++b)
                if (d[j] == static_cast<uint32_t>(b)) dst = pos[b]++;
            key_out[dst] = k[j];
            set_out[dst] = s[j];
        }
    }
}

// ---- generic exclusive scan of uint32 -> uint64 (message byte offsets) ---------------
__global__ void __launch_bounds__(1024)
scan_block_sums_kernel(const uint32_t* __restrict__ v, long long n, unsigned long long* __restrict__ block_sum) {
    __shared__ unsigned long long sh[32];
    const long long i = static_cast<long long>(blockIdx.x) * 1024 + threadIdx.x;
    unsigned long long x = i < n ? v[i] : 0ull;
    for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
        x = sh[threadIdx.x];
        for (int o = 16; o; o >>= 1) x += __shfl_xor_sync(0xffffffffu, x, o);
        if (threadIdx.x == 0) block_sum[blockIdx.x] = x;
    }
}
// exclusive scan of the block sums, in place: one CTA, 1024 values per trip
__global__ void __launch_bounds__(1024) scan_blocks_kernel(unsigned long long* __restrict__ a, long long n) {
    __shared__ unsigned long long warp_sum[32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    unsigned long long carry = 0;
    for (long long base = 0; base < n; base += 1024) {
        const long long i = base + threadIdx.x;
        const unsigned long long val = i < n ? a[i] : 0ull;
        unsigned long long x = val;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
            if (lane >= o) x += y;
        }
        if (lane == 31) warp_sum[warp] = x;
        __syncthreads();
        if (warp == 0) {
            unsigned long long w = warp_sum[lane];
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
                if (lane >= o) w += y;
            }
            warp_sum[lane] = w;
        }
        __syncthreads();
        if (i < n) a[i] = carry + x + (warp ? warp_sum[warp - 1] : 0ull) - val;
        carry += warp_sum[31];
        __syncthreads();
    }
}
__global__ void __launch_bounds__(1024)
scan_apply_kernel(const uint32_t* __restrict__ v, long long n, const unsigned long long* __restrict__ block_off,
                  unsigned long long* __restrict__ out /* [n + 1] */) {
    __shared__ unsigned long long warp_sum[32];
    const long long i = static_cast<long long>(blockIdx.x) * 1024 + threadIdx.x;
    const unsigned long long val = i < n ? v[i] : 0ull;
    unsigned long long x = val;
    const int lane = threadIdx.x & 31;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
        if (lane >= o) x += y;
    }
    if (lane == 31) warp_sum[threadIdx.x >> 5] = x;
    __syncthreads();
    if (threadIdx.x < 32) {
        unsigned long long w = warp_sum[threadIdx.x];
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long y = __shfl_up_sync(0xffffffffu, w, o);
            if (threadIdx.x >= o) w += y;
        }
        warp_sum[threadIdx.x] = w;
    }
    __syncthreads();
    const unsigned long long wprev = (threadIdx.x >> 5) ? warp_sum[(threadIdx.x >> 5) - 1] : 0ull;
    const unsigned long long incl = x + wprev + block_off[blockIdx.x];
    if (i < n) {
        out[i] = incl - val;
        if (i == n - 1) out[n] = incl;
    }
}

// after the sort: length (+1) of every sorted ID, recovered from its key
__global__ void sorted_len_kernel(const unsigned long long* __restrict__ key, long long n, uint32_t* __restrict__ len1) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const unsigned long long k = key[i];
    // characters are left-aligned: length = 16 - (trailing zero nibbles)
    const int tz = k ? (__ffsll(static_cast<long long>(k)) - 1) >> 2 : 16;
    len1[i] = static_cast<uint32_t>(16 - tz) + 1u;
}

// message layout: set s starts at msg_base[s] (64-byte aligned); ID i of the sorted array
// sits at msg_base[s] + (pref[i] - pref[set_start[s]])
__global__ void set_layout_kernel(const long long* __restrict__ set_off, long long n_sets,
                                  const unsigned long long* __restrict__ pref, unsigned long long* __restrict__ msg_base,
                                  unsigned long long* __restrict__ msg_len) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        unsigned long long run = 0;
        for (long long s = 0; s < n_sets; ++s) {
            const unsigned long long bytes = pref[set_off[s + 1]] - pref[set_off[s]];
            const unsigned long long len = bytes ? bytes - 1 : 0;  // no ':' after the last ID
            msg_base[s] = run;
            msg_len[s] = len;
            run += (len + 64 + 63) & ~63ull;  // room for SHA-256 padding, keep 64-byte alignment
        }
        msg_base[n_sets] = run;
    }
}

__global__ void render_kernel(const unsigned long long* __restrict__ key, const uint32_t* __restrict__ set, long long n,
                              const long long* __restrict__ set_off, const unsigned long long* __restrict__ pref,
                              const unsigned long long* __restrict__ msg_base, unsigned char* __restrict__ msg) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = set[i];
    unsigned char* p = msg + msg_base[s] + (pref[i] - pref[set_off[s]]);
    const unsigned long long k = key[i];
    int l = 0;
    for (int j = 0; j < 16; ++j) {
        const uint32_t c = static_cast<uint32_t>(k >> (60 - 4 * j)) & 15u;
        if (!c) break;
        p[l++] = static_cast<unsigned char>(code_char(c));
    }
    if (i + 1 < set_off[s + 1]) p[l] = ':';
}

// ---- SHA-256 (FIPS 180-4), one message per thread -------------------------------------
__constant__ uint32_t kSha[64] = {
    0x428a2f98, 0x71374491, 0xb5c0fbcf, 0xe9b5dba5, 0x3956c25b, 0x59f111f1, 0x923f82a4, 0xab1c5ed5,
    0xd807aa98, 0x12835b01, 0x243185be, 0x550c7dc3, 0x72be5d74, 0x80deb1fe, 0x9bdc06a7, 0xc19bf174,
    0xe49b69c1, 0xefbe4786, 0x0fc19dc6, 0x240ca1cc, 0x2de92c6f, 0x4a7484aa, 0x5cb0a9dc, 0x76f988da,
    0x983e5152, 0xa831c66d, 0xb00327c8, 0xbf597fc7, 0xc6e00bf3, 0xd5a79147, 0x06ca6351, 0x14292967,
    0x27b70a85, 0x2e1b2138, 0x4d2c6dfc, 0x53380d13, 0x650a7354, 0x766a0abb, 0x81c2c92e, 0x92722c85,
    0xa2bfe8a1, 0xa81a664b, 0xc24b8b70, 0xc76c51a3, 0xd192e819, 0xd6990624, 0xf40e3585, 0x106aa070,
    0x19a4c116, 0x1e376c08, 0x2748774c, 0x34b0bcb5, 0x391c0cb3, 0x4ed8aa4a, 0x5b9cca4f, 0x682e6ff3,
    0x748f82ee, 0x78a5636f, 0x84c87814, 0x8cc70208, 0x90befffa, 0xa4506ceb, 0xbef9a3f7, 0xc67178f2};

__device__ __forceinline__ uint32_t rotr32(uint32_t x, int n) { return __funnelshift_r(x, x, n); }
// a + b on the FMA pipe (IMAD): in the one-lane compression chain the ALU pipe (two cycles per warp
// instruction) is what bounds a round - ten rotations / logic ops live there - so the additions go next door
__device__ __forceinline__ uint32_t add_fma(uint32_t a, uint32_t b) {
    uint32_t r;
    asm("mad.lo.u32 %0, %1, 1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}

__global__ void sha256_sets_kernel(unsigned char* __restrict__ msg, const unsigned long long* __restrict__ msg_base,
                                   const unsigned long long* __restrict__ msg_len, long long n_sets,
                                   uint32_t* __restrict__ digest /* [n_sets][8] */) {
    const long long s = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (s >= n_sets) return;
    unsigned char* m = msg + msg_base[s];
    const unsigned long long len = msg_len[s];
    // padding in place (the layout reserved the room): 0x80, zeros, 64-bit big-endian bit length
    const unsigned long long total = ((len + 8) / 64 + 1) * 64;
    m[len] = 0x80;
    for (unsigned long long i = len + 1; i < total - 8; ++i) m[i] = 0;
    const unsigned long long bits = len * 8;
    for (int i = 0; i < 8; ++i) m[total - 1 - i] = static_cast<unsigned char>(bits >> (8 * i));
    uint32_t h0 = 0x6a09e667, h1 = 0xbb67ae85, h2 = 0x3c6ef372, h3 = 0xa54ff53a, h4 = 0x510e527f, h5 = 0x9b05688c,
             h6 = 0x1f83d9ab, h7 = 0x5be0cd19;
    const uint32_t* words = reinterpret_cast<const uint32_t*>(m);  // 64-byte aligned base
    for (unsigned long long blk = 0; blk < total / 64; ++blk) {
        uint32_t w[16];
#pragma unroll
        for (int i = 0; i < 16; ++i) w[i] = __byte_perm(words[blk * 16 + i], 0, 0x0123);  // big-endian load
        uint32_t a = h0, b = h1, c = h2, d = h3, e = h4, f = h5, g = h6, h = h7;
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            uint32_t wi;
            if (i < 16) {
                wi = w[i];
            } else {
                const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
                const uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
                const uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
                wi = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
                w[i & 15] = wi;
            }
            const uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
            const uint32_t ch = (e & f) ^ (~e & g);
            const uint32_t t1 = h + S1 + ch + kSha[i] + wi;
            const uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
            const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
            const uint32_t t2 = S0 + mj;
            h = g; g = f; f = e; e = d + t1; d = c; c = b; b = a; a = t1 + t2;
        }
        h0 += a; h1 += b; h2 += c; h3 += d; h4 += e; h5 += f; h6 += g; h7 += h;
    }
    uint32_t* o = digest + s * 8;
    o[0] = h0; o[1] = h1; o[2] = h2; o[3] = h3; o[4] = h4; o[5] = h5; o[6] = h6; o[7] = h7;
}

// ---- SHA-256 of LONG messages: one CTA (two warps) per message -------------------------
// The compression chain of one message is serial (block k needs the state after block k - 1), so a
// node-scale batch - ~100 sets of 4 K .. 16 K IDs, 0.5 .. 2 K blocks each - is bound by the latency
// of the longest chain, not by throughput.  What can be taken off the chain is: the loads, the
// byte swaps and the whole message schedule W[16..63] (48 of the 64 rounds' extra work), and the
// additions of the round constants.  Warp 1 does all of that for 32 blocks at a time (lane = block)
// into a shared-memory ring of K[i] + W[i] words; lane 0 of warp 0 walks the blocks in order with
// nothing but the 64 rounds left: per round the dependent path is three instructions
// (rotations -> xor -> 3-input add).  Double-buffered, one __syncthreads per 32 blocks.
constexpr int kShaGroup = 32;
__global__ void __launch_bounds__(64)
sha256_long_kernel(unsigned char* __restrict__ msg, const unsigned long long* __restrict__ msg_base,
                   const unsigned long long* __restrict__ msg_len, long long n_sets, uint32_t* __restrict__ digest) {
    // K[i] + W[i] of 2 x 32 blocks; rows padded to 65 words: lane = row writes column i into bank (row + i) mod 32 -
    // conflict-free - and the reader's offsets are compile-time constants (no address arithmetic on its ALU pipe)
    __shared__ uint32_t kw[2][kShaGroup][65];
    const long long s = blockIdx.x;
    if (s >= n_sets) return;
    unsigned char* m = msg + msg_base[s];
    const unsigned long long len = msg_len[s];
    const unsigned long long total = ((len + 8) / 64 + 1) * 64;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    // padding in place (the layout reserved the room), by the whole CTA
    for (unsigned long long i = len + tid; i < total; i += 64) {
        unsigned char v = 0;
        if (i == len) v = 0x80;
        else if (i >= total - 8) v = static_cast<unsigned char>((len * 8) >> (8 * (total - 1 - i)));
        m[i] = v;
    }
    __syncthreads();
    const unsigned long long n_blk = total / 64;
    const uint4* words = reinterpret_cast<const uint4*>(m);  // 64-byte aligned base
    auto produce = [&](unsigned long long g) {  // warp 1: schedule of blocks g*32 .. g*32+31 into buffer g & 1
        const unsigned long long blk = g * kShaGroup + lane;
        if (blk >= n_blk) return;
        uint32_t w[16];
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const uint4 v = words[blk * 4 + q];
            w[4 * q] = __byte_perm(v.x, 0, 0x0123);
            w[4 * q + 1] = __byte_perm(v.y, 0, 0x0123);
            w[4 * q + 2] = __byte_perm(v.z, 0, 0x0123);
            w[4 * q + 3] = __byte_perm(v.w, 0, 0x0123);
        }
        uint32_t* out = kw[g & 1][lane];
#pragma unroll
        for (int i = 0; i < 64; ++i) {
            uint32_t wi;
            if (i < 16) {
                wi = w[i];
            } else {
                const uint32_t w15 = w[(i - 15) & 15], w2 = w[(i - 2) & 15];
                const uint32_t s0 = rotr32(w15, 7) ^ rotr32(w15, 18) ^ (w15 >> 3);
                const uint32_t s1 = rotr32(w2, 17) ^ rotr32(w2, 19) ^ (w2 >> 10);
                wi = w[i & 15] + s0 + w[(i - 7) & 15] + s1;
                w[i & 15] = wi;
            }
            out[i] = wi + kSha[i];
        }
    };
    uint32_t h0 = 0x6a09e667, h1 = 0xbb67ae85, h2 = 0x3c6ef372, h3 = 0xa54ff53a, h4 = 0x510e527f, h5 = 0x9b05688c,
             h6 = 0x1f83d9ab, h7 = 0x5be0cd19;
    const unsigned long long n_grp = (n_blk + kShaGroup - 1) / kShaGroup;
    if (warp == 1) produce(0);
    __syncthreads();
    for (unsigned long long g = 0; g < n_grp; ++g) {
        if (warp == 1) {
            if (g + 1 < n_grp) produce(g + 1);
        } else if (lane == 0) {
            const unsigned long long b_end = (g + 1) * kShaGroup < n_blk ? kShaGroup : n_blk - g * kShaGroup;
            for (int bi = 0; bi < static_cast<int>(b_end); ++bi) {
                const uint32_t* x = kw[g & 1][bi];
                uint32_t a = h0, b = h1, c = h2, d = h3, e = h4, f = h5, gg = h6, h = h7;
#pragma unroll
                for (int i = 0; i < 64; ++i) {
                    const uint32_t t0 = add_fma(h, x[i]);   // off the dependent path
                    const uint32_t S1 = rotr32(e, 6) ^ rotr32(e, 11) ^ rotr32(e, 25);
                    const uint32_t ch = (e & f) ^ (~e & gg);
                    const uint32_t t1 = add_fma(add_fma(t0, ch), S1);
                    const uint32_t S0 = rotr32(a, 2) ^ rotr32(a, 13) ^ rotr32(a, 22);
                    const uint32_t mj = (a & b) ^ (a & c) ^ (b & c);
                    h = gg; gg = f; f = e; e = add_fma(d, t1); d = c; c = b; b = a; a = add_fma(add_fma(t1, mj), S0);
                }
                h0 += a; h1 += b; h2 += c; h3 += d; h4 += e; h5 += f; h6 += gg; h7 += h;
            }
        }
        __syncthreads();
    }
    if (tid == 0) {
        uint32_t* o = digest + s * 8;
        o[0] = h0; o[1] = h1; o[2] = h2; o[3] = h3; o[4] = h4; o[5] = h5; o[6] = h6; o[7] = h7;
    }
}

// Device.Equals against set 0: one thread per candidate ID compares with the request's ID
// at the same sorted rank; any difference clears the candidate's flag
__global__ void locate_compare_kernel(const unsigned long long* __restrict__ key, const uint32_t* __restrict__ set,
                                      long long n, const long long* __restrict__ set_off, int* __restrict__ equal) {
    const long long i = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const uint32_t s = set[i];
    if (s == 0) return;
    const long long n0 = set_off[1] - set_off[0];
    const long long ns = set_off[s + 1] - set_off[s];
    if (ns != n0) {
        equal[s] = 0;
        return;
    }
    if (key[i] != key[set_off[0] + (i - set_off[s])]) equal[s] = 0;
}
__global__ void locate_init_kernel(int* __restrict__ equal, const long long* __restrict__ set_off, long long n_sets) {
    const long long s = static_cast<long long>(blockIdx.x) * blockDim.x + threadIdx.x;
    if (s >= n_sets) return;
    // sets of a different size never match; equal-size sets start as "equal" and are knocked out
    equal[s] = (s > 0 && (set_off[s + 1] - set_off[s]) == (set_off[1] - set_off[0])) ? 1 : 0;
}

// ---- the sort and the scan for other pipelines of the library (egpu_prefalloc.cu) -------
size_t radix_hist_words(long long n) {
    const long long tiles = (n + kSortTile - 1) / kSortTile;
    return 16 * static_cast<size_t>(tiles > 0 ? tiles : 1);
}

int radix_sort_pairs(cudaStream_t s, unsigned long long*& key, uint32_t*& val, unsigned long long*& key_tmp,
                     uint32_t*& val_tmp, long long n, int n_digits, uint32_t* hist) {
    if (n <= 0) return 0;
    const unsigned tiles = static_cast<unsigned>((n + kSortTile - 1) / kSortTile);
    for (int j = 0; j < n_digits; ++j) {
        radix_hist_kernel<<<tiles, kSortThreads, 0, s>>>(key, val, n, 4 * j, hist);
        radix_scan_kernel<<<1, 1024, 0, s>>>(hist, static_cast<int>(16 * tiles));
        radix_scatter_kernel<<<tiles, kSortThreads, 0, s>>>(key, val, n, 4 * j, hist, key_tmp, val_tmp);
        std::swap(key, key_tmp);
        std::swap(val, val_tmp);
    }
    return 3 * n_digits;
}

int exclusive_scan_u32(cudaStream_t s, const uint32_t* v, long long n, unsigned long long* blk, unsigned long long* out) {
    if (n <= 0) return 0;
    const unsigned nblk = static_cast<unsigned>((n + 1023) / 1024);
    scan_block_sums_kernel<<<nblk, 1024, 0, s>>>(v, n, blk);
    scan_blocks_kernel<<<1, 1024, 0, s>>>(blk, nblk);
    scan_apply_kernel<<<nblk, 1024, 0, s>>>(v, n, blk, out);
    return 3;
}

}  // namespace egpu

using namespace egpu;

namespace {

struct DevBuf {
    void* p = nullptr;
    template <class T>
    T* as() { return static_cast<T*>(p); }
};

// common pipeline: pack, sort, layout, render, hash.  Leaves digests on the device and, for
// locate, the sorted keys.  All on the context's stream.
struct HashRun {
    DevBuf flat, id_off, set_off, set_of, key_a, key_b, set_a, set_b, len1, pref, blk, hist, msg_base, msg_len, msg, digest, err,
        equal;
    unsigned long long* sorted_key = nullptr;
    uint32_t* sorted_set = nullptr;
};

int run_hash(egpu_ctx* ctx, HashRun& r, const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
             const int64_t* set_offsets, int64_t n_sets, bool need_digest) {
    cudaStream_t s = ctx->stream;
    if (n_ids < 0 || n_sets < 1 || !id_offsets || !set_offsets) return EGPU_ERR_INVALID;
    if (set_offsets[0] != 0 || set_offsets[n_sets] != n_ids || id_offsets[0] != 0) return EGPU_ERR_INVALID;
    if (n_sets > (1ll << 24) || n_ids > (1ll << 31) - 1) return EGPU_ERR_INVALID;
    const int64_t flat_bytes = id_offsets[n_ids];
    if (flat_bytes < 0 || (flat_bytes > 0 && !ids_flat)) return EGPU_ERR_INVALID;
    int64_t max_set = 0;
    for (int64_t q = 0; q < n_sets; ++q) {
        if (set_offsets[q + 1] < set_offsets[q]) return EGPU_ERR_INVALID;
        max_set = std::max<int64_t>(max_set, set_offsets[q + 1] - set_offsets[q]);
    }
    const bool smem_sort = max_set <= kSortSmemMaxKeys && n_sets <= 65536;
    // the n_ids-long arrays are not walked here: lengths, bounds, set membership and the longest ID
    // come from pack_ids_kernel (a pageable 1 M-ID batch spent more host time on that than the GPU on the sort)
    const size_t n = static_cast<size_t>(n_ids);
    const int64_t tiles = (n_ids + kSortTile - 1) / kSortTile;
    const size_t msg_cap = static_cast<size_t>(flat_bytes) + n + static_cast<size_t>(n_sets) * 128 + 64;
    // scratch: the context's grow-only arena (cudaMalloc/cudaFree per call would cost more than the kernels)
    const ArenaWant wants[] = {
        {&r.flat.p, static_cast<size_t>(flat_bytes)}, {&r.id_off.p, sizeof(long long) * (n + 1)},
        {&r.set_off.p, sizeof(long long) * (n_sets + 1)}, {&r.key_a.p, 8 * n}, {&r.key_b.p, 8 * n}, {&r.set_a.p, 4 * n},
        {&r.set_b.p, 4 * n}, {&r.len1.p, 4 * n}, {&r.pref.p, 8 * (n + 1)}, {&r.blk.p, 8 * ((n + 1023) / 1024 + 1)},
        {&r.hist.p, 4 * 16 * static_cast<size_t>(tiles > 0 ? tiles : 1)}, {&r.msg_base.p, 8 * static_cast<size_t>(n_sets + 1)},
        {&r.msg_len.p, 8 * static_cast<size_t>(n_sets)}, {&r.digest.p, 32 * static_cast<size_t>(n_sets)}, {&r.err.p, sizeof(HashErr)},
        {&r.equal.p, sizeof(int) * static_cast<size_t>(n_sets)}, {&r.msg.p, need_digest ? msg_cap : 16}};
    EGPU_CUDA(ctx, arena_carve(ctx, wants, sizeof wants / sizeof wants[0]));
    EGPU_CUDA(ctx, cudaMemsetAsync(r.err.p, 0, sizeof(HashErr), s));
    if (flat_bytes) EGPU_CUDA(ctx, cudaMemcpyAsync(r.flat.p, ids_flat, flat_bytes, cudaMemcpyHostToDevice, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(r.id_off.p, id_offsets, sizeof(long long) * (n + 1), cudaMemcpyHostToDevice, s));
    EGPU_CUDA(ctx, cudaMemcpyAsync(r.set_off.p, set_offsets, sizeof(long long) * (n_sets + 1), cudaMemcpyHostToDevice, s));
    unsigned long long* ka = r.key_a.as<unsigned long long>();
    unsigned long long* kb = r.key_b.as<unsigned long long>();
    uint32_t* sa = r.set_a.as<uint32_t>();
    uint32_t* sb = r.set_b.as<uint32_t>();
    const unsigned nb256 = static_cast<unsigned>((n_ids + 255) / 256);
    if (n) {
        pack_ids_kernel<<<nb256, 256, 0, s>>>(r.flat.as<char>(), flat_bytes, r.id_off.as<long long>(), n_ids,
                                              r.set_off.as<long long>(), n_sets, ka, sa, r.len1.as<uint32_t>(), r.err.as<HashErr>());
        ctx->launches += 1;
    }
    if (n && smem_sort) {
        int np = 2;
        while (np < max_set) np <<= 1;
        const size_t smem = sizeof(unsigned long long) * static_cast<size_t>(np);
        if (!ctx->sort_sets_configured) {
            EGPU_CUDA(ctx, cudaFuncSetAttribute(sort_sets_smem_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                static_cast<int>(sizeof(unsigned long long) * kSortSmemMaxKeys)));
            ctx->sort_sets_configured = true;
        }
        const int threads = np / 2 >= 1024 ? 1024 : (np / 2 < 32 ? 32 : np / 2);
        sort_sets_smem_kernel<<<static_cast<unsigned>(n_sets), threads, smem, s>>>(ka, r.set_off.as<long long>());
        ctx->launches += 1;
        EGPU_CUDA(ctx, cudaGetLastError());
    } else if (n) {
        HashErr first{0, 0};
        EGPU_CUDA(ctx, cudaMemcpyAsync(&first, r.err.p, sizeof first, cudaMemcpyDeviceToHost, s));
        EGPU_CUDA(ctx, cudaStreamSynchronize(s));
        ctx->prev_is_scan = false;
        if (first.bad) return EGPU_ERR_PARSE;
        const int max_len = first.max_len;
        // LSD: last character first, then the set index
        int set_digits = 0;
        while ((1ll << (4 * set_digits)) < n_sets) ++set_digits;
        std::vector<int> shifts;
        for (int j = max_len - 1; j >= 0; --j) shifts.push_back(60 - 4 * j);
        for (int j = 0; j < set_digits; ++j) shifts.push_back(64 + 4 * j);
        for (int shift : shifts) {
            radix_hist_kernel<<<static_cast<unsigned>(tiles), kSortThreads, 0, s>>>(ka, sa, n_ids, shift, r.hist.as<uint32_t>());
            radix_scan_kernel<<<1, 1024, 0, s>>>(r.hist.as<uint32_t>(), static_cast<int>(16 * tiles));
            radix_scatter_kernel<<<static_cast<unsigned>(tiles), kSortThreads, 0, s>>>(ka, sa, n_ids, shift, r.hist.as<uint32_t>(), kb, sb);
            ctx->launches += 3;
            std::swap(ka, kb);
            std::swap(sa, sb);
        }
        EGPU_CUDA(ctx, cudaGetLastError());
    }
    r.sorted_key = ka;
    r.sorted_set = sa;
    HashErr herr{0, 0};
    if (need_digest) {
        const unsigned nblk = static_cast<unsigned>((n_ids + 1023) / 1024);
        if (n) {
            sorted_len_kernel<<<nb256, 256, 0, s>>>(ka, n_ids, r.len1.as<uint32_t>());
            scan_block_sums_kernel<<<nblk, 1024, 0, s>>>(r.len1.as<uint32_t>(), n_ids, r.blk.as<unsigned long long>());
            scan_blocks_kernel<<<1, 1024, 0, s>>>(r.blk.as<unsigned long long>(), nblk);
            scan_apply_kernel<<<nblk, 1024, 0, s>>>(r.len1.as<uint32_t>(), n_ids, r.blk.as<unsigned long long>(),
                                                    r.pref.as<unsigned long long>());
            ctx->launches += 4;
        } else {
            EGPU_CUDA(ctx, cudaMemsetAsync(r.pref.p, 0, 8, s));
        }
        set_layout_kernel<<<1, 32, 0, s>>>(r.set_off.as<long long>(), n_sets, r.pref.as<unsigned long long>(),
                                           r.msg_base.as<unsigned long long>(), r.msg_len.as<unsigned long long>());
        ctx->launches += 1;
        // (message buffer: every ID contributes len + 1 <= 17 bytes, every set <= 127 bytes of padding)
        if (n) {
            render_kernel<<<nb256, 256, 0, s>>>(ka, sa, n_ids, r.set_off.as<long long>(), r.pref.as<unsigned long long>(),
                                                r.msg_base.as<unsigned long long>(), r.msg.as<unsigned char>());
            ctx->launches += 1;
        }
        // few long messages (node-scale Locate: sets of thousands of IDs): one CTA per message, schedule and
        // loads off the chain; many short ones (one Allocate's worth of IDs each): one message per thread
        if (n_sets <= 8192 && n_ids / n_sets >= 256)
            sha256_long_kernel<<<static_cast<unsigned>(n_sets), 64, 0, s>>>(
                r.msg.as<unsigned char>(), r.msg_base.as<unsigned long long>(), r.msg_len.as<unsigned long long>(), n_sets,
                r.digest.as<uint32_t>());
        else
            sha256_sets_kernel<<<static_cast<unsigned>((n_sets + 63) / 64), 64, 0, s>>>(
                r.msg.as<unsigned char>(), r.msg_base.as<unsigned long long>(), r.msg_len.as<unsigned long long>(), n_sets,
                r.digest.as<uint32_t>());
        ctx->launches += 1;
        EGPU_CUDA(ctx, cudaGetLastError());
    }
    EGPU_CUDA(ctx, cudaMemcpyAsync(&herr, r.err.p, sizeof herr, cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    ctx->prev_is_scan = false;
    if (herr.bad) return EGPU_ERR_PARSE;
    return EGPU_OK;
}

}  // namespace

extern "C" {

int egpu_device_hash_batch(egpu_ctx* ctx, const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
                           const int64_t* set_offsets, int64_t n_sets, char* out_hash8, uint8_t* out_digest) {
    if (!ctx) return EGPU_ERR_INVALID;
    std::lock_guard<std::mutex> g(ctx->mu);
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    HashRun r;
    const int rc = run_hash(ctx, r, ids_flat, id_offsets, n_ids, set_offsets, n_sets, true);
    if (rc != EGPU_OK) return rc;
    std::vector<uint32_t> dg(static_cast<size_t>(n_sets) * 8);
    EGPU_CUDA(ctx, cudaMemcpy(dg.data(), r.digest.p, 32 * n_sets, cudaMemcpyDeviceToHost));
    static const char hex[] = "0123456789abcdef";
    for (int64_t q = 0; q < n_sets; ++q) {
        if (out_digest)
            for (int w = 0; w < 8; ++w)
                for (int b = 0; b < 4; ++b) out_digest[q * 32 + w * 4 + b] = static_cast<uint8_t>(dg[q * 8 + w] >> (24 - 8 * b));
        if (out_hash8) {
            const uint32_t w0 = dg[q * 8];
            for (int k = 0; k < 8; ++k) out_hash8[q * 9 + k] = hex[(w0 >> (28 - 4 * k)) & 15u];
            out_hash8[q * 9 + 8] = 0;
        }
    }
    return EGPU_OK;
}

int egpu_device_hash(egpu_ctx* ctx, const char* const* ids, int64_t n, char* out_hash8) {
    if (!ctx || n < 0 || (n > 0 && !ids) || !out_hash8) return EGPU_ERR_INVALID;
    std::vector<char> flat;
    std::vector<int64_t> off(static_cast<size_t>(n) + 1, 0);
    for (int64_t i = 0; i < n; ++i) {
        if (!ids[i]) return EGPU_ERR_INVALID;
        const size_t l = std::strlen(ids[i]);
        flat.insert(flat.end(), ids[i], ids[i] + l);
        off[i + 1] = static_cast<int64_t>(flat.size());
    }
    const int64_t sets[2] = {0, n};
    return egpu_device_hash_batch(ctx, flat.data(), off.data(), n, sets, 1, out_hash8, nullptr);
}

int egpu_device_locate(egpu_ctx* ctx, const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
                       const int64_t* set_offsets, int64_t n_sets, int64_t* out_match) {
    if (!ctx || !out_match) return EGPU_ERR_INVALID;
    *out_match = -1;
    std::lock_guard<std::mutex> g(ctx->mu);
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    HashRun r;
    // Equals = same hash AND same sorted list; comparing the sorted lists decides both, so the
    // digests are not needed here
    const int rc = run_hash(ctx, r, ids_flat, id_offsets, n_ids, set_offsets, n_sets, false);
    if (rc != EGPU_OK) return rc;
    if (n_sets < 2) return EGPU_OK;
    cudaStream_t s = ctx->stream;
    locate_init_kernel<<<static_cast<unsigned>((n_sets + 255) / 256), 256, 0, s>>>(r.equal.as<int>(), r.set_off.as<long long>(), n_sets);
    if (n_ids)
        locate_compare_kernel<<<static_cast<unsigned>((n_ids + 255) / 256), 256, 0, s>>>(r.sorted_key, r.sorted_set, n_ids,
                                                                                         r.set_off.as<long long>(), r.equal.as<int>());
    ctx->launches += 2;
    EGPU_CUDA(ctx, cudaGetLastError());
    std::vector<int> eq(static_cast<size_t>(n_sets));
    EGPU_CUDA(ctx, cudaMemcpyAsync(eq.data(), r.equal.p, sizeof(int) * n_sets, cudaMemcpyDeviceToHost, s));
    EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    for (int64_t q = 1; q < n_sets; ++q)
        if (eq[q]) {
            *out_match = q;
            break;
        }
    return EGPU_OK;
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------
// Placement-state restore (include/egpu_restore.h, SURVEY.md §8 row n3)
// ---------------------------------------------------------------------------------------------
namespace egpu {

constexpr int kResBadHash = -2;  // host-side marker: the stored Hash is not 8 hex digits

// One thread per stored entry: check the stored Hash against the recomputed identity, resolve
// its symlinks, add what it holds to the per-GPU usage sums (int64: 64 x 2^18 MiB fits easily,
// but so does any corrupt input).
__global__ void restore_usage_kernel(const long long* __restrict__ set_off, long long n_sets,
                                     const uint32_t* __restrict__ digest /* [n_sets][8] or nullptr */,
                                     const uint32_t* __restrict__ stored_hash, const int32_t* __restrict__ resource,
                                     const long long* __restrict__ link_off, const int32_t* __restrict__ link_gpu,
                                     int D, unsigned long long* __restrict__ usage /* [2][kMaxD] */,
                                     int32_t* __restrict__ status) {
    const long long s = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x;
    if (s >= n_sets) return;
    const long long n = set_off[s + 1] - set_off[s];
    const int res = resource[s];
    int st = EGPU_REC_OK;
    if (res != EGPU_RESOURCE_CORE && res != EGPU_RESOURCE_MEM && res != kResBadHash) {
        st = EGPU_REC_FOREIGN;
    } else if (n == 0) {
        st = EGPU_REC_EMPTY;
    } else if (res == kResBadHash || (digest && digest[s * 8] != stored_hash[s])) {
        st = EGPU_REC_HASH_MISMATCH;
    } else {
        const long long l0 = link_off[s], nl = link_off[s + 1] - l0;
        const long long need = (res == EGPU_RESOURCE_CORE && n > 100) ? n / 100 : 1;
        if (nl < need) st = EGPU_REC_NO_LINK;
        for (long long i = 0; st == EGPU_REC_OK && i < need; ++i) {
            const int g = link_gpu[l0 + i];
            if (g < 0 || g >= D) st = EGPU_REC_NO_LINK;
        }
        if (st == EGPU_REC_OK) {
            if (res == EGPU_RESOURCE_MEM) {
                atomicAdd(&usage[kMaxD + link_gpu[l0]], static_cast<unsigned long long>(n));
            } else if (n <= 100) {
                atomicAdd(&usage[link_gpu[l0]], static_cast<unsigned long long>(n));
            } else {
                for (long long i = 0; i < need; ++i) atomicAdd(&usage[link_gpu[l0 + i]], 100ull);
            }
        }
    }
    status[s] = st;
}

// free = capacity - usage, saturated at 0, with the oversubscription flag of table'
__global__ void __launch_bounds__(kMaxD)
restore_table_kernel(const int32_t* __restrict__ cap /* [2][kMaxD] */, const unsigned long long* __restrict__ usage, int D,
                     int32_t* __restrict__ table_out /* [3 * D] */) {
    const int d = threadIdx.x;
    if (d >= D) return;
    const long long c = static_cast<long long>(cap[d]) - static_cast<long long>(usage[d]);
    const long long m = static_cast<long long>(cap[kMaxD + d]) - static_cast<long long>(usage[kMaxD + d]);
    table_out[d] = c < 0 ? 0 : static_cast<int32_t>(c);
    table_out[D + d] = m < 0 ? 0 : static_cast<int32_t>(m);
    table_out[2 * D + d] = (c < 0 || m < 0) ? 1 : 0;
}

}  // namespace egpu

extern "C" int egpu_table_restore_flat(egpu_ctx* ctx, const char* ids_flat, const int64_t* id_offsets, int64_t n_ids,
                                       const int64_t* set_offsets, int64_t n_sets, const char* set_hash8,
                                       const int32_t* set_resource, const int64_t* link_offsets, const int32_t* link_gpu,
                                       const int32_t* cap_core, const int32_t* cap_mem, int32_t D, int flags,
                                       int32_t* out_table, int32_t* out_status) {
    if (!ctx || !out_table || !cap_core || !cap_mem || D < 1 || D > EGPU_MAX_DEVICES || n_sets < 0 || n_ids < 0)
        return EGPU_ERR_INVALID;
    if (flags & ~(EGPU_RESTORE_VERIFY | EGPU_RESTORE_INSTALL | EGPU_RESTORE_CHARGE | EGPU_RESTORE_RELEASE))
        return EGPU_ERR_INVALID;
    // CHARGE / RELEASE: the entries' usage against the context's current table (DESIGN.md §2.7)
    const int delta = flags & (EGPU_RESTORE_CHARGE | EGPU_RESTORE_RELEASE);
    if (delta == (EGPU_RESTORE_CHARGE | EGPU_RESTORE_RELEASE) || (delta && (flags & EGPU_RESTORE_INSTALL)))
        return EGPU_ERR_INVALID;
    for (int d = 0; d < D; ++d) {
        if (cap_core[d] < 0 || cap_core[d] > EGPU_CORE_MAX) return EGPU_ERR_INVALID;
        if (cap_mem[d] < 0 || cap_mem[d] > EGPU_MEM_MAX) return EGPU_ERR_INVALID;
    }
    const bool verify = (flags & EGPU_RESTORE_VERIFY) != 0;
    std::vector<uint32_t> stored(static_cast<size_t>(n_sets), 0);
    std::vector<int32_t> res(static_cast<size_t>(n_sets), 0);
    if (n_sets > 0) {
        if (!set_offsets || !id_offsets || !set_resource || !link_offsets || !set_hash8) return EGPU_ERR_INVALID;
        if (link_offsets[0] != 0) return EGPU_ERR_INVALID;
        for (int64_t q = 0; q < n_sets; ++q) {
            if (link_offsets[q + 1] < link_offsets[q]) return EGPU_ERR_INVALID;
            uint32_t w = 0;
            bool ok = true;
            for (int k = 0; k < 8; ++k) {
                const char c = set_hash8[q * 8 + k];
                const int v = (c >= '0' && c <= '9') ? c - '0' : (c >= 'a' && c <= 'f') ? c - 'a' + 10 : -1;
                ok = ok && v >= 0;
                w = (w << 4) | static_cast<uint32_t>(v & 15);
            }
            stored[q] = w;
            res[q] = set_resource[q];
            // a stored Hash that is not 8 lowercase hex digits can never equal a recomputed one
            if (!ok && verify && (res[q] == EGPU_RESOURCE_CORE || res[q] == EGPU_RESOURCE_MEM)) res[q] = kResBadHash;
        }
        if (link_offsets[n_sets] > 0 && !link_gpu) return EGPU_ERR_INVALID;
    }
    std::lock_guard<std::mutex> g(ctx->mu);
    if (delta && !ctx->has_table) return EGPU_ERR_NO_TABLE;
    if (delta && D != ctx->D) return EGPU_ERR_INVALID;
    EGPU_CUDA(ctx, cudaSetDevice(ctx->dev));
    cudaStream_t s = ctx->stream;
    std::vector<int32_t> table(static_cast<size_t>(3) * D, 0);
    std::vector<int32_t> status(static_cast<size_t>(n_sets), EGPU_REC_OK);
    unsigned long long usage[2 * kMaxD] = {0};  // CHARGE / RELEASE: [core 0..63, mem 64..127]
    if (n_sets == 0) {
        for (int d = 0; d < D; ++d) table[d] = cap_core[d], table[D + d] = cap_mem[d];
    } else {
        HashRun r;
        // the hash pipeline carves the arena first; the restore buffers are separate small allocations
        const int rc = run_hash(ctx, r, ids_flat, id_offsets, n_ids, set_offsets, n_sets, verify);
        if (rc != EGPU_OK) return rc;
        const int64_t n_links = link_offsets[n_sets];
        struct Tmp {
            void* p = nullptr;
            ~Tmp() { if (p) cudaFree(p); }
        } buf;
        const size_t o_stored = 0, o_res = o_stored + 4 * static_cast<size_t>(n_sets), o_status = o_res + 4 * static_cast<size_t>(n_sets);
        size_t o_loff = (o_status + 4 * static_cast<size_t>(n_sets) + 7) & ~static_cast<size_t>(7);
        const size_t o_lgpu = o_loff + 8 * static_cast<size_t>(n_sets + 1);
        size_t o_usage = (o_lgpu + 4 * static_cast<size_t>(n_links > 0 ? n_links : 1) + 7) & ~static_cast<size_t>(7);
        const size_t o_cap = o_usage + 8 * 2 * kMaxD, o_table = o_cap + 4 * 2 * kMaxD, total = o_table + 4 * 3 * kMaxD;
        EGPU_CUDA(ctx, cudaMalloc(&buf.p, total));
        char* b = static_cast<char*>(buf.p);
        int32_t cap[2 * kMaxD] = {0};
        for (int d = 0; d < D; ++d) cap[d] = cap_core[d], cap[kMaxD + d] = cap_mem[d];
        EGPU_CUDA(ctx, cudaMemcpyAsync(b + o_stored, stored.data(), 4 * n_sets, cudaMemcpyHostToDevice, s));
        EGPU_CUDA(ctx, cudaMemcpyAsync(b + o_res, res.data(), 4 * n_sets, cudaMemcpyHostToDevice, s));
        EGPU_CUDA(ctx, cudaMemcpyAsync(b + o_loff, link_offsets, 8 * (n_sets + 1), cudaMemcpyHostToDevice, s));
        if (n_links) EGPU_CUDA(ctx, cudaMemcpyAsync(b + o_lgpu, link_gpu, 4 * n_links, cudaMemcpyHostToDevice, s));
        EGPU_CUDA(ctx, cudaMemcpyAsync(b + o_cap, cap, sizeof cap, cudaMemcpyHostToDevice, s));
        EGPU_CUDA(ctx, cudaMemsetAsync(b + o_usage, 0, 8 * 2 * kMaxD, s));
        restore_usage_kernel<<<static_cast<unsigned>((n_sets + 127) / 128), 128, 0, s>>>(
            r.set_off.as<long long>(), n_sets, verify ? r.digest.as<uint32_t>() : nullptr,
            reinterpret_cast<const uint32_t*>(b + o_stored), reinterpret_cast<const int32_t*>(b + o_res),
            reinterpret_cast<const long long*>(b + o_loff), reinterpret_cast<const int32_t*>(b + o_lgpu), D,
            reinterpret_cast<unsigned long long*>(b + o_usage), reinterpret_cast<int32_t*>(b + o_status));
        ctx->launches += 1;
        if (delta) {
            // 2 x 64 sums against a table of at most 64 rows: read back, applied below
            EGPU_CUDA(ctx, cudaMemcpyAsync(usage, b + o_usage, sizeof usage, cudaMemcpyDeviceToHost, s));
        } else {
            restore_table_kernel<<<1, kMaxD, 0, s>>>(reinterpret_cast<const int32_t*>(b + o_cap),
                                                     reinterpret_cast<const unsigned long long*>(b + o_usage), D,
                                                     reinterpret_cast<int32_t*>(b + o_table));
            ctx->launches += 1;
            EGPU_CUDA(ctx, cudaMemcpyAsync(table.data(), b + o_table, 4 * 3 * static_cast<size_t>(D), cudaMemcpyDeviceToHost, s));
        }
        EGPU_CUDA(ctx, cudaGetLastError());
        EGPU_CUDA(ctx, cudaMemcpyAsync(status.data(), b + o_status, 4 * n_sets, cudaMemcpyDeviceToHost, s));
        EGPU_CUDA(ctx, cudaStreamSynchronize(s));
    }
    if (delta) {
        // the current table, read as egpu_table_get reads it: the context's stream is idle (synchronised
        // above, or nothing was enqueued), and ctx->mu keeps every other call of this context out until
        // the result is installed
        EGPU_CUDA(ctx, cudaStreamSynchronize(s));
        EGPU_CUDA(ctx, cudaMemcpy(ctx->h_table, ctx->d_state, sizeof(int32_t) * 3 * kMaxD, cudaMemcpyDeviceToHost));
        const int32_t* cur = ctx->h_table;
        for (int d = 0; d < D; ++d) {
            const long long uc = static_cast<long long>(usage[d]), um = static_cast<long long>(usage[kMaxD + d]);
            const int32_t ov = cur[2 * kMaxD + d];
            if (delta == EGPU_RESTORE_CHARGE) {
                // max(max(a, 0) - u, 0) = max(a - u, 0) for u >= 0: charging a restored table is restoring the union
                const long long c = cur[d] - uc, m = cur[kMaxD + d] - um;
                table[d] = c < 0 ? 0 : static_cast<int32_t>(c);
                table[D + d] = m < 0 ? 0 : static_cast<int32_t>(m);
                table[2 * D + d] = (ov || c < 0 || m < 0) ? 1 : 0;
                continue;
            }
            const long long c = cur[d] + uc, m = cur[kMaxD + d] + um;
            const char* why = nullptr;
            if ((uc || um) && ov) why = "is oversubscribed: the stored table lost the deficit; restore the node instead";
            else if ((uc || um) && (c > cap_core[d] || m > cap_mem[d]))
                why = "would exceed its capacity: more is released than is in use";
            if (why) {
                std::snprintf(ctx->last_err, sizeof ctx->last_err, "egpu_table_restore: release on device %d %s", d, why);
                return EGPU_ERR_STATE;
            }
            table[d] = static_cast<int32_t>(c);
            table[D + d] = static_cast<int32_t>(m);
            table[2 * D + d] = ov;
        }
    }
    std::memcpy(out_table, table.data(), sizeof(int32_t) * 3 * static_cast<size_t>(D));
    if (out_status && n_sets) std::memcpy(out_status, status.data(), sizeof(int32_t) * static_cast<size_t>(n_sets));
    // the installed table keeps the oversubscription flags, as a committing batch's table does (DESIGN.md §2.4)
    if ((flags & EGPU_RESTORE_INSTALL) || delta)
        return egpu_table_set_locked(ctx, table.data(), table.data() + D, table.data() + 2 * D, D);
    return EGPU_OK;
}

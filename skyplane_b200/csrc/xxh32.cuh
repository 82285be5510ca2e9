// xxh32.cuh -- XXH32 (seed 0), the LZ4 frame format's content and block checksum, in the pieces the kernels need:
// the four-accumulator stripe round (md5_warp runs it over the words its MD5 lanes already hold), the finish over the
// last 0-15 bytes, and a warp-wide hash of one stored block for the receiver's block checksums.
#pragma once
#include <stdint.h>

namespace sky {

constexpr uint32_t kXxhP1 = 2654435761u, kXxhP2 = 2246822519u, kXxhP3 = 3266489917u, kXxhP4 = 668265263u, kXxhP5 = 374761393u;

struct XxhState {
    uint32_t v1, v2, v3, v4;
};

__device__ __forceinline__ uint32_t xxh_rotl(uint32_t x, int s) { return __funnelshift_l(x, x, s); }

__device__ __forceinline__ void xxh_init(XxhState &x) {
    x.v1 = kXxhP1 + kXxhP2;
    x.v2 = kXxhP2;
    x.v3 = 0;
    x.v4 = 0u - kXxhP1;
}

__device__ __forceinline__ uint32_t xxh_round(uint32_t v, uint32_t w) { return xxh_rotl(v + w * kXxhP2, 13) * kXxhP1; }

// One 16-byte stripe: four little-endian words, one per accumulator.
__device__ __forceinline__ void xxh_stripe(XxhState &x, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3) {
    x.v1 = xxh_round(x.v1, w0);
    x.v2 = xxh_round(x.v2, w1);
    x.v3 = xxh_round(x.v3, w2);
    x.v4 = xxh_round(x.v4, w3);
}

// The hash before its last 0-15 bytes: the accumulators merged (inputs of 16 bytes or more) or XXH32's short form, plus
// the input length (mod 2^32).
__device__ __forceinline__ uint32_t xxh_merge(const XxhState &x, uint64_t len) {
    const uint32_t h = len >= 16 ? xxh_rotl(x.v1, 1) + xxh_rotl(x.v2, 7) + xxh_rotl(x.v3, 12) + xxh_rotl(x.v4, 18) : kXxhP5;
    return h + (uint32_t)len;
}

__device__ __forceinline__ uint32_t xxh_word(uint32_t h, uint32_t w) { return xxh_rotl(h + w * kXxhP3, 17) * kXxhP4; }
__device__ __forceinline__ uint32_t xxh_byte(uint32_t h, uint32_t b) { return xxh_rotl(h + b * kXxhP5, 11) * kXxhP1; }

__device__ __forceinline__ uint32_t xxh_avalanche(uint32_t h) {
    h ^= h >> 15;
    h *= kXxhP2;
    h ^= h >> 13;
    h *= kXxhP3;
    h ^= h >> 16;
    return h;
}

__device__ __forceinline__ uint32_t xxh_ld32(const uint8_t *p) {
    return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24);
}

// XXH32 of p[0, n) (any alignment), on every lane of the warp.  The four accumulators are serial chains, so lanes 0..3
// each run one (lane k takes word k of every stripe) and lane 0 finishes; the other lanes only wait.
__device__ __forceinline__ uint32_t xxh32_warp(const uint8_t *p, uint32_t n, unsigned lane) {
    uint32_t v = lane == 0 ? kXxhP1 + kXxhP2 : lane == 1 ? kXxhP2 : lane == 2 ? 0u : 0u - kXxhP1;
    const uint32_t nstripes = n >> 4;
    if (lane < 4) {
        const uint8_t *q = p + 4 * lane;
#pragma unroll 8
        for (uint32_t s = 0; s < nstripes; s++) v = xxh_round(v, xxh_ld32(q + 16 * s));
    }
    XxhState x;
    x.v1 = __shfl_sync(0xffffffffu, v, 0);
    x.v2 = __shfl_sync(0xffffffffu, v, 1);
    x.v3 = __shfl_sync(0xffffffffu, v, 2);
    x.v4 = __shfl_sync(0xffffffffu, v, 3);
    uint32_t h = xxh_merge(x, n);
    uint32_t k = nstripes << 4;
    for (; k + 4 <= n; k += 4) h = xxh_word(h, xxh_ld32(p + k));
    for (; k < n; k++) h = xxh_byte(h, p[k]);
    return xxh_avalanche(h);
}

}  // namespace sky

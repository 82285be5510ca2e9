// secretbox.cuh -- XSalsa20-Poly1305 (NaCl crypto_secretbox) on sm_90a, behind the LZ4 frame.
//
// Replaces, per chunk, the CPU call the sender makes when end-to-end encryption is on
//     data = nacl.secret.SecretBox(key).encrypt(data)            skyplane/gateway/operators/gateway_operator.py:362-364
// and its inverse on the receiver (skyplane/gateway/operators/gateway_receiver.py:191-193).  Layout of one box, exactly
// PyNaCl's EncryptedMessage:  nonce(24) | tag(16) | ciphertext(n).
//
//   * XSalsa20 is a counter-mode stream: subkey = HSalsa20(key, nonce[0:16]); stream block b = Salsa20(subkey,
//     nonce[16:24], counter b).  Block 0's first 32 bytes are the one-time Poly1305 key, the message is XORed with the
//     stream from byte 32 on.  One thread = one 64-byte stream block (20 rounds of add-rotate-xor on 16 registers).
//   * Poly1305 is one tag per message: h = sum(m_i * r^(n-i)) mod 2^130-5.  One CTA per message: thread t takes blocks
//     t, t+T, t+2T, ... with Horner in R = r^T, weighs its partial sum with r^(distance of its last block from the end),
//     and the CTA adds the partial sums (26-bit limbs, 64-bit products: the poly1305-donna arithmetic).
// Both are integer ALU work (about 15 + 5 ops per byte): bandwidth-trivial next to the MD5 chain of the same chunk.
#pragma once
#include <stdint.h>

namespace sky {

constexpr int kBoxOverhead = 40;   // nonce + tag
constexpr int kPolyThreads = 256;  // threads per message in the tag kernel

struct BoxChunk {
    uint8_t *box;        // nonce(24) | tag(16) | ciphertext ; box + 40 is 16-byte aligned (box = 16-byte aligned base + 8)
    const uint8_t *msg;  // plaintext (seal) -- 16-byte aligned; for open: where the plaintext goes
    uint64_t len;        // message bytes
};

// XSalsa20 stream blocks (work items of sky_box_xor_kernel) of a `len`-byte message: it starts 32 bytes into block 0.
__host__ __device__ __forceinline__ uint64_t box_stream_blocks(uint64_t len) { return (len + 32 + 63) / 64; }

__device__ __forceinline__ uint32_t rotl(uint32_t x, int s) { return __funnelshift_l(x, x, s); }

__device__ __forceinline__ void salsa20_rounds(uint32_t (&x)[16]) {
#define SKY_QR(a, b, c, d)          \
    x[b] ^= rotl(x[a] + x[d], 7);   \
    x[c] ^= rotl(x[b] + x[a], 9);   \
    x[d] ^= rotl(x[c] + x[b], 13);  \
    x[a] ^= rotl(x[d] + x[c], 18);
#pragma unroll
    for (int i = 0; i < 10; i++) {
        SKY_QR(0, 4, 8, 12) SKY_QR(5, 9, 13, 1) SKY_QR(10, 14, 2, 6) SKY_QR(15, 3, 7, 11)   // columns
        SKY_QR(0, 1, 2, 3) SKY_QR(5, 6, 7, 4) SKY_QR(10, 11, 8, 9) SKY_QR(15, 12, 13, 14)   // rows
    }
#undef SKY_QR
}

// key words k[8], 16 input bytes as words in4[4] -> Salsa20 input block
__device__ __forceinline__ void salsa_init(uint32_t (&x)[16], const uint32_t (&k)[8], const uint32_t (&in4)[4]) {
    x[0] = 0x61707865u; x[5] = 0x3320646eu; x[10] = 0x79622d32u; x[15] = 0x6b206574u;  // "expand 32-byte k"
    x[1] = k[0]; x[2] = k[1]; x[3] = k[2]; x[4] = k[3];
    x[11] = k[4]; x[12] = k[5]; x[13] = k[6]; x[14] = k[7];
    x[6] = in4[0]; x[7] = in4[1]; x[8] = in4[2]; x[9] = in4[3];
}

__device__ __forceinline__ uint32_t ld_le32(const uint8_t *p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }

// ---- per chunk: subkey (8 words) and the Poly1305 key (8 words) from key + nonce.  One thread per chunk.
// sub[c*16 + 0..7] = HSalsa20 subkey, sub[c*16 + 8..15] = first 32 bytes of stream block 0 (r | s).
__global__ void sky_box_keys_kernel(const BoxChunk *chunks, uint32_t n, const uint8_t *key32, uint32_t *sub) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    const uint8_t *nonce = chunks[c].box;  // the caller put the 24 nonce bytes there
    uint32_t k[8], in4[4], x[16];
#pragma unroll
    for (int i = 0; i < 8; i++) k[i] = ld_le32(key32 + 4 * i);
#pragma unroll
    for (int i = 0; i < 4; i++) in4[i] = ld_le32(nonce + 4 * i);
    salsa_init(x, k, in4);
    salsa20_rounds(x);
    uint32_t sk[8] = {x[0], x[5], x[10], x[15], x[6], x[7], x[8], x[9]};  // HSalsa20: no feed-forward
#pragma unroll
    for (int i = 0; i < 8; i++) sub[c * 16 + i] = sk[i];
    uint32_t in0[4] = {ld_le32(nonce + 16), ld_le32(nonce + 20), 0u, 0u}, y[16], y0[16];
    salsa_init(y, sk, in0);
#pragma unroll
    for (int i = 0; i < 16; i++) y0[i] = y[i];
    salsa20_rounds(y);
#pragma unroll
    for (int i = 0; i < 8; i++) sub[c * 16 + 8 + i] = y[i] + y0[i];
}

// ---- XOR with the XSalsa20 stream.  Work item = (chunk, stream block b): message bytes [64b - 32, 64b + 32).
// blk_base[c] = first work item of chunk c (prefix sum of box_stream_blocks(len)), total items = blk_base[n].
// seal: src = plaintext msg, dst = box + 40.   open: src = box + 40, dst = msg.
__global__ void sky_box_xor_kernel(const BoxChunk *chunks, const uint64_t *blk_base, uint32_t n, const uint32_t *sub, int open) {
    const uint64_t total = blk_base[n];
    for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < total; w += (uint64_t)gridDim.x * blockDim.x) {
        // chunk of this work item: binary search in the prefix array (n <= a few thousand)
        uint32_t lo = 0, hi = n;
        while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (blk_base[mid] <= w) lo = mid; else hi = mid;
        }
        const uint32_t c = lo;
        const uint64_t b = w - blk_base[c];
        const BoxChunk cd = chunks[c];
        uint32_t sk[8], x[16], x0[16];
#pragma unroll
        for (int i = 0; i < 8; i++) sk[i] = sub[c * 16 + i];
        const uint8_t *nonce = cd.box;
        uint32_t in4[4] = {ld_le32(nonce + 16), ld_le32(nonce + 20), (uint32_t)b, (uint32_t)(b >> 32)};
        salsa_init(x, sk, in4);
#pragma unroll
        for (int i = 0; i < 16; i++) x0[i] = x[i];
        salsa20_rounds(x);
#pragma unroll
        for (int i = 0; i < 16; i++) x[i] += x0[i];
        const uint8_t *src = open ? cd.box + kBoxOverhead : cd.msg;
        uint8_t *dst = open ? const_cast<uint8_t *>(cd.msg) : cd.box + kBoxOverhead;
        // stream bytes [0,32) of block b pair with message bytes [64b-32, 64b) (none for b == 0); [32,64) with [64b, 64b+32)
#pragma unroll
        for (int half = 0; half < 2; half++) {
            if (b == 0 && half == 0) continue;
            const uint64_t m0 = 64 * b - 32 + 32 * half;
            if (m0 >= cd.len) continue;
            const uint32_t avail = (uint32_t)min((uint64_t)32, cd.len - m0);
            if (avail == 32) {
                const uint4 a = *reinterpret_cast<const uint4 *>(src + m0), bq = *reinterpret_cast<const uint4 *>(src + m0 + 16);
                uint4 o0, o1;
                o0.x = a.x ^ x[8 * half + 0]; o0.y = a.y ^ x[8 * half + 1]; o0.z = a.z ^ x[8 * half + 2]; o0.w = a.w ^ x[8 * half + 3];
                o1.x = bq.x ^ x[8 * half + 4]; o1.y = bq.y ^ x[8 * half + 5]; o1.z = bq.z ^ x[8 * half + 6]; o1.w = bq.w ^ x[8 * half + 7];
                *reinterpret_cast<uint4 *>(dst + m0) = o0;
                *reinterpret_cast<uint4 *>(dst + m0 + 16) = o1;
            } else {
                for (uint32_t i = 0; i < avail; i++) dst[m0 + i] = src[m0 + i] ^ (uint8_t)(x[8 * half + (i >> 2)] >> (8 * (i & 3)));
            }
        }
    }
}

// ---- Poly1305 in 5 x 26-bit limbs
struct P1305 {
    uint32_t h[5];
};
__device__ __forceinline__ P1305 p_mul(const P1305 &a, const P1305 &r) {
    const uint64_t r0 = r.h[0], r1 = r.h[1], r2 = r.h[2], r3 = r.h[3], r4 = r.h[4];
    const uint64_t s1 = r1 * 5, s2 = r2 * 5, s3 = r3 * 5, s4 = r4 * 5;
    const uint64_t h0 = a.h[0], h1 = a.h[1], h2 = a.h[2], h3 = a.h[3], h4 = a.h[4];
    uint64_t d0 = h0 * r0 + h1 * s4 + h2 * s3 + h3 * s2 + h4 * s1;
    uint64_t d1 = h0 * r1 + h1 * r0 + h2 * s4 + h3 * s3 + h4 * s2;
    uint64_t d2 = h0 * r2 + h1 * r1 + h2 * r0 + h3 * s4 + h4 * s3;
    uint64_t d3 = h0 * r3 + h1 * r2 + h2 * r1 + h3 * r0 + h4 * s4;
    uint64_t d4 = h0 * r4 + h1 * r3 + h2 * r2 + h3 * r1 + h4 * r0;
    P1305 o;
    uint64_t c = d0 >> 26; o.h[0] = (uint32_t)d0 & 0x3ffffff;
    d1 += c; c = d1 >> 26; o.h[1] = (uint32_t)d1 & 0x3ffffff;
    d2 += c; c = d2 >> 26; o.h[2] = (uint32_t)d2 & 0x3ffffff;
    d3 += c; c = d3 >> 26; o.h[3] = (uint32_t)d3 & 0x3ffffff;
    d4 += c; c = d4 >> 26; o.h[4] = (uint32_t)d4 & 0x3ffffff;
    const uint32_t t = o.h[0] + (uint32_t)c * 5;
    o.h[0] = t & 0x3ffffff;
    o.h[1] += t >> 26;
    return o;
}
// 16 message bytes (as 4 LE words) + the 2^128 bit (hibit = 1 << 24, or 0 for a padded final block) added to acc
__device__ __forceinline__ void p_add_block(P1305 &acc, uint32_t w0, uint32_t w1, uint32_t w2, uint32_t w3, uint32_t hibit) {
    acc.h[0] += w0 & 0x3ffffff;
    acc.h[1] += ((w0 >> 26) | (w1 << 6)) & 0x3ffffff;
    acc.h[2] += ((w1 >> 20) | (w2 << 12)) & 0x3ffffff;
    acc.h[3] += ((w2 >> 14) | (w3 << 18)) & 0x3ffffff;
    acc.h[4] += (w3 >> 8) | hibit;
}

// One CTA (kPolyThreads) per chunk: tag over the ciphertext at box + 40.  open != 0: compare with the stored tag and
// write status[c] = 0 / kBoxAuthFailed instead of storing the tag.
constexpr int32_t kBoxAuthFailed = -7;
__global__ void __launch_bounds__(kPolyThreads) sky_box_tag_kernel(const BoxChunk *chunks, const uint32_t *sub, int open, int32_t *status) {
    __shared__ P1305 pw[kPolyThreads];      // pw[i] = r^(i+1)
    __shared__ uint64_t red[5][kPolyThreads / 32];
    const uint32_t c = blockIdx.x, t = threadIdx.x;
    const BoxChunk cd = chunks[c];
    const uint8_t *m = cd.box + kBoxOverhead;
    // r (clamped) and s
    uint32_t k[8];
#pragma unroll
    for (int i = 0; i < 8; i++) k[i] = sub[c * 16 + 8 + i];
    P1305 r;
    r.h[0] = k[0] & 0x3ffffff;
    r.h[1] = ((k[0] >> 26) | (k[1] << 6)) & 0x3ffff03;
    r.h[2] = ((k[1] >> 20) | (k[2] << 12)) & 0x3ffc0ff;
    r.h[3] = ((k[2] >> 14) | (k[3] << 18)) & 0x3f03fff;
    r.h[4] = (k[3] >> 8) & 0x00fffff;
    {   // r^(t+1) by square-and-multiply
        P1305 base = r, acc;
        acc.h[0] = 1; acc.h[1] = acc.h[2] = acc.h[3] = acc.h[4] = 0;
        uint32_t e = t + 1;
        while (e) {
            if (e & 1) acc = p_mul(acc, base);
            base = p_mul(base, base);
            e >>= 1;
        }
        pw[t] = acc;
    }
    __syncthreads();
    const P1305 R = pw[kPolyThreads - 1];
    const uint64_t nblk = (cd.len + 15) / 16;
    P1305 acc;
    acc.h[0] = acc.h[1] = acc.h[2] = acc.h[3] = acc.h[4] = 0;
    uint64_t last = 0;
    bool any = false;
    for (uint64_t b = t; b < nblk; b += kPolyThreads) {
        if (any) acc = p_mul(acc, R);
        const uint64_t o = b * 16;
        if (o + 16 <= cd.len) {
            const uint4 v = *reinterpret_cast<const uint4 *>(m + o);  // m is 16-byte aligned
            p_add_block(acc, v.x, v.y, v.z, v.w, 1u << 24);
        } else {
            uint32_t w[4] = {0, 0, 0, 0};
            const uint32_t rem = (uint32_t)(cd.len - o);
            for (uint32_t i = 0; i < rem; i++) w[i >> 2] |= (uint32_t)m[o + i] << (8 * (i & 3));
            w[rem >> 2] |= 1u << (8 * (rem & 3));
            p_add_block(acc, w[0], w[1], w[2], w[3], 0);
        }
        any = true;
        last = b;
    }
    // weigh with r^(nblk - last) and add up over the CTA (limb sums stay below 2^34)
    uint64_t part[5] = {0, 0, 0, 0, 0};
    if (any) {
        const P1305 wgt = p_mul(acc, pw[(uint32_t)(nblk - last) - 1]);
#pragma unroll
        for (int i = 0; i < 5; i++) part[i] = wgt.h[i];
    }
#pragma unroll
    for (int i = 0; i < 5; i++) {
        uint64_t v = part[i];
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
        if ((t & 31) == 0) red[i][t >> 5] = v;
    }
    __syncthreads();
    if (t == 0) {
        uint64_t h[5];
#pragma unroll
        for (int i = 0; i < 5; i++) {
            h[i] = 0;
            for (int wdx = 0; wdx < kPolyThreads / 32; wdx++) h[i] += red[i][wdx];
        }
        // carry, then full reduction mod 2^130 - 5 (poly1305-donna's finish)
        uint64_t cy;
        cy = h[0] >> 26; h[0] &= 0x3ffffff; h[1] += cy;
        cy = h[1] >> 26; h[1] &= 0x3ffffff; h[2] += cy;
        cy = h[2] >> 26; h[2] &= 0x3ffffff; h[3] += cy;
        cy = h[3] >> 26; h[3] &= 0x3ffffff; h[4] += cy;
        cy = h[4] >> 26; h[4] &= 0x3ffffff; h[0] += cy * 5;
        cy = h[0] >> 26; h[0] &= 0x3ffffff; h[1] += cy;
        cy = h[1] >> 26; h[1] &= 0x3ffffff; h[2] += cy;
        cy = h[2] >> 26; h[2] &= 0x3ffffff; h[3] += cy;
        cy = h[3] >> 26; h[3] &= 0x3ffffff; h[4] += cy;
        cy = h[4] >> 26; h[4] &= 0x3ffffff; h[0] += cy * 5;
        cy = h[0] >> 26; h[0] &= 0x3ffffff; h[1] += cy;
        uint32_t h0 = (uint32_t)h[0], h1 = (uint32_t)h[1], h2 = (uint32_t)h[2], h3 = (uint32_t)h[3], h4 = (uint32_t)h[4];
        uint32_t g0 = h0 + 5, g1, g2, g3, g4, cc;
        cc = g0 >> 26; g0 &= 0x3ffffff;
        g1 = h1 + cc; cc = g1 >> 26; g1 &= 0x3ffffff;
        g2 = h2 + cc; cc = g2 >> 26; g2 &= 0x3ffffff;
        g3 = h3 + cc; cc = g3 >> 26; g3 &= 0x3ffffff;
        g4 = h4 + cc - (1u << 26);
        const uint32_t mask = (g4 >> 31) - 1;  // all ones if h >= p
        h0 = (h0 & ~mask) | (g0 & mask); h1 = (h1 & ~mask) | (g1 & mask); h2 = (h2 & ~mask) | (g2 & mask);
        h3 = (h3 & ~mask) | (g3 & mask); h4 = (h4 & ~mask) | (g4 & mask);
        const uint32_t t0 = h0 | (h1 << 26), t1 = (h1 >> 6) | (h2 << 20), t2 = (h2 >> 12) | (h3 << 14), t3 = (h3 >> 18) | (h4 << 8);
        uint64_t f;
        uint32_t tag[4];
        f = (uint64_t)t0 + k[4]; tag[0] = (uint32_t)f;
        f = (uint64_t)t1 + k[5] + (f >> 32); tag[1] = (uint32_t)f;
        f = (uint64_t)t2 + k[6] + (f >> 32); tag[2] = (uint32_t)f;
        f = (uint64_t)t3 + k[7] + (f >> 32); tag[3] = (uint32_t)f;
        uint8_t *tp = cd.box + 24;
        if (open) {
            uint32_t diff = 0;
            for (int i = 0; i < 16; i++) diff |= tp[i] ^ (uint8_t)(tag[i >> 2] >> (8 * (i & 3)));
            status[c] = diff ? kBoxAuthFailed : 0;
        } else {
            for (int i = 0; i < 16; i++) tp[i] = (uint8_t)(tag[i >> 2] >> (8 * (i & 3)));
        }
    }
}

}  // namespace sky

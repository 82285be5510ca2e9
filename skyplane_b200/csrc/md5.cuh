// md5.cuh -- RFC 1321 MD5, one digest stream per lane, for sm_90a.
//
// Replaces hashlib.md5().update()/digest() at skyplane/obj_store/s3_interface.py:181-192.
// One chunk is ONE serial chain (the digest must equal hashlib.md5(whole chunk)), so a warp
// carries 32 chunks, lane = chunk.  The per-step dependent chain is 3 SASS ops, all on the ALU pipe:
//   LOP3 (F/G/H/I of the newest b) -> IADD3 (+ (a + M[g]) + K[i]; a + M[g] is an IMAD on the FMA pipe, off the chain)
//   -> LEA.HI (b + rotl(t, s): ptxas fuses the funnel shift and the add).
// Each ALU -> ALU hop is 4 cycles, so a step is scheduled at 12 (tools/md5_schedule.py reads it from the SASS).
// Message words are staged into shared memory with 16-byte cp.async a ring's depth of blocks ahead of the chain (ring of
// kSlots x 64 B per lane, laid out [slot][piece][lane] so LDS.128 is conflict-free): SKY_MD5_SLOTS = 8 on the sender,
// whose copies compete with the compressors' stream, 4 on the receiver.
#pragma once
#include <stdint.h>
#include "xxh32.cuh"
#include <type_traits>
#include <utility>

#ifndef SKY_MD5_SLOTS
#define SKY_MD5_SLOTS 8
#endif

namespace sky {

#ifdef SKY_MD5_TRACE
// Diagnostic build only (tools/build_variants.py md5_trace, read by tools/md5_trace.py): lane 0 of each sender MD5 warp
// stamps %globaltimer and %clock at its group's start and end and every kTraceEvery blocks, and sums the cycles the warp
// spends in the ring's cp.async wait.  The default build has none of this.
constexpr int kTraceGroups = 256, kTraceStamps = 512, kTraceEvery = 1024;
struct Md5TraceStamp {
    uint64_t t;     // %globaltimer (ns)
    uint32_t clk;   // %clock
    uint32_t wait;  // ring-wait cycles so far
};
struct Md5Trace {
    uint32_t smid, warpid, cta, stamps;
    uint64_t t0, t1;
    uint32_t c0, c1, wait, blocks;
    Md5TraceStamp s[kTraceStamps];  // s[k]: after block (k + 1) * kTraceEvery
};
__device__ Md5Trace g_md5_trace[kTraceGroups];
__device__ __forceinline__ uint64_t trace_globaltimer() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ uint32_t trace_clock() {
    uint32_t c;
    asm volatile("mov.u32 %0, %%clock;" : "=r"(c));
    return c;
}
__device__ __forceinline__ uint32_t trace_smid() {
    uint32_t s;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
    return s;
}
__device__ __forceinline__ uint32_t trace_warpid() {
    uint32_t w;
    asm volatile("mov.u32 %0, %%warpid;" : "=r"(w));
    return w;
}
#define SKY_MD5_TRACE_PARAM , Md5Trace *trace = nullptr
#else
#define SKY_MD5_TRACE_PARAM
#endif

struct Md5State {
    uint32_t a, b, c, d;
};

__device__ __forceinline__ void md5_init(Md5State &s) {
    s.a = 0x67452301u;
    s.b = 0xefcdab89u;
    s.c = 0x98badcfeu;
    s.d = 0x10325476u;
}

// a + M[g] is formed as M[g] * one + a, where `one` is 1 but ptxas cannot prove it (md5_one), so it stays an IMAD
// on the FMA pipe, off the chain.  The on-chain add F + (a + M[g]) + K[i] is then one IADD3 with an immediate, which
// has no IMAD form.  With a plain add ptxas forms a + M[g] + K[i] as the off-chain IADD3 and moves the on-chain add
// to the FMA pipe as IMAD.IADD, and each hop between the pipes costs 5 cycles instead of 4 (14 cycles per step).
__device__ __forceinline__ uint32_t md5_am(uint32_t a, uint32_t m, uint32_t one) {
    uint32_t r;
    asm("mad.lo.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(m), "r"(one), "r"(a));
    return r;
}
// 1, read from special registers: the only bit set in %lanemask_eq is bit %laneid.
__device__ __forceinline__ uint32_t md5_one() {
    uint32_t eq, lane;
    asm("mov.u32 %0, %%lanemask_eq;" : "=r"(eq));
    asm("mov.u32 %0, %%laneid;" : "=r"(lane));
    return eq >> lane;
}
#define SKY_MD5_STEP(FN, a, b, c, d, m, k, s)                      \
    {                                                              \
        uint32_t t_ = FN(b, c, d) + md5_am(a, (m), one) + (k);     \
        a = b + __funnelshift_l(t_, t_, s);                        \
    }
#define SKY_F(b, c, d) ((d) ^ ((b) & ((c) ^ (d))))
#define SKY_G(b, c, d) ((c) ^ ((d) & ((b) ^ (c))))
#define SKY_H(b, c, d) ((b) ^ (c) ^ (d))
#define SKY_I(b, c, d) ((c) ^ ((b) | ~(d)))

// Round R (16 steps) of one 64-byte block on the working state; w[16] = little-endian message words, one = md5_one().
// md5_warp interleaves its staging between the rounds, so they are separate functions.
template <int R>
__device__ __forceinline__ void md5_round(uint32_t &a, uint32_t &b, uint32_t &c, uint32_t &d, const uint32_t (&w)[16],
                                          uint32_t one) {
    if constexpr (R == 0) {
        SKY_MD5_STEP(SKY_F, a, b, c, d, w[0], 0xd76aa478, 7)
        SKY_MD5_STEP(SKY_F, d, a, b, c, w[1], 0xe8c7b756, 12)
        SKY_MD5_STEP(SKY_F, c, d, a, b, w[2], 0x242070db, 17)
        SKY_MD5_STEP(SKY_F, b, c, d, a, w[3], 0xc1bdceee, 22)
        SKY_MD5_STEP(SKY_F, a, b, c, d, w[4], 0xf57c0faf, 7)
        SKY_MD5_STEP(SKY_F, d, a, b, c, w[5], 0x4787c62a, 12)
        SKY_MD5_STEP(SKY_F, c, d, a, b, w[6], 0xa8304613, 17)
        SKY_MD5_STEP(SKY_F, b, c, d, a, w[7], 0xfd469501, 22)
        SKY_MD5_STEP(SKY_F, a, b, c, d, w[8], 0x698098d8, 7)
        SKY_MD5_STEP(SKY_F, d, a, b, c, w[9], 0x8b44f7af, 12)
        SKY_MD5_STEP(SKY_F, c, d, a, b, w[10], 0xffff5bb1, 17)
        SKY_MD5_STEP(SKY_F, b, c, d, a, w[11], 0x895cd7be, 22)
        SKY_MD5_STEP(SKY_F, a, b, c, d, w[12], 0x6b901122, 7)
        SKY_MD5_STEP(SKY_F, d, a, b, c, w[13], 0xfd987193, 12)
        SKY_MD5_STEP(SKY_F, c, d, a, b, w[14], 0xa679438e, 17)
        SKY_MD5_STEP(SKY_F, b, c, d, a, w[15], 0x49b40821, 22)
    } else if constexpr (R == 1) {
        SKY_MD5_STEP(SKY_G, a, b, c, d, w[1], 0xf61e2562, 5)
        SKY_MD5_STEP(SKY_G, d, a, b, c, w[6], 0xc040b340, 9)
        SKY_MD5_STEP(SKY_G, c, d, a, b, w[11], 0x265e5a51, 14)
        SKY_MD5_STEP(SKY_G, b, c, d, a, w[0], 0xe9b6c7aa, 20)
        SKY_MD5_STEP(SKY_G, a, b, c, d, w[5], 0xd62f105d, 5)
        SKY_MD5_STEP(SKY_G, d, a, b, c, w[10], 0x02441453, 9)
        SKY_MD5_STEP(SKY_G, c, d, a, b, w[15], 0xd8a1e681, 14)
        SKY_MD5_STEP(SKY_G, b, c, d, a, w[4], 0xe7d3fbc8, 20)
        SKY_MD5_STEP(SKY_G, a, b, c, d, w[9], 0x21e1cde6, 5)
        SKY_MD5_STEP(SKY_G, d, a, b, c, w[14], 0xc33707d6, 9)
        SKY_MD5_STEP(SKY_G, c, d, a, b, w[3], 0xf4d50d87, 14)
        SKY_MD5_STEP(SKY_G, b, c, d, a, w[8], 0x455a14ed, 20)
        SKY_MD5_STEP(SKY_G, a, b, c, d, w[13], 0xa9e3e905, 5)
        SKY_MD5_STEP(SKY_G, d, a, b, c, w[2], 0xfcefa3f8, 9)
        SKY_MD5_STEP(SKY_G, c, d, a, b, w[7], 0x676f02d9, 14)
        SKY_MD5_STEP(SKY_G, b, c, d, a, w[12], 0x8d2a4c8a, 20)
    } else if constexpr (R == 2) {
        SKY_MD5_STEP(SKY_H, a, b, c, d, w[5], 0xfffa3942, 4)
        SKY_MD5_STEP(SKY_H, d, a, b, c, w[8], 0x8771f681, 11)
        SKY_MD5_STEP(SKY_H, c, d, a, b, w[11], 0x6d9d6122, 16)
        SKY_MD5_STEP(SKY_H, b, c, d, a, w[14], 0xfde5380c, 23)
        SKY_MD5_STEP(SKY_H, a, b, c, d, w[1], 0xa4beea44, 4)
        SKY_MD5_STEP(SKY_H, d, a, b, c, w[4], 0x4bdecfa9, 11)
        SKY_MD5_STEP(SKY_H, c, d, a, b, w[7], 0xf6bb4b60, 16)
        SKY_MD5_STEP(SKY_H, b, c, d, a, w[10], 0xbebfbc70, 23)
        SKY_MD5_STEP(SKY_H, a, b, c, d, w[13], 0x289b7ec6, 4)
        SKY_MD5_STEP(SKY_H, d, a, b, c, w[0], 0xeaa127fa, 11)
        SKY_MD5_STEP(SKY_H, c, d, a, b, w[3], 0xd4ef3085, 16)
        SKY_MD5_STEP(SKY_H, b, c, d, a, w[6], 0x04881d05, 23)
        SKY_MD5_STEP(SKY_H, a, b, c, d, w[9], 0xd9d4d039, 4)
        SKY_MD5_STEP(SKY_H, d, a, b, c, w[12], 0xe6db99e5, 11)
        SKY_MD5_STEP(SKY_H, c, d, a, b, w[15], 0x1fa27cf8, 16)
        SKY_MD5_STEP(SKY_H, b, c, d, a, w[2], 0xc4ac5665, 23)
    } else {
        SKY_MD5_STEP(SKY_I, a, b, c, d, w[0], 0xf4292244, 6)
        SKY_MD5_STEP(SKY_I, d, a, b, c, w[7], 0x432aff97, 10)
        SKY_MD5_STEP(SKY_I, c, d, a, b, w[14], 0xab9423a7, 15)
        SKY_MD5_STEP(SKY_I, b, c, d, a, w[5], 0xfc93a039, 21)
        SKY_MD5_STEP(SKY_I, a, b, c, d, w[12], 0x655b59c3, 6)
        SKY_MD5_STEP(SKY_I, d, a, b, c, w[3], 0x8f0ccc92, 10)
        SKY_MD5_STEP(SKY_I, c, d, a, b, w[10], 0xffeff47d, 15)
        SKY_MD5_STEP(SKY_I, b, c, d, a, w[1], 0x85845dd1, 21)
        SKY_MD5_STEP(SKY_I, a, b, c, d, w[8], 0x6fa87e4f, 6)
        SKY_MD5_STEP(SKY_I, d, a, b, c, w[15], 0xfe2ce6e0, 10)
        SKY_MD5_STEP(SKY_I, c, d, a, b, w[6], 0xa3014314, 15)
        SKY_MD5_STEP(SKY_I, b, c, d, a, w[13], 0x4e0811a1, 21)
        SKY_MD5_STEP(SKY_I, a, b, c, d, w[4], 0xf7537e82, 6)
        SKY_MD5_STEP(SKY_I, d, a, b, c, w[11], 0xbd3af235, 10)
        SKY_MD5_STEP(SKY_I, c, d, a, b, w[2], 0x2ad7d2bb, 15)
        SKY_MD5_STEP(SKY_I, b, c, d, a, w[9], 0xeb86d391, 21)
    }
}

// One 64-byte block.
__device__ __forceinline__ void md5_block(Md5State &st, const uint32_t (&w)[16], uint32_t one) {
    uint32_t a = st.a, b = st.b, c = st.c, d = st.d;
    md5_round<0>(a, b, c, d, w, one);
    md5_round<1>(a, b, c, d, w, one);
    md5_round<2>(a, b, c, d, w, one);
    md5_round<3>(a, b, c, d, w, one);
    st.a += a;
    st.b += b;
    st.c += c;
    st.d += d;
}

// Stages one 64-byte block from `gptr` into ring slot `kSlot` of this lane (`lane_ring` = shared address of the lane's
// piece 0 of slot 0; pieces are 512 B apart, slots 2 KiB), if `pred`.  The predicate is applied inside the asm, so no
// branch goes around the copies, and the slot offsets are immediates.
template <int kSlot>
__device__ __forceinline__ void cp_async_block(bool pred, uint32_t lane_ring, const uint8_t *gptr) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %2, 0;\n\t"
        "@p cp.async.cg.shared.global [%0+%3], [%1], 16;\n\t"
        "@p cp.async.cg.shared.global [%0+%4], [%1+16], 16;\n\t"
        "@p cp.async.cg.shared.global [%0+%5], [%1+32], 16;\n\t"
        "@p cp.async.cg.shared.global [%0+%6], [%1+48], 16;\n\t}" ::"r"(lane_ring),
        "l"(gptr), "r"((uint32_t)pred), "n"(kSlot * 2048), "n"(kSlot * 2048 + 512), "n"(kSlot * 2048 + 1024),
        "n"(kSlot * 2048 + 1536)
        : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(N) : "memory");
}

// f(std::integral_constant<int, 0>()), ..., f(std::integral_constant<int, N - 1>()): an unrolled loop whose index is a
// constant expression (ring slots are template arguments of cp_async_block).
template <class F, int... I>
__device__ __forceinline__ void md5_unroll_(F &&f, std::integer_sequence<int, I...>) {
    (f(std::integral_constant<int, I>()), ...);
}
template <int N, class F>
__device__ __forceinline__ void md5_unroll(F &&f) {
    md5_unroll_(f, std::make_integer_sequence<int, N>());
}

// md5_warp<true> also runs XXH32 (the LZ4 content checksum) over the same words: one 16-byte stripe after each MD5 round,
// where its four short chains fill issue slots the MD5 chain leaves idle.
// Digest of one chunk per lane.  `ring` = this warp's kSlots x 2 KiB shared-memory area,
// `src` 16-byte aligned (or len == 0), `active` false for lanes without a chunk.
// Writes 16 digest bytes to `out` for active lanes.  kXxh: also returns XXH32(chunk, seed 0) (0 without kXxh or when
// the lane is inactive).
// `gate(row, wants)`: called (warp-converged) before the first byte of 64 KiB row `row` is fetched; `wants` tells
// whether this lane has data in that row.  The receiver side uses it to wait until the row has been decoded.
struct Md5NoGate {
    __device__ __forceinline__ void operator()(uint64_t, bool) const {}
};

template <bool kXxh = false, class Gate = Md5NoGate, int kSlots = SKY_MD5_SLOTS>
__device__ __forceinline__ uint32_t md5_warp(uint32_t *ring, const uint8_t *src, uint64_t len, bool active, uint8_t *out,
                                             unsigned lane, Gate gate = Gate() SKY_MD5_TRACE_PARAM) {
    // kSlots: ring depth in blocks and the prefetch distance -- block i + kSlots is staged into block i's slot while block
    // i is hashed (its words are in registers by then).  The loop body is kUnroll blocks whatever the depth: a deeper
    // ring only moves where the copies land, not the chain's instruction stream.
    constexpr int kUnroll = 4;
    static_assert((kSlots & (kSlots - 1)) == 0 && kSlots % kUnroll == 0 && 1024 % kSlots == 0,
                  "the MD5 ring: a power of two, a multiple of 4 and at most 1024 blocks");
    constexpr bool kGated = !std::is_same<Gate, Md5NoGate>::value;
    // Block counts are 32-bit: the host rejects chunks over 128 GiB (kMaxChunkBlocks in skychunk.cu), so nfull <= 2^31
    // and the trip count rounded up to kUnroll cannot wrap.
    const uint32_t nfull = active ? (uint32_t)(len >> 6) : 0;
    const uint32_t wmax = __reduce_max_sync(0xffffffffu, nfull);
    const uint32_t trips = (wmax + (kUnroll - 1)) & ~(uint32_t)(kUnroll - 1);
    Md5State st;  // runs on through the blocks past this lane's end (the loop has no branch per lane) ...
    md5_init(st);
    Md5State fin = st;  // ... so the state after the lane's last full block is kept here, off the chain
    XxhState xs, xfin;  // (kXxh) the same for the XXH32 accumulators
    if constexpr (kXxh) {
        xxh_init(xs);
        xfin = xs;
    }
    // slot s, piece q of this lane lives at ring[((s*4 + q)*32 + lane) * 4 words]: a per-lane base plus an immediate
    const uint32_t *lring = ring + lane * 4;
    const uint32_t lring_s = (uint32_t)__cvta_generic_to_shared(lring);
    const uint32_t one = md5_one();
#ifdef SKY_MD5_TRACE
    uint32_t wait_cycles = 0;
    if (trace && lane == 0) {
        trace->smid = trace_smid();
        trace->warpid = trace_warpid();
        trace->cta = blockIdx.x;
        trace->t0 = trace_globaltimer();
        trace->c0 = trace_clock();
    }
#endif

    gate(0, active && len > 0);
    md5_unroll<kSlots>([&](auto sc) {
        constexpr int s = decltype(sc)::value;
        cp_async_block<s>((uint32_t)s < nfull, lring_s, src + s * 64);
        cp_async_commit();
    });
    // the words of the block in the slot at byte offset `so` of the ring (a multiple of 2 KiB)
    auto load_words = [&](uint32_t (&w)[16], uint32_t so) {
#pragma unroll
        for (int q = 0; q < 4; q++) {
            const uint4 v = *reinterpret_cast<const uint4 *>(lring + so / 4 + q * 128);
            w[4 * q + 0] = v.x;
            w[4 * q + 1] = v.y;
            w[4 * q + 2] = v.z;
            w[4 * q + 3] = v.w;
        }
    };
    // Software pipeline over two word buffers: the words of block i+1 are pulled from the ring (LDS) while block i's
    // chain runs.  Every lane hashes every block up to `trips`; a lane past its end hashes stale ring words and keeps
    // only `fin`.
    uint32_t w[2][16];
    cp_async_wait<kSlots - 1>();  // block 0 has landed
    load_words(w[0], 0);
    const uint8_t *pf_src = src + kSlots * 64;  // block i + kSlots, the next one to stage
    // Blocks i .. i + kUnroll - 1 (i a multiple of kUnroll) as one branch-free stretch: the staging sits between the
    // rounds, where ptxas can issue it in the chain's idle cycles.  Their slots are consecutive from block i's, so each
    // is the stretch's ring offset (off the chain, once per stretch) plus an immediate.
    auto blocks = [&](uint32_t i) {
        const uint32_t so = (i & (kSlots - 1)) * 2048, so_next = ((i + kUnroll) & (kSlots - 1)) * 2048;
        md5_unroll<kUnroll>([&](auto uc) {
            constexpr int u = decltype(uc)::value;
            uint32_t a = st.a, b = st.b, c = st.c, d = st.d;
            const uint32_t(&wu)[16] = w[u & 1];
            auto stripe = [&](int q) {
                if constexpr (kXxh) xxh_stripe(xs, wu[4 * q], wu[4 * q + 1], wu[4 * q + 2], wu[4 * q + 3]);
            };
            md5_round<0>(a, b, c, d, wu, one);
            stripe(0);
            cp_async_block<u>(i + u + kSlots < nfull, lring_s + so, pf_src + u * 64);  // block i+u+kSlots into block i+u's slot
            md5_round<1>(a, b, c, d, wu, one);
            stripe(1);
            cp_async_commit();
#ifdef SKY_MD5_TRACE
            const uint32_t wait_from = trace_clock();
#endif
            cp_async_wait<kSlots - 1>();  // block i+u+1 has landed
#ifdef SKY_MD5_TRACE
            wait_cycles += trace_clock() - wait_from;
#endif
            md5_round<2>(a, b, c, d, wu, one);
            stripe(2);
            load_words(w[(u + 1) & 1], u + 1 < kUnroll ? so + (u + 1) * 2048 : so_next);
            md5_round<3>(a, b, c, d, wu, one);
            stripe(3);
            st.a += a;
            st.b += b;
            st.c += c;
            st.d += d;
            if (i + u < nfull) {
                fin = st;
                if constexpr (kXxh) xfin = xs;
            }
        });
        pf_src += kUnroll * 64;
    };
    if constexpr (kGated) {
        // Receiver side: a row-granular outer loop keeps the gate (a spin with a scheduling barrier) out of the
        // chain-bound inner loop; the prefetch runs kSlots blocks ahead, so a row is gated one row early.  A row
        // (1024 blocks) is a whole number of kUnroll-block stretches.
        for (uint32_t base = 0; base < trips; base += 1024) {
            gate((base >> 10) + 1, (uint64_t)(base + 1024) * 64 < len);
            const uint32_t iend = min(base + 1024, trips);
            for (uint32_t i = base; i < iend; i += kUnroll) blocks(i);
        }
    } else {
        // Sender side: one flat loop (measured 1.027x faster per block than the nested form).
        for (uint32_t i = 0; i < trips; i += kUnroll) {
            blocks(i);
#ifdef SKY_MD5_TRACE
            const uint32_t done = i + kUnroll;
            if (trace && lane == 0 && done % kTraceEvery == 0 && done / kTraceEvery <= kTraceStamps)
                trace->s[done / kTraceEvery - 1] = Md5TraceStamp{trace_globaltimer(), trace_clock(), wait_cycles};
#endif
        }
    }
#ifdef SKY_MD5_TRACE
    if (trace && lane == 0) {
        trace->t1 = trace_globaltimer();
        trace->c1 = trace_clock();
        trace->wait = wait_cycles;
        trace->blocks = trips;
        trace->stamps = min(trips / kTraceEvery, (uint32_t)kTraceStamps);
    }
#endif
    cp_async_wait<0>();
    st = fin;
    uint32_t xxh = 0;
    if (active) {
        // tail: rem bytes + 0x80 + zeros + u64le bit length -> one or two more blocks (slow path, once per chunk)
        const uint32_t rem = (uint32_t)(len & 63);
        const uint8_t *tp = src + ((uint64_t)nfull << 6);
        uint32_t tw[32];
#pragma unroll
        for (int k = 0; k < 32; k++) tw[k] = 0;
        for (uint32_t k = 0; k < rem; k++) tw[k >> 2] |= (uint32_t)tp[k] << (8 * (k & 3));
        if constexpr (kXxh) {
            // XXH32 of the tail: its 0-3 whole stripes, then 4-byte words, then single bytes, then the avalanche
            xs = xfin;
            const uint32_t nstripes = rem >> 4;
            for (uint32_t q = 0; q < nstripes; q++) xxh_stripe(xs, tw[4 * q], tw[4 * q + 1], tw[4 * q + 2], tw[4 * q + 3]);
            uint32_t h = xxh_merge(xs, len);
            for (uint32_t k = 4 * nstripes; k < (rem >> 2); k++) h = xxh_word(h, tw[k]);
            for (uint32_t k = rem & ~3u; k < rem; k++) h = xxh_byte(h, (tw[k >> 2] >> (8 * (k & 3))) & 0xffu);
            xxh = xxh_avalanche(h);
        }
        tw[rem >> 2] |= 0x80u << (8 * (rem & 3));
        const bool two = rem >= 56;
        const uint64_t bits = len << 3;
        tw[two ? 30 : 14] = (uint32_t)bits;
        tw[two ? 31 : 15] = (uint32_t)(bits >> 32);
        for (int t = 0; t < (two ? 2 : 1); t++) {
            uint32_t w[16];
#pragma unroll
            for (int k = 0; k < 16; k++) w[k] = tw[16 * t + k];
            md5_block(st, w, one);
        }
        uint4 dg = make_uint4(st.a, st.b, st.c, st.d);
        *reinterpret_cast<uint4 *>(out) = dg;  // out is 16-byte aligned (md5 array base is 256-aligned)
    }
    return xxh;
}

}  // namespace sky

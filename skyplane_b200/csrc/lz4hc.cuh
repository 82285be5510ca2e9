// lz4hc.cuh -- high-ratio LZ4 block compressor for sm_90a (SKY_F_HC): exact hash chains, a bounded search per position
// and a lazy parse, in the same frame layout as the fast compressor (independent 64 KiB blocks, stored-raw fallback).
//
// tools/lz4hc_model.c is the sequential twin: it states the chain rule, candidate order, tie rule, lazy rule and emission,
// and the frames of this kernel are byte-identical to it (tests/test_gpu_hc.py).  One CTA owns one 64 KiB block at a time,
// claimed row-major from the batch's work counter (claim_block), in five steps:
//   load   : one bulk async copy of the block into shared memory (the head table is cleared meanwhile);
//   chains : warp 0 inserts the positions 32 at a time.  A lane's predecessor is the highest lower lane with its hash
//            (match.any), else head[hash]; then the highest lane of each hash writes head.  That is sequential insertion.
//            chain[p] is the distance to p's predecessor (u16, 0 = none), head[h] the latest position + 1 (u16, 0 = none);
//   search : every thread takes positions tid, tid + 1024, ...: walk at most kHcDepth (the level's depth) candidates
//            nearest first, keep the longest common prefix up to min(kHcNice, matchlimit - p), the nearer one on a tie,
//            stop at the cap.  Lengths
//            (u8) and offsets (u16) go to the CTA's scratch in global memory (L2-resident); the lengths are then copied
//            back into shared memory over the chains, which the parse no longer needs;
//   parse  : warp 0 scans 32 positions per step: a position starts a match when its length is >= 4 and the next
//            position's is not longer (lazy).  Lengths at the cap are extended with the same candidate.  Sequences are
//            emitted 32 at a time (flush_seqs) into the scratch; the block is stored raw when that is not smaller;
//   place  : the OFF chain gives the block's frame offset (place_block), and all warps copy it there.
// Claim, load, placement and write-out are frame.cuh's, shared with sky_fused_kernel.
//
// Optimal parse (SKY_F_OPTIMAL, sky_hc_kernel's kOpt): between search and emission every warp
// parses its own 2 KiB segment of the block by the bytes the sequences cost (opt_segment, the twin's
// hc_compress_block_opt), and warp 0 then emits the matches the segments chose instead of the lazy parse's.
//
// Linked blocks (SKY_F_LINKED, sky_hc_kernel's kLinked): block j >= 1 of a chunk also sees the chunk's 64 KiB before it
// (the twin's hc_compress_block_linked).  Shared memory has no room for that window, so it stays where it is:
//   window bytes : read from the chunk in global memory (d.src - 65536, L2-resident) by load32x / load8x, which read shared
//                  memory for a position in the block and global memory for one before it;
//   window chains: u16 distances of the window's positions in the CTA's scratch (kHcHistOff, 128 KiB more per CTA);
//   head         : still u16.  A bitmap in shared memory (kHcBitOff, 2 KiB) marks the hashes whose head this block has
//                  written; an unmarked non-zero head is a window position, stored as its index in the previous block.
// Chains: all warps hash the window into the chain array (free until the block's own chains), then warp 0 inserts the
// window's positions 1 .. 65535 and then the block's, in order: exact sequential insertion.  (Window position 0 lies
// 65536 bytes before every block position, so leaving it out changes no walk.)  A link longer than 65535 bytes is stored
// as "none"; a walk stops at the first candidate more than 65535 bytes back, as the twin's does.
#pragma once
#include "frame.cuh"

namespace sky {

// Levels (SKY_F_HC_LEVEL): liblz4's hash-chain levels 3..9, defined by the search budget -- level L walks 2^(L-1) chain
// candidates per position.  Everything else (hash, chains, tie rule, stop length, lazy rule, emission) is the same at every
// level; the kernel is instantiated once per level, so each depth is a compile-time loop bound.
constexpr int kHcMinLevel = 3, kHcMaxLevel = 9, kHcDefaultLevel = 5;
__host__ __device__ constexpr uint32_t hc_depth(int level) { return 1u << (level - 1); }
constexpr uint32_t kHcHashBits = 14;         // head table: 1 << 14 entries
constexpr uint32_t kHcNice = 32;             // a position's search stops at this length; the parse extends such matches
constexpr int kHcWarps = 32;
constexpr int kHcThreads = kHcWarps * 32;
static_assert(kHcNice < 256 && kHcNice % 4 == 0, "lengths are kept as u8; the search compares 4 bytes at a time");

struct HcCtl {
    uint64_t in_full;   // the block's bulk copy has landed
    BlockDesc desc;
    uint64_t data;  // frame offset of the block's first data byte
    uint32_t csize, raw;
    PendingChecksum pend;  // kBlkChk: the CTA's last block until warp 1 hashes it
};
constexpr uint32_t kHcInOff = 0;                                  // the block (+ slack for unaligned 4-byte reads)
constexpr uint32_t kHcChainOff = kInBytes;                        // u16 per position; after the search: u8 length per position
constexpr uint32_t kHcHeadOff = kHcChainOff + 2 * kBlock;         // u16 per hash
constexpr uint32_t kHcCtlOff = kHcHeadOff + (2u << kHcHashBits);
constexpr uint32_t kHcSmemBytes = kHcCtlOff + (uint32_t)sizeof(HcCtl);
static_assert(kHcSmemBytes <= 232448, "one HC CTA per SM: at most 227 KiB of shared memory");
constexpr uint32_t kHcBitOff = (kHcSmemBytes + 15u) & ~15u;                // linked: 1 bit per hash, "head written in this block"
constexpr uint32_t kHcLinkedSmemBytes = kHcBitOff + (1u << kHcHashBits) / 8;
static_assert(kHcLinkedSmemBytes <= 232448, "one linked HC CTA per SM: at most 227 KiB of shared memory");
// per-CTA scratch in global memory: lengths (u8), offsets (u16) and the compressed block; linked, the window's chains (u16)
constexpr uint32_t kHcLenOff = 0, kHcOffOff = kBlock, kHcOutOff = 3 * kBlock;
constexpr uint32_t kHcScratchBytes = 4 * kBlock + 2048;
constexpr uint32_t kHcHistOff = kHcScratchBytes, kHcLinkedScratchBytes = kHcHistOff + 2 * kBlock;
constexpr uint32_t kHcWindow = 65535;  // the largest offset

// Linked: the source bytes at position x of the block (x < 0: the previous block's, x >= -65536), from shared memory
// (in_s) in the block and from the chunk in global memory (src = the block's start, 16-byte aligned) before it.
__device__ __forceinline__ uint32_t load32x(uint32_t in_s, const uint8_t *src, int32_t x) {
    if (x >= 0) return load32s(in_s, (uint32_t)x);
    const uint32_t *w = reinterpret_cast<const uint32_t *>(src + (x & ~3));
    return __funnelshift_r(__ldg(w), __ldg(w + 1), (uint32_t)(x & 3) * 8u);
}
__device__ __forceinline__ uint32_t load8x(uint32_t in_s, const uint8_t *src, int32_t x) {
    return x >= 0 ? lds8(in_s + (uint32_t)x) : (uint32_t)__ldg(src + x);
}

// ---- optimal parse (SKY_F_OPTIMAL): the twin's hc_compress_block_opt, whose header states the rule.  Each warp parses its
// own kHcOptSeg-byte segments (one per warp in a 64 KiB block) in the shared memory the search leaves free:
//   len_s (chains, first half): the search's u8 length per position; a window's lengths are cleared once its forward pass
//          is done, and the backtrace writes there the length of every match the parse starts (255 + u16 length in the
//          next two bytes for a long match), which is what warp 0 emits from;
//   dec_s (chains, second half, and the head table's first byte at p = 65536): per position, the length of the match
//          that ends there in its kept state, 0 = reached by a literal.  A window [a, e] writes it at a < p <= e only, so
//          a warp writes and reads dec_s in (s0, s1] alone: the next warp's segment starts at s1 but never writes there.
// Forward pass: lane j holds the state of position p + j, packed as cost << 17 | run << 5 | last, so that the twin's
// lexicographic (cost, run, last) order is the u32 order.  Lane 0's state is final; lane 1 takes the literal from p, lanes
// 4 .. min(len(p), e - p) the match of their own length; then the states move down one lane.
constexpr uint32_t kHcOptSeg = 2048;
static_assert(kHcOptSeg * kHcWarps == kBlock, "one parse segment per warp of a whole block");
static_assert(kHcOptSeg < 4096 && kHcNice <= 32, "a state packs its run in 12 bits and its last match in 5");
constexpr uint32_t kOptCost = 17, kOptLong = 255;
template <bool kLinked>
__device__ __forceinline__ void opt_segment(uint32_t in_s, const uint8_t *src, uint32_t len_s, uint32_t dec_s, const uint16_t *g_off,
                                            uint32_t s0, uint32_t s1, uint32_t mflimit, uint32_t matchlimit, unsigned lane) {
    const uint32_t need = lane == 1u ? 0u : lane >= kMinMatch ? lane : 0xffu;  // lane 1: the literal; 4..31: match length
    const uint32_t mstep = ((3u + (lane >= kMinMatch + 15u ? 1u : 0u)) << kOptCost) | lane;
    for (uint32_t a = s0; a < s1;) {
        uint32_t e = s1;  // the first long position at or after a
        for (uint32_t b = a; b < s1; b += 32) {
            const uint32_t x = b + lane;
            const unsigned m = __ballot_sync(kFull, x < s1 && x <= mflimit && s1 - x >= kHcNice && lds8(len_s + x) == kHcNice);
            if (m) {
                e = b + (uint32_t)__ffs(m) - 1u;
                break;
            }
        }
        uint32_t st = lane == 0 ? 0u : 0xffffffffu;
        for (uint32_t p = a; p < e; p++) {
            const uint32_t k0 = __shfl_sync(kFull, st, 0);
            if (lane == 0 && p != a) sts8(dec_s + p, k0 & 31u);  // (the backtrace stops at a)
            const uint32_t len = p <= mflimit ? lds8(len_s + p) : 0u;
            const uint32_t run = ((k0 >> 5) & 0xfffu) + 1u;
            const uint32_t bump = (run + 240u) * 0xFEFEFEFFu <= 0x01010101u ? 2u : 1u;  // a length byte more at 15, 270, ...
            const uint32_t cand = lane == 1u ? (((k0 >> kOptCost) + bump) << kOptCost) | (run << 5) : (k0 & ~((1u << kOptCost) - 1u)) + mstep;
            if (need <= min(len, e - p)) st = min(st, cand);
            st = __shfl_down_sync(kFull, st, 1);
            if (lane == 31) st = 0xffffffffu;
        }
        if (lane == 0 && e != a) sts8(dec_s + e, st & 31u);
        for (uint32_t x = a + lane; x < e; x += 32) sts8(len_s + x, 0u);
        __syncwarp();
        for (uint32_t q = e; q > a;) {  // backtrace: the nearest position at or before q reached by a match, 32 at a time
            const uint32_t v = lane < q - a ? lds8(dec_s + q - lane) : 0u;
            const unsigned m = __ballot_sync(kFull, v != 0u);
            if (!m) {
                q = q - a > 32u ? q - 32u : a;
                continue;
            }
            const uint32_t f = (uint32_t)__ffs(m) - 1u, ml = __shfl_sync(kFull, v, f);
            q -= f + ml;
            if (lane == 0) sts8(len_s + q, ml);
        }
        if (e == s1) break;
        const uint32_t cand = e - __ldcg(g_off + e), lim = min(matchlimit, s1) - e;
        uint32_t ml;
        if constexpr (kLinked) ml = extend_coop([in_s, src](uint32_t x) { return load32x(in_s, src, (int32_t)x); }, e, cand, kHcNice, lim, lane);
        else ml = extend_coop_s(in_s, e, cand, kHcNice, lim, lane);
        if (lane == 0) {
            sts8(len_s + e, kOptLong);
            sts8(len_s + e + 1u, ml & 0xffu);
            sts8(len_s + e + 2u, ml >> 8);
        }
        __syncwarp();
        a = e + ml;
    }
}

// kHcDepth: chain candidates walked per position, hc_depth(level).  kBlkChk (SKY_F_BLOCK_CHECKSUM): every block gets its
// checksum (block_checksum), hashed from the frame by warp 1 during the next block's chain step, which only warp 0 works
// on (or before the CTA exits).  kLinked (SKY_F_LINKED): blocks after a chunk's first match into its previous 64 KiB.
// kOpt (SKY_F_OPTIMAL): every warp parses its segment optimally (opt_segment) before warp 0 emits the chosen matches.
template <uint32_t kHcDepth, bool kBlkChk, bool kLinked, bool kOpt>
__device__ __forceinline__ void hc_body(const Params &p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const unsigned tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    uint8_t *in = smem + kHcInOff;
    HcCtl *ctl = reinterpret_cast<HcCtl *>(smem + kHcCtlOff);
    const uint32_t in_s = smem_u32(in), chain_s = smem_u32(smem + kHcChainOff), head_s = smem_u32(smem + kHcHeadOff);
    uint8_t *scr = p.scratch + (size_t)blockIdx.x * (kLinked ? kHcLinkedScratchBytes : kHcScratchBytes);
    uint8_t *g_len = scr + kHcLenOff;
    uint16_t *g_off = reinterpret_cast<uint16_t *>(scr + kHcOffOff);
    uint8_t *cout = scr + kHcOutOff;
    uint16_t *g_hist = reinterpret_cast<uint16_t *>(scr + kHcHistOff);  // linked: chain distance of window position i
    const uint32_t bit_s = smem_u32(smem + kHcBitOff);
    if (tid == 0) {
        mbar_init(&ctl->in_full, 1);
        if constexpr (kBlkChk) ctl->pend.data = nullptr;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    for (uint32_t in_phase = 0;; in_phase ^= 1) {
        if (tid == 0) claim_block<kLinked>(p, &ctl->desc);
        __syncthreads();  // (also: every warp is done with the previous block)
        const BlockDesc d = ctl->desc;
        if (!d.valid) {
            if constexpr (kBlkChk) {
                if (warp == 1) run_pending(&ctl->pend, lane);
            }
            break;
        }
        const uint32_t L = d.L;
        if (tid == 0) load_block(in, d.src, L, &ctl->in_full);
        uint4 *h4 = reinterpret_cast<uint4 *>(smem + kHcHeadOff);
        for (uint32_t k = tid; k < (2u << kHcHashBits) / 16; k += kHcThreads) h4[k] = make_uint4(0, 0, 0, 0);
        const bool window = kLinked && d.j > 0 && L >= kMfLimit + 1;  // linked: this block sees the previous one
        if constexpr (kLinked) {
            uint4 *b4 = reinterpret_cast<uint4 *>(smem + kHcBitOff);
            for (uint32_t k = tid; k < (1u << kHcHashBits) / 128; k += kHcThreads) b4[k] = make_uint4(0, 0, 0, 0);
            if (window) {  // the window's hashes, into the chain array: position i of the previous block at i * 2
                const uint8_t *prev = d.src - kBlock;
                for (uint32_t i = tid; i < kBlock; i += kHcThreads) {
                    const uint32_t *w = reinterpret_cast<const uint32_t *>(prev + (i & ~3u));
                    const uint32_t v = __funnelshift_r(__ldg(w), __ldg(w + 1), (i & 3u) * 8u);
                    sts16(chain_s + i * 2u, (v * 2654435761u) >> (32 - kHcHashBits));
                }
            }
        }
        mbar_wait(&ctl->in_full, in_phase);
        __syncthreads();  // the head table is clear

        const uint32_t mflimit = L - kMfLimit, matchlimit = L - kLastLiterals;  // (meaningful when L > kMfLimit)
        const bool has_matches = L >= kMfLimit + 1;
        // ---------------------------------------------------------------- chains (warp 0)
        if (window && warp == 0) {  // the window's positions 1 .. 65535 first; head = the position's index, 1 .. 65535
            for (uint32_t base = 0; base < kBlock; base += 32) {
                const uint32_t i = base + lane;
                const bool valid = i != 0;
                const uint32_t h = valid ? lds16(chain_s + i * 2u) : 0x80000000u;
                const unsigned same = __match_any_sync(kFull, h);
                const unsigned lower = same & ((1u << lane) - 1u);
                const uint32_t prev = lower ? base + bfind(lower) : (valid ? lds16(head_s + h * 2u) : 0u);
                __syncwarp();
                if (valid) {
                    if ((same >> lane) == 1u) sts16(head_s + h * 2u, i);
                    g_hist[i] = (uint16_t)(prev ? i - prev : 0u);
                }
                __syncwarp();
            }
        }
        if (has_matches && warp == 0) {
            for (uint32_t base = 0; base <= mflimit; base += 32) {
                const uint32_t q = base + lane;
                const bool valid = q <= mflimit;
                const uint32_t h = valid ? (load32s(in_s, q) * 2654435761u) >> (32 - kHcHashBits) : 0x80000000u | lane;
                const unsigned same = __match_any_sync(kFull, h);
                const unsigned lower = same & ((1u << lane) - 1u);
                uint32_t dist;
                if constexpr (kLinked) {  // a head this block has not written is a window position's index (or 0)
                    const uint32_t hv = valid ? lds16(head_s + h * 2u) : 0u;
                    const bool mine = valid && ((lds32(bit_s + (h >> 5) * 4u) >> (h & 31u)) & 1u);
                    dist = lower ? lane - bfind(lower) : !hv ? 0u : mine ? q + 1u - hv : q + kBlock - hv;
                    if (dist > kHcWindow) dist = 0u;
                } else {
                    const uint32_t prev = lower ? base + bfind(lower) + 1u : (valid ? lds16(head_s + h * 2u) : 0u);  // position + 1
                    dist = prev ? q + 1u - prev : 0u;
                }
                __syncwarp();  // every read of head before any update
                if (valid) {
                    if ((same >> lane) == 1u) {  // the highest lane of this hash
                        sts16(head_s + h * 2u, q + 1u);
                        if constexpr (kLinked) atomicOr(reinterpret_cast<uint32_t *>(smem + kHcBitOff) + (h >> 5), 1u << (h & 31u));
                    }
                    sts16(chain_s + q * 2u, dist);
                }
                __syncwarp();
            }
        }
        if constexpr (kBlkChk) {
            if (warp == 1) run_pending(&ctl->pend, lane);  // the previous block's checksum, beside warp 0's chains
        }
        __syncthreads();
        // ---------------------------------------------------------------- best match per position (all warps)
        if (has_matches) {
            for (uint32_t q = tid; q <= mflimit; q += kHcThreads) {
                const uint32_t cap = min(kHcNice, matchlimit - q);
                uint32_t best = 0, boff = 0, c = q, dist = lds16(chain_s + q * 2u);
                for (uint32_t k = 0; k < kHcDepth && dist; k++) {
                    c -= dist;
                    if constexpr (kLinked) {
                        if (q - c > kHcWindow) break;  // (c < 0: a window position)
                    }
                    // a longer match than `best` must agree at byte `best` (best < cap here): others are skipped unmeasured
                    const uint32_t cb = kLinked ? load8x(in_s, d.src, (int32_t)(c + best)) : lds8(in_s + c + best);
                    if (cb == lds8(in_s + q + best)) {
                        uint32_t len = 0;
                        for (;;) {
                            const uint32_t x = load32s(in_s, q + len) ^
                                               (kLinked ? load32x(in_s, d.src, (int32_t)(c + len)) : load32s(in_s, c + len));
                            if (x) {
                                len += (uint32_t)(__ffs(x) - 1) >> 3;
                                break;
                            }
                            len += 4;
                            if (len >= cap) break;
                        }
                        len = min(len, cap);
                        if (len > best) {
                            best = len;
                            boff = q - c;
                            if (best == cap) break;
                        }
                    }
                    if constexpr (kLinked) dist = (int32_t)c >= 0 ? lds16(chain_s + c * 2u) : (uint32_t)__ldcg(g_hist + (c + kBlock));
                    else dist = lds16(chain_s + c * 2u);
                }
                g_len[q] = (uint8_t)(best >= kMinMatch ? best : 0u);
                g_off[q] = (uint16_t)boff;
            }
        }
        __syncthreads();
        if (has_matches) {  // lengths back into shared memory, over the chains
            const uint4 *src4 = reinterpret_cast<const uint4 *>(g_len);
            uint4 *dst4 = reinterpret_cast<uint4 *>(smem + kHcChainOff);
            for (uint32_t k = tid; k < (mflimit + 16u) / 16u; k += kHcThreads) dst4[k] = __ldcg(src4 + k);
        }
        __syncthreads();
        if constexpr (kOpt) {  // ------------------------------------------- optimal parse, one segment per warp
            if (has_matches)
                for (uint32_t s0 = warp * kHcOptSeg; s0 < L; s0 += kHcWarps * kHcOptSeg)
                    opt_segment<kLinked>(in_s, d.src, chain_s, chain_s + kBlock, g_off, s0, min(s0 + kHcOptSeg, L), mflimit, matchlimit, lane);
            __syncthreads();
        }
        // ---------------------------------------------------------------- lazy parse + emission (warp 0), then placement
        if (warp == 0) {
            uint32_t op = 0, anchor = 0;
            if (has_matches) {
                uint32_t cur = 0, nseq = 0, q0 = 0, q1 = 0;
                for (;;) {
                    if (cur <= mflimit) {
                        const uint32_t x = cur + lane;
                        const uint32_t len = x <= mflimit ? lds8(chain_s + x) : 0u;
                        unsigned take;
                        if constexpr (kOpt) {  // the matches the optimal parse chose
                            take = __ballot_sync(kFull, len != 0u);
                        } else {
                            uint32_t nxt = __shfl_down_sync(kFull, len, 1);
                            if (lane == 31) nxt = x + 1u <= mflimit ? lds8(chain_s + x + 1u) : 0u;
                            take = __ballot_sync(kFull, len >= kMinMatch && nxt <= len);
                        }
                        if (!take) {
                            cur += 32;
                            continue;
                        }
                        const uint32_t f = (uint32_t)__ffs(take) - 1u, pos = cur + f;
                        uint32_t ml = __shfl_sync(kFull, len, f);
                        if constexpr (kOpt) {
                            if (ml == kOptLong) ml = lds8(chain_s + pos + 1u) | (lds8(chain_s + pos + 2u) << 8);
                        } else if (ml == kHcNice) {
                            const uint32_t cand = pos - __ldcg(g_off + pos);
                            if constexpr (kLinked) {
                                const uint8_t *src = d.src;
                                ml = extend_coop([in_s, src](uint32_t x) { return load32x(in_s, src, (int32_t)x); }, pos, cand, ml, matchlimit - pos, lane);
                            } else {
                                ml = extend_coop_s(in_s, pos, cand, ml, matchlimit - pos, lane);
                            }
                        }
                        if (lane == nseq) {
                            q0 = (pos - anchor) | (ml << 16);
                            q1 = anchor | (pos << 16);  // (the offset is fetched for 32 sequences at once when they are emitted)
                        }
                        anchor = cur = pos + ml;
                        if (++nseq < 32) continue;
                    }
                    if (nseq) {  // 32 sequences, or the last ones of the block
                        if (lane < nseq) q1 = (q1 & 0xffffu) | ((uint32_t)__ldcg(g_off + (q1 >> 16)) << 16);
                        op = flush_seqs(cout, op, in, q0, q1, nseq, false, lane);
                        nseq = 0;
                    }
                    if (cur > mflimit) break;
                }
            }
            op = emit_seq(cout, op, in, anchor, L - anchor, 0, 0, lane);  // the final literals
            if (lane == 0) {
                const BlockPlace pl = place_block<kBlkChk>(p, d, op, L);
                ctl->data = pl.data;
                ctl->csize = op;
                ctl->raw = pl.raw;
            }
        }
        __syncthreads();
        // the block to its final place, straight from the input when stored raw
        uint8_t *out = d.dst + ctl->data;
        if (ctl->raw) copy_block<kHcWarps, true>(out, d.src, L, warp, lane);
        else copy_block<kHcWarps, false>(out, cout, ctl->csize, warp, lane);
        if constexpr (kBlkChk) {
            if (warp == 1) set_pending(&ctl->pend, out, ctl->raw ? L : ctl->csize, lane);
        }
    }
}

// Linked kernels take kHcLinkedSmemBytes of shared memory and kHcLinkedScratchBytes of scratch per CTA, the others
// kHcSmemBytes and kHcScratchBytes; the optimal parse needs no more than the lazy one.
template <uint32_t kHcDepth, bool kBlkChk, bool kLinked, bool kOpt>
__global__ void __launch_bounds__(kHcThreads, 1) sky_hc_kernel(const Params p) { hc_body<kHcDepth, kBlkChk, kLinked, kOpt>(p); }

}  // namespace sky

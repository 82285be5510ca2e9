// skychunk.cu -- fused LZ4-frame + MD5 chunk stage for H100 (sm_90a) and its C ABI (include/skychunk.h).
//
// One persistent kernel per batch (sky_fused_kernel), two CTAs per SM, 14 warps per CTA, one role per CTA at a time:
//   * digest CTAs : the first few CTAs carry the MD5 groups -- 32 chunks per warp, lane = chunk (md5.cuh), one MD5 warp
//                   per CTA while the groups are few.  An MD5 chain is latency bound (3 dependent ALU ops per step, one
//                   64-byte block per ~1044 cycles) and keeps its scheduler's issue port busy; when a CTA's groups are done
//                   it joins the compressors.
//   * compressor CTAs : one 64 KiB block at a time, claimed from a global atomic counter in row-major order (block row j of
//                   every chunk, then row j+1 ...): bulk-load the block into shared memory, warps 0-1 probe, warps 2-13
//                   parse segment by segment into an L2-resident scratch (lz4.cuh), warp 0 plans the block's layout.
// Output placement (single pass, no compaction kernel): a block's final place in the frame is only known when every block
// before it has been sized, so one per-chunk word, the OFF chain (frame.cuh), orders the blocks.  Block j sizes itself
// from its segments' records, takes its frame offset from the chain and passes it on (place_block), then writes its bytes
// to the final place exactly once (stored blocks straight from the input).  The last block's CTA writes the EndMark and
// the frame length.  The high-ratio compressor (lz4hc.cuh, SKY_F_HC) claims, loads and places its blocks through the
// same frame.cuh helpers.
//
// Digest lanes and compressors each read their own input from HBM, and a digest lane never waits for a compressor.  A
// compressor CTA that shares an SM with a running chain steps aside while the LZ4 work is projected to finish well before
// the chain (wait_for_chain), so the chain keeps its SM's issue slots.
//
// Host side: sky_ctx owns every stream, event and buffer through move-only owners that release them in their destructors:
// per slot a kernel stream, batch metadata, the receiver's and the E2EE arrays and (optionally) input / output slabs for
// the host-buffer path (H2D and D2H on two streams shared by the slots, the kernels on the slot's stream).
// There is NO CPU fallback anywhere in this file: without a CUDA device every entry point fails.

#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <algorithm>
#include <array>
#include <memory>
#include <new>
#include <numeric>
#include <string>
#include <utility>
#include <vector>

#include "../../include/skychunk.h"
#include "frame.cuh"
#include "lz4.cuh"
#include "lz4dec.cuh"
#include "lz4hc.cuh"
#include "lz4verify.cuh"
#include "md5.cuh"
#include "secretbox.cuh"

namespace sky {

#ifndef SKY_PARSERS
#define SKY_PARSERS 12
#endif
constexpr int kParsers = SKY_PARSERS;     // parser warps per CTA
constexpr int kProbers = 2;               // prober warps (0 and 1): they take alternate 256-slot batches
constexpr int kWarps = kProbers + kParsers;
constexpr int kThreads = kWarps * 32;
#ifndef SKY_RING_EXTRA
#define SKY_RING_EXTRA 2
#endif
constexpr int kRing = kParsers + SKY_RING_EXTRA;       // segment slots between the prober and the parsers
constexpr int kMd5WarpsPerCta = 4;        // digest CTAs run 4 MD5 groups (one per SM sub-partition), see sky_fused_kernel
constexpr uint32_t kRingBytes = SKY_MD5_SLOTS * 2048;  // sender's MD5 staging ring: slots x 64 B x 32 lanes
constexpr int kDecMd5Slots = 4;           // the receiver's MD5 ring (its copies are of bytes the decode warps just wrote, in L2)
constexpr uint32_t kDecRingBytes = kDecMd5Slots * 2048;
constexpr int kCtasPerSm = 2;             // fused kernel: 2 x ~110 KiB of shared memory per SM
constexpr uint64_t kMaxChunkBlocks = 1ull << 21;  // 64 KiB blocks = 128 GiB per chunk: md5_warp counts 64-byte blocks in 32 bits

// ---- shared-memory layout of the fused kernel (dynamic, 128-byte aligned base) -------------------------
struct Ctl {
    uint64_t in_full;               // bulk copy of the block has landed
    uint64_t full[kRing], empty[kRing];
    BlockDesc desc[2];              // by block-iteration parity
    uint32_t claim;                 // next segment sequence number a parser may take (runs across blocks)
    volatile uint32_t block_end_seq;  // sequence number after the current block's last segment (0xffffffff while probing)
    volatile uint32_t nseg;
    volatile uint32_t seg_hit[4];     // per segment (mod 4): OR of its batches' hit masks (decides the stride two segments on)
    uint32_t raw, last_lits, tail_off;  // plan results: stored?, final literal run and where it goes
    uint64_t data;                      // frame offset of the block's first data byte
    uint32_t size;                      // the block's data bytes in the frame (kBlkChk only)
    PendingChecksum pend;               // kBlkChk: the CTA's last compressed block until kSumWarp hashes it
    uint64_t t0;                        // %clock64 when the CTA started (wait_for_chain)
};
constexpr uint32_t kInOff = 0;
constexpr uint32_t kTabOff = kInOff + kInBytes;
constexpr uint32_t kRingOff = kTabOff + kTableBytes;
constexpr uint32_t kRecOff = kRingOff + kRing * (uint32_t)sizeof(SegSlot);
constexpr uint32_t kPlanOff = kRecOff + kMaxSegs * (uint32_t)sizeof(SegRec);
constexpr uint32_t kCtlOff = kPlanOff + kMaxSegs * (uint32_t)sizeof(SegPlan);
constexpr uint32_t kSmemBytes = (kCtlOff + (uint32_t)sizeof(Ctl) + 127u) & ~127u;
static_assert(kSmemBytes <= 232448 / 2 - 1024, "two CTAs per SM need <= 112.5 KiB each: lower SKY_PARSERS or SKY_LZ4_ENTRIES");
static_assert(kEntries % 128 == 0, "SKY_LZ4_ENTRIES must be a multiple of 128");
static_assert(kMd5WarpsPerCta * kRingBytes <= kInBytes, "the MD5 rings live in the block buffer of a digest CTA");
static_assert(sizeof(SegSlot) % 16 == 0 && sizeof(SegRec) == 16 && sizeof(SegPlan) == 16, "layout");

#ifdef SKY_MD5_TRACE
// Diagnostic build only (see md5.cuh): thread 0 of every fused-kernel CTA that compresses records its SM, when it
// started, when it claimed its first and last block and when it found the claim counter exhausted.
constexpr int kTraceCtas = 1024;
struct CtaTrace {
    uint32_t smid, digest, claims, pad;
    uint64_t entry, first, last, exhausted;
};
__device__ CtaTrace g_cta_trace[kTraceCtas];
#endif

// ---- compressors step aside for the MD5 chains of their SM ----------------------------------------------------------
// A digest CTA in a launch that also compresses publishes, in its SM's word behind the claim counter, the %clock64 by which
// its warp 0's chains would end at the chain's floor rate.  Before each block claim, thread 0 of a compressing CTA on that
// SM reads the word: while the chains run and the claims so far project the LZ4 work to end well before them, the CTA
// waits instead of claiming, since its probers and parsers would take issue slots from the chain (§4.1: an MD5 chain ran
// 3.5 % slower per block while the compressor beside it claimed blocks).  Where compressing is the longer stage (config 3)
// the projection says so and nothing waits.  The wait ends on the clock, so it needs nothing to clear it, and a CTA waits
// only between blocks, holding no OFF-chain word: every block before the ones it would claim was claimed by a CTA that is
// running, so the OFF chain stays deadlock-free (frame.cuh).
#ifndef SKY_CHAIN_WAIT
#define SKY_CHAIN_WAIT 1
#endif
constexpr bool kChainWait = SKY_CHAIN_WAIT != 0;        // 0: compressors never wait (tools/build_variants.py no_chain_wait)
constexpr uint32_t kSmWords = 256;                      // per-SM words (%smid < kSmWords) after the counters' first 64 bytes
constexpr uint32_t kCountersBytes = 64 + kSmWords * 8;  // cleared before every launch
constexpr uint64_t kChainCyclesPerBlock = 780;          // 12.16 cycles x 64 steps: the static schedule (under load it runs slower)
__device__ __forceinline__ uint64_t *sm_chain_end(const Params &p) { return reinterpret_cast<uint64_t *>(p.counters + 16); }
__device__ __forceinline__ uint32_t sm_id() {
    uint32_t s;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(s));
    return s;
}
// One thread of a digest CTA, as its chains start.  md5_order lists each group's longest chunk first.
__device__ __forceinline__ void publish_chain_end(const Params &p) {
    uint64_t blocks = 0;
    for (uint32_t g = blockIdx.x; g < p.n_groups; g += p.n_md5_ctas * kMd5WarpsPerCta) blocks += p.chunks[p.md5_order[g * 32]].len >> 6;
    const uint32_t s = sm_id();
    if (s < kSmWords)
        atomicMax(reinterpret_cast<unsigned long long *>(sm_chain_end(p) + s), (unsigned long long)(clock64() + blocks * kChainCyclesPerBlock));
}
// Thread 0 of a compressing CTA, before it claims a block; t0 = its %clock64 at start.
__device__ __forceinline__ void wait_for_chain(const Params &p, uint64_t t0) {
    const uint32_t s = sm_id();
    if (s >= kSmWords) return;
    uint64_t end;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(end) : "l"(sm_chain_end(p) + s) : "memory");
    const uint32_t total = p.rows * p.n_chunks;
    for (;;) {
        const uint64_t now = clock64();
        const uint32_t w = ld_relaxed32(p.counters);
        // the chain is done, too few claims to project from (1/64 of the blocks), or none left
        if (now >= end || w <= total / 64 || w >= total) return;
        const float left = (float)(now - t0) * ((float)(total - w) / (float)w);  // the rest at the claims' rate so far
        if (1.25f * left >= (float)(end - now)) return;  // not clearly ahead of the chain: keep compressing
        __nanosleep(10000);
    }
}

// named-barrier token between the two prober warps: the releaser arrives, the waiter syncs (ids 1 and 2, 64 threads)
template <int kId>
__device__ __forceinline__ void bar_arrive() { asm volatile("bar.arrive %0, 64;" ::"n"(kId) : "memory"); }
template <int kId>
__device__ __forceinline__ void bar_wait() { asm volatile("bar.sync %0, 64;" ::"n"(kId) : "memory"); }

// Fused LZ4-frame + MD5 kernel body.  Grid = 2 CTAs per SM, kWarps warps each.
//   digest CTAs (blockIdx < n_md5_ctas): warps 0..3 each carry one MD5 group (32 chunks, lane = chunk, md5.cuh) at a time;
//       when the groups are done the CTA joins the compressors.  kXxh: the MD5 lanes also write XXH32(chunk) to xxh_out.
//   compressor CTAs: one 64 KiB block at a time -- bulk-load it into shared memory, warp 0 probes, warps 1.. parse
//       (lz4.cuh), warp 0 plans the block's layout and takes its frame offset from the OFF chain, all warps write it out.
//       kBlkChk (SKY_F_BLOCK_CHECKSUM): the last parser warp also hashes every block the CTA writes (block_checksum).  A
//       block is only whole in the frame once every warp has written its part, so its hash is deferred to the CTA's next
//       block: the warp reads it back from the frame between two of its segment claims, and the other parsers take up
//       its share of the segments meanwhile.  (Hashing a stored block from the block buffer during its own write-out
//       instead made ptxas spill in the main loop.)
template <bool kXxh, bool kBlkChk>
__device__ __forceinline__ void fused_body(const Params &p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t *in = smem + kInOff;
    uint32_t *tab = reinterpret_cast<uint32_t *>(smem + kTabOff);
    SegSlot *ring = reinterpret_cast<SegSlot *>(smem + kRingOff);
    SegRec *recs = reinterpret_cast<SegRec *>(smem + kRecOff);
    SegPlan *plans = reinterpret_cast<SegPlan *>(smem + kPlanOff);
    Ctl *ctl = reinterpret_cast<Ctl *>(smem + kCtlOff);
    uint32_t smem_s = smem_u32(smem);  // shared-window address of the CTA's buffer, kept in a register: left to itself the
    asm volatile("" : "+r"(smem_s));   // compiler re-derives it (S2UR SR_CgaCtaId + ULEA) at the top of every prober batch

    const bool do_md5 = (p.flags & SKY_F_MD5) != 0, do_lz4 = (p.flags & SKY_F_LZ4) != 0;
#ifdef SKY_MD5_TRACE
    CtaTrace tr{};
    if (warp == 0 && lane == 0) {
        tr.smid = trace_smid();
        tr.digest = do_md5 && blockIdx.x < p.n_md5_ctas;
        tr.entry = trace_globaltimer();
    }
#endif
    if (warp == 0 && lane == 0) {
        mbar_init(&ctl->in_full, 1);
        for (int i = 0; i < kRing; i++) {
            mbar_init(&ctl->full[i], 1);
            mbar_init(&ctl->empty[i], 1);
        }
        ctl->claim = 0;
        ctl->t0 = clock64();
        if constexpr (kBlkChk) ctl->pend.data = nullptr;
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    if (do_md5 && blockIdx.x < p.n_md5_ctas) {
        if (kChainWait && do_lz4 && warp == kWarps - 1 && lane == 0) publish_chain_end(p);  // (an idle warp: warps 0-3 carry the chains)
        if (warp < kMd5WarpsPerCta) {
            for (uint32_t g = warp * p.n_md5_ctas + blockIdx.x; g < p.n_groups; g += p.n_md5_ctas * kMd5WarpsPerCta) {
                const uint32_t c = p.md5_order[g * 32 + lane];
                const bool active = c != 0xffffffffu;
                const uint8_t *src = nullptr;
                uint64_t len = 0;
                if (active) {
                    src = p.chunks[c].src;
                    len = p.chunks[c].len;
                }
                const uint32_t x = md5_warp<kXxh>(reinterpret_cast<uint32_t *>(in + warp * kRingBytes), src, len, active,
                                                  p.md5_out + (size_t)(active ? c : 0) * 16, lane
#ifdef SKY_MD5_TRACE
                                                  , Md5NoGate(), g < kTraceGroups ? &g_md5_trace[g] : nullptr
#endif
                );
                if constexpr (kXxh) {
                    if (active) p.xxh_out[c] = x;
                }
                __syncwarp();
            }
        }
        if (!do_lz4) return;
        __syncthreads();  // the rings overlapped the block buffer
    }
    if (!do_lz4) return;

    uint8_t *scratch = p.scratch + (size_t)blockIdx.x * kScratchBytes;
    uint32_t gseq = 0;        // probers: sequence number of the next segment they publish (runs across blocks)
    uint32_t batches_done = 0;  // prober 0: nothing to wait for before the kernel's very first batch
    uint32_t my_seq = 0;      // parser: the sequence number it holds a claim on
    bool have_claim = false;
    uint32_t in_phase = 0;
    constexpr unsigned kSumWarp = kWarps - 1;  // kBlkChk: the warp that hashes the blocks
    for (uint32_t it = 0;; it++) {
        BlockDesc *dsc = &ctl->desc[it & 1];
        if (warp == 0 && lane == 0) {
            if (kChainWait && p.n_md5_ctas) wait_for_chain(p, ctl->t0);  // (the CTA's other threads wait at the barrier below)
            claim_block(p, dsc);
            ctl->block_end_seq = 0xffffffffu;
            ctl->nseg = 0;
#ifdef SKY_MD5_TRACE
            const uint64_t t = trace_globaltimer();
            if (dsc->valid) {
                if (tr.claims++ == 0) tr.first = t;
                tr.last = t;
            } else {
                tr.exhausted = t;
                if (blockIdx.x < kTraceCtas) g_cta_trace[blockIdx.x] = tr;
            }
#endif
        }
        __syncthreads();  // (also: every warp is done with the previous block's buffer, records and plan)
        if (!dsc->valid) {
            if constexpr (kBlkChk) {
                if (warp == kSumWarp) run_pending(&ctl->pend, lane);
            }
            break;
        }
        const uint8_t *src = dsc->src;
        const uint32_t L = dsc->L;

        if (warp < kProbers) {
            // ---------------------------------------------------------------- probers (warps 0 and 1, alternate batches of every segment)
            if (warp == 0) {
                if (lane == 0) load_block(in, src, L, &ctl->in_full);
                // clear the table meanwhile: entry 0 = (position 0, tag 0) doubles as "empty".  (Warp 1's first table access
                // follows warp 0's first table phase through the token, so it sees the cleared table.)
                uint4 *t4 = reinterpret_cast<uint4 *>(tab);
                const uint4 z = make_uint4(0, 0, 0, 0);
#pragma unroll 4
                for (uint32_t k = lane; k < kEntries / 4; k += 32) t4[k] = z;
                __syncwarp();
            }
            mbar_wait(&ctl->in_full, in_phase);
            in_phase ^= 1;
            uint32_t nseg = 0;
            if (L >= kMfLimit + 1) {
                const uint32_t mflimit = L - kMfLimit;
                uint32_t seg_pos = 0, slog = 0;
                while (seg_pos <= mflimit) {
                    if (nseg >= 2) {  // the verdict on segment nseg-2 decides this segment's stride
                        const bool h = ctl->seg_hit[(nseg - 2) & 3u] != 0u;
                        slog = h ? 0u : min(slog + 1u, kMaxStepLog);
                    }
                    const uint32_t si = gseq % kRing, ph = (gseq / kRing) & 1u;
                    SegSlot *slot = ring + si;
#pragma unroll 1
                    for (uint32_t b = warp; b < 4; b += kProbers) {
                        const uint32_t slot_s = smem_s + kRingOff + si * (uint32_t)sizeof(SegSlot);
                        const uint32_t hits = probe_batch(smem_s + kInOff, smem_s + kTabOff, slot_s + (uint32_t)offsetof(SegSlot, offs),
                                                          slot_s + (uint32_t)offsetof(SegSlot, masks), seg_pos, slog, b, mflimit, lane, [&]() {
                            // my turn at the table: the other prober has finished the previous batch
                            if (warp == 0) {
                                if (batches_done) bar_wait<2>();
                                if (b == 0) mbar_wait(&ctl->empty[si], ph ^ 1u);  // the ring slot is free again
                            } else {
                                bar_wait<1>();
                            }
                        });
                        batches_done = 1;
                        if (lane == 0) {
                            ctl->seg_hit[nseg & 3u] = (b == 0 ? 0u : ctl->seg_hit[nseg & 3u]) | hits;
                            if (b == 0) {
                                slot->seg_pos = seg_pos;
                                slot->slog = slog;
                                slot->sidx = nseg;
                            }
                        }
                        __syncwarp();
                        if (b == 3 && lane == 0) mbar_arrive(&ctl->full[si]);  // (release: both probers' slot writes are ordered before it)
                        __threadfence_block();
                        if (warp == 0) bar_arrive<1>(); else bar_arrive<2>();  // pass the token
                    }
                    seg_pos += kSegSlots << slog;
                    gseq++;
                    nseg++;
                }
            }
            if (warp == kProbers - 1 && lane == 0) {
                ctl->nseg = nseg;
                __threadfence_block();
                atomicExch(const_cast<uint32_t *>(&ctl->block_end_seq), gseq);  // (atomic: the parsers poll this word)
            }
        } else {
            // ---------------------------------------------------------------- parsers
            mbar_wait(&ctl->in_full, in_phase);  // the block is in shared memory (the prober may still be clearing the table)
            in_phase ^= 1;
            for (;;) {
                if (!have_claim) {
                    uint32_t t = 0;
                    if (lane == 0) t = atomicAdd(&ctl->claim, 1u);
                    my_seq = __shfl_sync(kFull, t, 0);
                    have_claim = true;
                }
                const uint32_t si = my_seq % kRing, ph = (my_seq / kRing) & 1u;
                bool got = true;
                // (mbarrier.try_wait's hardware suspend ends at every barrier event in the CTA, a few dozen ns apart here, so the
                // waiting loops are a quarter of the instructions issued -- but replacing them with timed sleeps gained
                // nothing measurable: the issue slots they take are not the ones the parsers lack.)
                while (!mbar_try_wait_hint(&ctl->full[si], ph, 1000u)) {
                    if (atomicAdd(const_cast<uint32_t *>(&ctl->block_end_seq), 0u) <= my_seq) {  // no such segment in this block: keep the claim
                        got = mbar_try_wait(&ctl->full[si], ph);
                        break;
                    }
                }
                if (!got) break;
                const SegSlot *slot = ring + si;
                const uint32_t sidx = slot->sidx;
                uint8_t *scr = scratch + slot->seg_pos + sidx * kSegPad;
                const SegRec r = parse_segment(in, slot, scr, L, lane);
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(&ctl->empty[si]);
                    recs[sidx] = r;
                }
                have_claim = false;
                if constexpr (kBlkChk) {
                    if (warp == kSumWarp) run_pending(&ctl->pend, lane);  // (between two claims: no segment waits for this warp meanwhile)
                }
            }
        }
        __syncthreads();

        // ---------------------------------------------------------------- plan (warp 0)
        const uint32_t nseg = ctl->nseg;
        if (warp == 0) {
            // String the segments together: the literals a segment leaves behind its last match (or a whole segment without
            // a match) are carried into the next first sequence.  carry_out(s) = has_match(s) ? t(s) : carry_in(s) + t(s) is
            // a scan of (reset, add) pairs: every lane folds its kPlanPerLane consecutive segments, the lanes are scanned with
            // shuffles, then every lane replays its segments with the true carry and sizes them; a second scan places them.
            constexpr uint32_t kPlanPerLane = (kMaxSegs + 31) / 32;
            uint32_t csize = 0;
            {
                const uint32_t s0 = lane * kPlanPerLane;
                uint32_t has = 0, val = 0;  // this lane's segments as one function of the incoming carry
                for (uint32_t k = 0; k < kPlanPerLane; k++) {
                    const uint32_t sg = s0 + k;
                    if (sg < nseg) {
                        const SegRec r = recs[sg];
                        const uint32_t t = r.off_t >> 16;
                        if (r.lead_ml >> 16) { has = 1; val = t; } else val += t;
                    }
                }
                uint32_t ihas = has, ival = val;  // inclusive scan of the composition (earlier lanes first)
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t ph_ = __shfl_up_sync(kFull, ihas, d), pv = __shfl_up_sync(kFull, ival, d);
                    if ((int)lane >= d && !ihas) { ihas = ph_; ival += pv; }
                }
                uint32_t carry = __shfl_up_sync(kFull, ival, 1);  // what reaches this lane's first segment
                if (lane == 0) carry = 0;
                const uint32_t carry_end = __shfl_sync(kFull, ival, 31);  // literals behind the block's last match
                uint32_t fll[kPlanPerLane], fsz[kPlanPerLane], msz[kPlanPerLane], mine_total = 0;
#pragma unroll
                for (uint32_t k = 0; k < kPlanPerLane; k++) {
                    const uint32_t sg = s0 + k;
                    fll[k] = fsz[k] = msz[k] = 0;
                    if (sg < nseg) {
                        const SegRec r = recs[sg];
                        const uint32_t ml = r.lead_ml >> 16, t = r.off_t >> 16;
                        msz[k] = r.mbytes;
                        if (ml) {
                            fll[k] = carry + (r.lead_ml & 0xffffu);
                            fsz[k] = seq_bytes_fast(fll[k], ml);
                            carry = t;
                        } else carry += t;
                        mine_total += fsz[k] + msz[k];
                    }
                }
                uint32_t incl = mine_total;
#pragma unroll
                for (int d = 1; d < 32; d <<= 1) {
                    const uint32_t t = __shfl_up_sync(kFull, incl, d);
                    if ((int)lane >= d) incl += t;
                }
                uint32_t o = incl - mine_total;
                const uint32_t total = __shfl_sync(kFull, incl, 31);
#pragma unroll
                for (uint32_t k = 0; k < kPlanPerLane; k++) {
                    const uint32_t sg = s0 + k;
                    if (sg < nseg) {
                        SegPlan pl;
                        pl.foff = o;
                        pl.moff = o + fsz[k];
                        pl.fll = fll[k];
                        pl.pad = 0;
                        plans[sg] = pl;
                        o += fsz[k] + msz[k];
                    }
                }
                const uint32_t last = nseg == 0 ? L : carry_end;
                if (lane == 0) {
                    ctl->last_lits = last;
                    ctl->tail_off = total;  // where the final literal run starts (relative to the block's first data byte)
                }
                csize = total + 1 + last + (last >= 15 ? (last - 15) / 255 + 1 : 0);
            }
            if (lane == 0) {
                const BlockPlace pl = place_block<kBlkChk>(p, *dsc, csize, L);
                ctl->raw = pl.raw;
                ctl->data = pl.data;
                if constexpr (kBlkChk) ctl->size = pl.raw ? L : csize;
            }
        }
        __syncthreads();

        // ---------------------------------------------------------------- write the block to its final place (all warps)
        {
            uint8_t *out = dsc->dst + ctl->data;
            if (ctl->raw) {
                // stored block: straight from the input (L2-hot: the bulk load just pulled it)
                copy_block<kWarps, true>(out, src, L, warp, lane);
            } else {
                for (uint32_t s = warp; s < nseg; s += kWarps) {
                    const SegRec r = recs[s];
                    const SegPlan pl = plans[s];
                    const uint32_t ml = r.lead_ml >> 16;
                    if (ml) {
                        const uint32_t lit_start = r.seg_pos + (r.lead_ml & 0xffffu) - pl.fll;
                        emit_seq(out, pl.foff, src, lit_start, pl.fll, ml, r.off_t & 0xffffu, lane);
                    }
                    if (r.mbytes) warp_copy_stream<false>(out + pl.moff, scratch + r.seg_pos + s * kSegPad, r.mbytes, lane);
                }
                if (warp == kWarps - 1) {
                    const uint32_t ll = ctl->last_lits;
                    emit_seq(out, ctl->tail_off, src, L - ll, ll, 0, 0, lane);
                }
            }
            if constexpr (kBlkChk) {
                if (warp == kSumWarp) {
                    run_pending(&ctl->pend, lane);  // (still pending only when this block had no segment to parse)
                    set_pending(&ctl->pend, out, ctl->size, lane);
                }
            }
        }
    }
}

__global__ void __launch_bounds__(kThreads, 2) sky_fused_kernel(const Params p) { fused_body<false, false>(p); }
// SKY_F_CHECKSUM: the same kernel with the content checksum computed by the MD5 lanes (sky_checksum_kernel writes it).
__global__ void __launch_bounds__(kThreads, 2) sky_fused_xxh_kernel(const Params p) { fused_body<true, false>(p); }
// SKY_F_BLOCK_CHECKSUM, without and with SKY_F_CHECKSUM: frames with LZ4's block checksums.
__global__ void __launch_bounds__(kThreads, 2) sky_fused_bc_kernel(const Params p) { fused_body<false, true>(p); }
__global__ void __launch_bounds__(kThreads, 2) sky_fused_xxh_bc_kernel(const Params p) { fused_body<true, true>(p); }

// SKY_F_CHECKSUM epilogue (finish_frame, frame.cuh), one thread per chunk, after the compressor has finished the frame.
__global__ void sky_checksum_kernel(const ChunkDesc *chunks, const uint32_t *xxh, uint64_t *out_len, uint32_t n) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= n) return;
    finish_frame(chunks[c].dst, out_len + c, xxh[c]);
}


// ------------------------------------------------------------------------------------ receiver side
struct DecParams {
    DecChunk *chunks;
    DecBlock *blocks;
    int32_t *status;     // per chunk, 0 = ok (mapped host memory)
    uint32_t *dec_done;  // per chunk: leading blocks fully decoded (linked frames wait on it)
    uint32_t *counter;   // work counter
    uint32_t *blk_done;  // per block: 1 once decoded (gates the MD5 lanes)
    const uint32_t *md5_order;
    uint8_t *md5_out;    // 16 bytes per chunk (every chunk has an MD5 lane, which also settles its status)
    uint32_t n_chunks;
    uint32_t n_groups;
    uint32_t rows;
};

__global__ void sky_frame_index_kernel(const DecParams p) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= p.n_chunks) return;
    DecChunk cd = p.chunks[c];
    int32_t st = kDecOk;
    frame_index(cd, p.blocks + cd.blk_base, &st);
    p.chunks[c].linked = cd.linked;
    p.chunks[c].checks = cd.checks;
    p.chunks[c].content_xxh = cd.content_xxh;
    p.status[c] = st;
}

// Gate for the MD5 lanes of the receiver: row `row` of a chunk may be hashed once its block has been decoded.
struct DecRowGate {
    const uint32_t *flags;  // this lane's chunk: one word per block, non-zero = decoded (or failed: hash garbage, status says so)
    __device__ __forceinline__ void operator()(uint64_t row, bool wants) const {
        // Poll with relaxed loads and acquire once: an acquire load at gpu scope invalidates the SM's L1 (CCTL.IVALL),
        // and an MD5 lane waiting on the decoder polls thousands of times, under the decode warps of its SM.
        unsigned ns = 128;
        for (;;) {
            const bool ready = !wants || ld_relaxed32(flags + row) != 0;
            if (__all_sync(kFull, ready)) break;
            __nanosleep(ns);
            if (ns < 4096) ns <<= 1;
        }
        asm volatile("fence.acq_rel.gpu;" ::: "memory");
    }
};

// Persistent: warps 0..3 of a CTA may host an MD5 group (digest of the decoded bytes, following the decode through
// per-block flags); every other warp (and MD5 warps once their groups are done) decodes blocks.  The MD5 lanes always
// compute the XXH32 of the decoded bytes too (whether a frame carries a content checksum is only known on the device)
// and compare it where the frame has one.
__global__ void __launch_bounds__(512, 1) sky_decode_kernel(const DecParams p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (warp < kMd5WarpsPerCta) {
        const uint32_t md5_slots = gridDim.x * kMd5WarpsPerCta;
        for (uint32_t g = warp * gridDim.x + blockIdx.x; g < p.n_groups; g += md5_slots) {
            const uint32_t c = p.md5_order[g * 32 + lane];
            const bool active = c != 0xffffffffu;
            const uint8_t *src = nullptr;
            uint64_t len = 0;
            DecRowGate gate{nullptr};
            if (active) {
                src = p.chunks[c].out;
                len = p.chunks[c].raw_len;
                gate.flags = p.blk_done + p.chunks[c].blk_base;
            }
            const uint32_t x = md5_warp<true, DecRowGate, kDecMd5Slots>(reinterpret_cast<uint32_t *>(smem + warp * kDecRingBytes), src, len,
                                                                        active, p.md5_out + (size_t)(active ? c : 0) * 16, lane, gate);
            // every row has passed the gate, so no decode warp reads or writes the status any more: settle a block failure
            // into its code (lz4dec.cuh); a content checksum mismatch only replaces ok
            if (active) {
                const int32_t s = settle_status(*reinterpret_cast<volatile int32_t *>(p.status + c));
                if (s != kDecOk) p.status[c] = s;
                else if ((p.chunks[c].checks & kChkContent) && x != p.chunks[c].content_xxh) atomicCAS(p.status + c, kDecOk, kDecChecksum);
            }
            __syncwarp();
        }
    }
    // A failing block folds block_fail(j, code) into the chunk's status with atomicMin, so the earliest failing block wins
    // whichever warp gets there first (liblz4 checks and decodes blocks in order and reports the first error); the chunk's
    // MD5 lane turns it back into that block's code.  A block is skipped only once the header or an earlier block failed.
    for (uint32_t c, j; claim_row_major(p.counter, p.n_chunks, p.rows, lane, c, j);) {
        const DecChunk cd = p.chunks[c];
        if (j >= cd.nblk) continue;
        int32_t st = *reinterpret_cast<volatile int32_t *>(p.status + c);
        const uint64_t pos = (uint64_t)j * kBlock;
        const uint32_t want = (uint32_t)min((uint64_t)kBlock, cd.raw_len - pos);
        if (cd.linked) {  // matches may reach into earlier blocks: decode in order within the chunk
            if (lane == 0) {
                unsigned ns = 64;
                while (ld_acquire32(p.dec_done + c) < j) {
                    __nanosleep(ns);
                    if (ns < 2048) ns <<= 1;
                }
            }
            __syncwarp();
            st = *reinterpret_cast<volatile int32_t *>(p.status + c);
        }
        if (block_may_run(st, j)) {
            const DecBlock b = p.blocks[cd.blk_base + j];
            const uint32_t sz = b.word & 0x7FFFFFFFu;
            if ((cd.checks & kChkBlock) && xxh32_warp(cd.frame + b.off, sz, lane) != b.chk) {
                st = kDecChecksum;
            } else if (b.word & 0x80000000u) {
                st = sz != want ? kDecLayout : kDecOk;
                if (st == kDecOk) warp_copy(cd.out + pos, cd.frame + b.off, sz, lane);
            } else {
                st = lz4_decode_block(cd.frame + b.off, sz, cd.out, pos, want, cd.linked ? 0 : pos, lane);
            }
            if (st != kDecOk && lane == 0) atomicMin(p.status + c, block_fail(j, st));
        }
        __syncwarp();
        if (lane == 0) {
            __threadfence();
            if (cd.linked) st_release32(p.dec_done + c, j + 1);
            st_release32(p.blk_done + cd.blk_base + j, 1u);  // lets the MD5 lane of this chunk enter the row
        }
    }
}

// ---- E2EE glue: describe one box per chunk once the frame lengths exist (they are only known on the device; the open
// side knows every length before it starts, so its descriptors are built on the host, see launch_open).
// seal: msg = the chunk's frame (or, without LZ4, its raw bytes), box = box_base + (frame offset in the frame slab) + 64*i + 8,
// so that box + 40 is 16-byte aligned; the nonce is copied in, out_len becomes the box length.
// kPass (SKY_F_PASSTHROUGH): msg = the frame where it is smaller than the chunk, otherwise the chunk's own bytes, and
// pass[i] = 1 for a chunk sealed raw.
template <bool kPass>
__device__ __forceinline__ void box_setup_body(BoxChunk *bc, uint64_t *blk_base, const ChunkDesc *desc, uint32_t n, uint64_t *out_len,
                                               const uint8_t *frame_slab, uint8_t *box_slab, const uint8_t *nonces, int use_frames,
                                               uint8_t *pass) {
    for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) {
        const ChunkDesc d = desc[i];
        BoxChunk b;
        b.box = box_slab + (d.dst - frame_slab) + 64ull * i + 8;
        if (kPass) {
            const bool raw = out_len[i] >= d.len;
            b.msg = raw ? d.src : d.dst;
            b.len = raw ? d.len : out_len[i];
            pass[i] = raw;
        } else {
            b.msg = use_frames ? d.dst : d.src;
            b.len = use_frames ? out_len[i] : d.len;
        }
        for (int k = 0; k < 24; k++) b.box[k] = nonces[24ull * i + k];
        bc[i] = b;
        out_len[i] = b.len + kBoxOverhead;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t acc = 0;
        for (uint32_t i = 0; i < n; i++) {
            blk_base[i] = acc;
            acc += box_stream_blocks(bc[i].len);
        }
        blk_base[n] = acc;
    }
}
__global__ void sky_box_setup_kernel(BoxChunk *bc, uint64_t *blk_base, const ChunkDesc *desc, uint32_t n, uint64_t *out_len,
                                     const uint8_t *frame_slab, uint8_t *box_slab, const uint8_t *nonces, int use_frames) {
    box_setup_body<false>(bc, blk_base, desc, n, out_len, frame_slab, box_slab, nonces, use_frames, nullptr);
}
__global__ void sky_box_setup_pass_kernel(BoxChunk *bc, uint64_t *blk_base, const ChunkDesc *desc, uint32_t n, uint64_t *out_len,
                                          const uint8_t *frame_slab, uint8_t *box_slab, const uint8_t *nonces, uint8_t *pass) {
    box_setup_body<true>(bc, blk_base, desc, n, out_len, frame_slab, box_slab, nonces, 1, pass);
}

// SKY_F_PASSTHROUGH without E2EE: a chunk whose final frame is not smaller than the chunk is sent as itself.  pass[i] = 1
// and out_len[i] = 0 for it, so that nothing is copied back (the caller holds the chunk's bytes).
__global__ void sky_passthrough_kernel(const ChunkDesc *desc, uint64_t *out_len, uint8_t *pass, uint32_t n) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const bool raw = out_len[i] >= desc[i].len;
    pass[i] = raw;
    if (raw) out_len[i] = 0;
}

}  // namespace sky

// ======================================================================================= host side
using namespace sky;

// Owner of one CUDA resource (a device or pinned allocation, an event, a stream): move-only, released by its destructor
// or reset().  put() releases what it holds and hands out the handle a cudaMalloc / cudaEventCreate / ... call fills.
template <class H, auto Release>
class Owned {
    H h_ = nullptr;

  public:
    Owned() = default;
    Owned(Owned &&o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
    Owned &operator=(Owned &&o) noexcept { std::swap(h_, o.h_); return *this; }
    ~Owned() { reset(); }
    void reset() { if (h_) Release(std::exchange(h_, nullptr)); }
    H *put() { reset(); return &h_; }
    operator H() const { return h_; }
};
template <class T> using DevMem = Owned<T *, cudaFree>;
template <class T> using PinnedMem = Owned<T *, cudaFreeHost>;
using Event = Owned<cudaEvent_t, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
// Mapped pinned memory: kernels store into it straight over PCIe through `d`, the device view of `h`.
template <class T>
struct Mapped {
    PinnedMem<T> h;
    T *d = nullptr;
    cudaError_t alloc(size_t n) {
        const cudaError_t e = cudaHostAlloc(h.put(), n * sizeof(T), cudaHostAllocMapped | cudaHostAllocPortable);
        return e == cudaSuccess ? cudaHostGetDevicePointer(&d, h, 0) : e;
    }
};

// A slot's memory, one part per role (pinned host mirror h_*, device array d_*).  The batch metadata is built with the
// slot; the decode and box arrays by the first call that needs them, all of a part or none of it.
struct BatchMeta {  // one batch's descriptors and results (the receiver uses the MD5 order, digests and counters)
    PinnedMem<ChunkDesc> h_desc; DevMem<ChunkDesc> d_desc;
    PinnedMem<uint32_t> h_order; DevMem<uint32_t> d_order;
    PinnedMem<uint64_t> h_chain; DevMem<uint64_t> d_chain;
    // results live in MAPPED pinned host memory: the kernel stores sizes / digests straight over PCIe, so no small
    // device->host copies sit in a copy-engine queue behind multi-GiB frame copies
    Mapped<uint64_t> outlen;
    Mapped<uint8_t> md5;
    Mapped<uint8_t> pass;     // SKY_F_PASSTHROUGH: per chunk 1 when its payload is the chunk itself, not its frame
    DevMem<uint32_t> xxh;     // per chunk XXH32 of the input (SKY_F_CHECKSUM)
    DevMem<uint32_t> counters;
    DevMem<uint8_t> scratch;  // compress scratch: kScratchBytes per CTA of the grid (kernels of different slots overlap)
};
struct HcArrays {  // SKY_F_HC: the HC kernel's scratch, and the stream the digests run on beside it (fork / join events)
    DevMem<uint8_t> scratch;  // kHcLinkedScratchBytes per CTA (one CTA per SM; kHcScratchBytes of it without SKY_F_LINKED)
    Stream md5_stream;
    Event ev_fork, ev_join;
};
using Kernel = void (*)(const Params);
// The fused kernel a batch runs, by [SKY_F_CHECKSUM][SKY_F_BLOCK_CHECKSUM].
static constexpr Kernel kFusedKernels[2][2] = {{sky_fused_kernel, sky_fused_bc_kernel}, {sky_fused_xxh_kernel, sky_fused_xxh_bc_kernel}};
constexpr uint32_t kHcLevelShift = 8, kHcLevelMask = 0xfu << kHcLevelShift;  // SKY_F_HC_LEVEL's field in `flags`
static_assert(SKY_F_HC_LEVEL(1) == (SKY_F_HC | (1u << kHcLevelShift)), "the level field of include/skychunk.h");
// The level a batch's flags select: the level field, or kHcDefaultLevel when it is 0.
static int hc_level(uint32_t flags) {
    const int l = (int)((flags & kHcLevelMask) >> kHcLevelShift);
    return l ? l : kHcDefaultLevel;
}
// Every HC kernel with the dynamic shared memory it is launched with: entry (row * kHcLevels + level - kHcMinLevel),
// where row's bits 2, 1, 0 are SKY_F_BLOCK_CHECKSUM, SKY_F_LINKED and SKY_F_OPTIMAL.
struct HcKernel {
    Kernel kernel;
    uint32_t smem;
};
constexpr int kHcLevels = kHcMaxLevel - kHcMinLevel + 1;
static_assert(kHcMinLevel >= 1 && kHcLevels >= 1 && kHcMaxLevel <= (int)(kHcLevelMask >> kHcLevelShift),
              "the HC levels are a range the level field can hold");
template <int I>
static constexpr HcKernel hc_kernel_at() {
    constexpr int row = I / kHcLevels;
    constexpr bool bc = row & 4, linked = row & 2, opt = row & 1;
    return {sky_hc_kernel<hc_depth(kHcMinLevel + I % kHcLevels), bc, linked, opt>, linked ? kHcLinkedSmemBytes : kHcSmemBytes};
}
template <int... I>
static constexpr std::array<HcKernel, sizeof...(I)> hc_kernels(std::integer_sequence<int, I...>) { return {hc_kernel_at<I>()...}; }
static constexpr std::array<HcKernel, 8 * kHcLevels> kHcKernels = hc_kernels(std::make_integer_sequence<int, 8 * kHcLevels>{});
// The HC kernel a batch's flags select (SKY_F_HC, its level checked by frame_flags_valid).
static const HcKernel &hc_kernel(uint32_t flags) {
    const int row = (flags & SKY_F_BLOCK_CHECKSUM ? 4 : 0) | (flags & SKY_F_LINKED ? 2 : 0) | (flags & SKY_F_OPTIMAL ? 1 : 0);
    return kHcKernels[row * kHcLevels + hc_level(flags) - kHcMinLevel];
}
struct BlockTable {  // per block of a batch, `cap` entries: what frame_index found; done = decoded (the receiver's MD5 gate)
    DevMem<DecBlock> blocks; DevMem<uint32_t> done; uint64_t cap = 0;
};
struct DecodeArrays {  // receiver side
    PinnedMem<DecChunk> h_chunks; DevMem<DecChunk> d_chunks;
    PinnedMem<int32_t> h_status; DevMem<int32_t> d_status;
    DevMem<uint32_t> d_dec_done;  // per chunk: leading blocks decoded (linked frames wait on it)
    BlockTable table;
};
struct BoxArrays {  // E2EE: box slab, per-chunk box descriptors, stream-block prefix, subkeys, nonces, tag verdicts
    DevMem<uint8_t> d_box;
    PinnedMem<BoxChunk> h_chunks; DevMem<BoxChunk> d_chunks;  // (the host writes h_chunks and h_blk_base to open boxes)
    PinnedMem<uint64_t> h_blk_base; DevMem<uint64_t> d_blk_base;
    DevMem<uint32_t> d_sub;
    PinnedMem<uint8_t> h_nonce; DevMem<uint8_t> d_nonce;
    PinnedMem<int32_t> h_status; DevMem<int32_t> d_status;
    Event ev_open;  // the boxes are on the device, the open kernels start (kernel_ms of a batch of sealed raw chunks)
};
struct VerifyArrays {  // SKY_F_VERIFY: block-table bases, statuses (device, and settled in mapped host memory), block table
    PinnedMem<uint64_t> h_blk_base; DevMem<uint64_t> d_blk_base;
    DevMem<int32_t> d_status;
    Mapped<int32_t> status;
    DevMem<uint32_t> d_counter;
    BlockTable table;
};
struct Ticket {  // the batch a slot has in flight on the host path
    bool busy = false, d2h_issued = false;
    uint64_t id = 0;
    uint32_t n = 0, flags = 0;
    std::vector<void *> dst;
    std::vector<uint64_t> out_off;
};

struct Slot {
    Stream stream;
    Event ev_k0, ev_k1;           // kernel_ms
    Event ev_res;                 // kernel(s) done: sizes + digests are in host memory
    Event ev_h2d, ev_d2h;         // input landed (on ctx->st_h2d) / frames landed (on ctx->st_d2h)
    DevMem<uint8_t> d_in, d_out;  // host-path slabs (n_slots > 0)
    BatchMeta meta;
    DecodeArrays dec;
    BoxArrays box;
    HcArrays hc;
    VerifyArrays verify;
    Ticket ticket;
};

struct sky_ctx {
    int device = 0;
    int sm_count = 0;
    uint32_t max_chunks = 0;
    uint64_t in_cap = 0, out_cap = 0;
    // Host path: every slot's input copies go FIFO through one H2D stream and every frame copy through one D2H
    // stream, so the two directions use different copy engines and batch k's frames leave while batch k+1's
    // input arrives (per-slot streams put both directions of all slots into one in-order engine queue).
    Stream st_h2d, st_d2h;
    std::vector<Slot> slots;  // slots[0] doubles as the metadata holder for sky_process_device
    DevMem<uint8_t> d_key;    // 32-byte SecretBox key (null: E2EE off); set => every slot has its box arrays
    uint64_t next_ticket = 1;
    uint64_t launches = 0;
    std::string err;
    // The members release their resources after this body: first let every copy and kernel that may use them finish.
    ~sky_ctx() {
        if (st_h2d) cudaStreamSynchronize(st_h2d);
        if (st_d2h) cudaStreamSynchronize(st_d2h);
        for (Slot &s : slots)
            if (s.stream) cudaStreamSynchronize(s.stream);
        for (Slot &s : slots)
            if (s.hc.md5_stream) cudaStreamSynchronize(s.hc.md5_stream);
    }
};

static thread_local std::string g_err;

#define CK(ctx, call)                                                                      \
    do {                                                                                   \
        cudaError_t e_ = (call);                                                           \
        if (e_ != cudaSuccess) {                                                           \
            char b_[512];                                                                  \
            snprintf(b_, sizeof b_, "%s -> %s (%s:%d)", #call, cudaGetErrorString(e_), __FILE__, __LINE__); \
            if (ctx) (ctx)->err = b_;                                                      \
            g_err = b_;                                                                    \
            return SKY_E_CUDA;                                                             \
        }                                                                                  \
    } while (0)

static int build_slot(sky_ctx *ctx, Slot &s, bool slabs) {
    const size_t nc = ctx->max_chunks, ng = (nc + 31) / 32 * 32;
    CK(ctx, cudaStreamCreateWithFlags(s.stream.put(), cudaStreamNonBlocking));
    CK(ctx, cudaEventCreate(s.ev_k0.put()));
    CK(ctx, cudaEventCreate(s.ev_k1.put()));
    CK(ctx, cudaEventCreate(s.ev_res.put()));
    CK(ctx, cudaEventCreateWithFlags(s.ev_h2d.put(), cudaEventDisableTiming));
    CK(ctx, cudaEventCreateWithFlags(s.ev_d2h.put(), cudaEventDisableTiming));
    BatchMeta &m = s.meta;
    CK(ctx, cudaMallocHost(m.h_desc.put(), nc * sizeof(ChunkDesc)));
    CK(ctx, cudaMalloc(m.d_desc.put(), nc * sizeof(ChunkDesc)));
    CK(ctx, cudaMallocHost(m.h_order.put(), ng * sizeof(uint32_t)));
    CK(ctx, cudaMalloc(m.d_order.put(), ng * sizeof(uint32_t)));
    CK(ctx, cudaMallocHost(m.h_chain.put(), nc * sizeof(uint64_t)));
    CK(ctx, cudaMalloc(m.d_chain.put(), nc * sizeof(uint64_t)));
    CK(ctx, m.outlen.alloc(nc));
    CK(ctx, m.md5.alloc(nc * 16));
    CK(ctx, m.pass.alloc(nc));
    CK(ctx, cudaMalloc(m.xxh.put(), nc * sizeof(uint32_t)));
    CK(ctx, cudaMalloc(m.counters.put(), kCountersBytes));
    CK(ctx, cudaMalloc(m.scratch.put(), (size_t)ctx->sm_count * kCtasPerSm * kScratchBytes));
    if (slabs) {
        cudaError_t e = cudaMalloc(s.d_in.put(), ctx->in_cap);
        if (e == cudaSuccess) e = cudaMalloc(s.d_out.put(), ctx->out_cap);
        if (e != cudaSuccess) { g_err = ctx->err = std::string("cudaMalloc(slab): ") + cudaGetErrorString(e); return SKY_E_NOMEM; }
    }
    return SKY_OK;
}

static int alloc_dec(sky_ctx *ctx, DecodeArrays &d) {
    if (d.d_chunks) return SKY_OK;
    const size_t nc = ctx->max_chunks;
    DecodeArrays a;
    CK(ctx, cudaMallocHost(a.h_chunks.put(), nc * sizeof(DecChunk)));
    CK(ctx, cudaMalloc(a.d_chunks.put(), nc * sizeof(DecChunk)));
    CK(ctx, cudaMallocHost(a.h_status.put(), nc * sizeof(int32_t)));
    CK(ctx, cudaMalloc(a.d_status.put(), nc * sizeof(int32_t)));
    CK(ctx, cudaMalloc(a.d_dec_done.put(), nc * sizeof(uint32_t)));
    d = std::move(a);
    return SKY_OK;
}

static int alloc_hc(sky_ctx *ctx, HcArrays &h) {
    if (h.scratch) return SKY_OK;
    HcArrays a;
    CK(ctx, cudaMalloc(a.scratch.put(), (size_t)ctx->sm_count * kHcLinkedScratchBytes));
    CK(ctx, cudaStreamCreateWithFlags(a.md5_stream.put(), cudaStreamNonBlocking));
    CK(ctx, cudaEventCreateWithFlags(a.ev_fork.put(), cudaEventDisableTiming));
    CK(ctx, cudaEventCreateWithFlags(a.ev_join.put(), cudaEventDisableTiming));
    h = std::move(a);
    return SKY_OK;
}

static int alloc_verify(sky_ctx *ctx, VerifyArrays &v) {
    if (v.d_status) return SKY_OK;
    const size_t nc = ctx->max_chunks;
    VerifyArrays a;
    CK(ctx, cudaMallocHost(a.h_blk_base.put(), nc * sizeof(uint64_t)));
    CK(ctx, cudaMalloc(a.d_blk_base.put(), nc * sizeof(uint64_t)));
    CK(ctx, cudaMalloc(a.d_status.put(), nc * sizeof(int32_t)));
    CK(ctx, a.status.alloc(nc));
    CK(ctx, cudaMalloc(a.d_counter.put(), sizeof(uint32_t)));
    v = std::move(a);
    return SKY_OK;
}

static int grow_block_table(sky_ctx *ctx, cudaStream_t st, BlockTable &t, uint64_t n) {
    if (n <= t.cap) return SKY_OK;
    CK(ctx, cudaStreamSynchronize(st));  // kernels queued earlier on `st` are done with the old arrays
    t.cap = 0;
    CK(ctx, cudaMalloc(t.blocks.put(), n * sizeof(DecBlock)));
    CK(ctx, cudaMalloc(t.done.put(), n * sizeof(uint32_t)));
    t.cap = n;
    return SKY_OK;
}

static int alloc_box(sky_ctx *ctx, BoxArrays &b) {
    if (b.d_box) return SKY_OK;
    const size_t nc = ctx->max_chunks;
    BoxArrays a;
    CK(ctx, cudaMalloc(a.d_box.put(), ctx->out_cap + 64 * nc + 256));
    CK(ctx, cudaMallocHost(a.h_chunks.put(), nc * sizeof(BoxChunk)));
    CK(ctx, cudaMalloc(a.d_chunks.put(), nc * sizeof(BoxChunk)));
    CK(ctx, cudaMallocHost(a.h_blk_base.put(), (nc + 1) * sizeof(uint64_t)));
    CK(ctx, cudaMalloc(a.d_blk_base.put(), (nc + 1) * sizeof(uint64_t)));
    CK(ctx, cudaMalloc(a.d_sub.put(), nc * 16 * sizeof(uint32_t)));
    CK(ctx, cudaMallocHost(a.h_nonce.put(), nc * 24));
    CK(ctx, cudaMalloc(a.d_nonce.put(), nc * 24));
    CK(ctx, cudaMallocHost(a.h_status.put(), nc * sizeof(int32_t)));
    CK(ctx, cudaMalloc(a.d_status.put(), nc * sizeof(int32_t)));
    CK(ctx, cudaEventCreate(a.ev_open.put()));
    b = std::move(a);
    return SKY_OK;
}

// Block geometry of a batch (sender and receiver): visit(i, nblk) for every chunk, nblk = its number of 64 KiB blocks, and
// rows = the largest nblk (at least 1): the persistent kernels take work item w = row * n + chunk from a 32-bit counter.
// A chunk over kMaxChunkBlocks blocks, or a batch of 2^32 - 1 work items or more, is SKY_E_CAPACITY.
template <class F>
static int batch_geometry(uint32_t n, const uint64_t *len, uint32_t &rows, F &&visit) {
    rows = 1;
    for (uint32_t i = 0; i < n; i++) {
        const uint64_t nb = (len[i] + kBlock - 1) / kBlock;
        if (nb > kMaxChunkBlocks) return SKY_E_CAPACITY;
        visit(i, (uint32_t)nb);
        rows = std::max(rows, (uint32_t)nb);
    }
    return (uint64_t)rows * n >= 0xffffffffull ? SKY_E_CAPACITY : SKY_OK;
}

extern "C" {

const char *sky_strerror(int code) {
    switch (code) {
    case SKY_OK: return "ok";
    case SKY_E_INVALID: return "invalid argument";
    case SKY_E_NOGPU: return "no CUDA device available (this library has no CPU fallback)";
    case SKY_E_CUDA: return "CUDA error";
    case SKY_E_CAPACITY: return "capacity exceeded";
    case SKY_E_BUSY: return "all slots busy";
    case SKY_E_TICKET: return "unknown ticket";
    case SKY_E_NOMEM: return "out of memory";
    case SKY_E_NOKEY: return "SKY_F_E2EE without a key (sky_set_e2ee_key) or without nonces";
    default: return "unknown error";
    }
}

const char *sky_last_error(const sky_ctx *ctx) { return ctx ? ctx->err.c_str() : g_err.c_str(); }
int sky_abi_version(void) { return SKY_ABI_VERSION; }

int sky_device_count(int *count) {
    if (!count) return SKY_E_INVALID;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n <= 0) {
        *count = 0;
        g_err = cudaGetErrorString(e);
        return SKY_E_NOGPU;
    }
    *count = n;
    return SKY_OK;
}

int sky_device_pci_bus_id(int device, char *buf, int len) {
    if (!buf || len < 16) return SKY_E_INVALID;
    cudaError_t e = cudaDeviceGetPCIBusId(buf, len, device);
    if (e != cudaSuccess) {
        g_err = cudaGetErrorString(e);
        return e == cudaErrorInvalidDevice ? SKY_E_INVALID : SKY_E_NOGPU;
    }
    return SKY_OK;
}

uint32_t sky_kernel_config(int what) {
    switch (what) {
    case 0: return kEntries;
    case 1: return (uint32_t)kWarps;
    case 2: return kSegSlots;
    case 3: return kMaxStepLog;
    case 4: return hc_depth(kHcDefaultLevel);
    case 5: return kHcHashBits;
    case 6: return kHcNice;
    case 7: return (uint32_t)kHcMaxLevel;
    case 8: return kHcOptSeg;
    default: return 0;
    }
}

uint64_t sky_frame_bound(uint64_t n) {
    if (n == 0) return 11;
    return kFrameHeaderBytes + n + 4 * ((n + kBlock - 1) / kBlock) + 4;
}

static uint64_t round16(uint64_t x) { return (x + 15) & ~15ull; }

int sky_ctx_create(int device, uint64_t max_batch_bytes, uint32_t max_chunks, uint32_t n_slots, sky_ctx **out) {
    if (!out || max_chunks == 0) return SKY_E_INVALID;
    *out = nullptr;
    int ndev = 0;
    if (sky_device_count(&ndev) != SKY_OK) return SKY_E_NOGPU;
    if (device < 0 || device >= ndev) return SKY_E_INVALID;
    std::unique_ptr<sky_ctx> ctx(new (std::nothrow) sky_ctx());  // an early return releases what was built so far
    if (!ctx) return SKY_E_NOMEM;
    ctx->device = device;
    ctx->max_chunks = max_chunks;
    // every chunk is placed at a 16-byte aligned offset; frames need bound(len) each (+ 4 with SKY_F_CHECKSUM), and a
    // received frame with block checksums 4 more bytes per block
    ctx->in_cap = round16(max_batch_bytes) + 16ull * max_chunks + 256;
    ctx->out_cap = max_batch_bytes + (uint64_t)max_chunks * (64 + 4 * 3) + 8 * (max_batch_bytes / kBlock + 1) + 256;
    CK(ctx, cudaSetDevice(device));
    CK(ctx, cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device));
    cudaError_t e = cudaSuccess;
    for (const auto &row : kFusedKernels)
        for (const Kernel k : row) {
            if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kSmemBytes);
            if (e == cudaSuccess) e = cudaFuncSetAttribute(k, cudaFuncAttributePreferredSharedMemoryCarveout, 100);
        }
    for (const HcKernel &k : kHcKernels)
        if (e == cudaSuccess) e = cudaFuncSetAttribute(k.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)k.smem);
    if (e != cudaSuccess) {
        g_err = ctx->err = std::string("cudaFuncSetAttribute(smem): ") + cudaGetErrorString(e) + " (this build carries sm_90a code only)";
        return SKY_E_CUDA;
    }
    if (n_slots) {
        CK(ctx, cudaStreamCreateWithFlags(ctx->st_h2d.put(), cudaStreamNonBlocking));
        CK(ctx, cudaStreamCreateWithFlags(ctx->st_d2h.put(), cudaStreamNonBlocking));
    }
    ctx->slots.resize(n_slots ? n_slots : 1);
    for (Slot &s : ctx->slots) {
        const int rc = build_slot(ctx.get(), s, n_slots != 0);
        if (rc != SKY_OK) return rc;
    }
    *out = ctx.release();
    return SKY_OK;
}

int sky_ctx_destroy(sky_ctx *ctx) {
    if (!ctx) return SKY_E_INVALID;
    cudaSetDevice(ctx->device);
    delete ctx;
    return SKY_OK;
}

void *sky_pinned_alloc(uint64_t bytes) {
    void *p = nullptr;
    cudaError_t e = cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable);
    if (e != cudaSuccess) {
        g_err = cudaGetErrorString(e);
        return nullptr;
    }
    return p;
}
int sky_pinned_free(void *p) {
    if (!p) return SKY_OK;
    return cudaFreeHost(p) == cudaSuccess ? SKY_OK : SKY_E_CUDA;
}

uint64_t sky_box_bound(uint64_t n) { return sky_frame_bound(n) + kBoxOverhead; }

int sky_set_e2ee_key(sky_ctx *ctx, const uint8_t *key32) {
    if (!ctx) return SKY_E_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    if (!key32) {
        ctx->d_key.reset();
        return SKY_OK;
    }
    for (Slot &s : ctx->slots) {  // boxes first: no key is installed unless every slot can seal and open
        const int rc = alloc_box(ctx, s.box);
        if (rc != SKY_OK) return rc;
    }
    DevMem<uint8_t> key;
    CK(ctx, cudaMalloc(key.put(), 32));
    CK(ctx, cudaMemcpy(key, key32, 32, cudaMemcpyHostToDevice));
    ctx->d_key = std::move(key);  // (the previous key, if any, is released with `key`)
    return SKY_OK;
}

// Seal the batch's frames (or raw chunks; with SKY_F_PASSTHROUGH each chunk's frame or the chunk, whichever is smaller) on
// `st` after the fused kernel: setup -> keys -> xor -> tag.
static int launch_seal(sky_ctx *ctx, Slot &s, cudaStream_t st, uint32_t n, uint8_t *d_dst, uint32_t flags) {
    const int use_frames = (flags & SKY_F_LZ4) ? 1 : 0;
    BoxArrays &b = s.box;
    if (flags & SKY_F_PASSTHROUGH)
        sky_box_setup_pass_kernel<<<1, 256, 0, st>>>(b.d_chunks, b.d_blk_base, s.meta.d_desc, n, s.meta.outlen.d, d_dst, b.d_box, b.d_nonce,
                                                     s.meta.pass.d);
    else
        sky_box_setup_kernel<<<1, 256, 0, st>>>(b.d_chunks, b.d_blk_base, s.meta.d_desc, n, s.meta.outlen.d, d_dst, b.d_box, b.d_nonce, use_frames);
    CK(ctx, cudaGetLastError());
    sky_box_keys_kernel<<<(n + 63) / 64, 64, 0, st>>>(b.d_chunks, n, ctx->d_key, b.d_sub);
    CK(ctx, cudaGetLastError());
    sky_box_xor_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(b.d_chunks, b.d_blk_base, n, b.d_sub, 0);
    CK(ctx, cudaGetLastError());
    sky_box_tag_kernel<<<n, kPolyThreads, 0, st>>>(b.d_chunks, b.d_sub, 0, nullptr);
    CK(ctx, cudaGetLastError());
    ctx->launches += 4;
    return SKY_OK;
}

// Open the n boxes on slot `s`: copy box i to the box slab at box_off[i] + 64 * i + 8 (box_off: 16-byte aligned, at least
// box_len[i] apart), and open it into d_msg + msg_off[i] (16-byte aligned; msg_len[i] = its message bytes) -- the frame
// slab when the messages are frames to decode, the input slab when they are the chunks themselves: keys -> tag -> xor,
// then the tag verdicts to the host.  Every offset and length is known before the kernels run, so the host writes the
// descriptors.
static int launch_open(sky_ctx *ctx, Slot &s, uint32_t n, const void *const *boxes, const uint64_t *box_len, const uint64_t *box_off,
                       uint8_t *d_msg, const uint64_t *msg_off, uint64_t *msg_len) {
    BoxArrays &b = s.box;
    const cudaStream_t st = s.stream;
    uint64_t acc = 0;
    for (uint32_t i = 0; i < n; i++) {
        uint8_t *box = b.d_box + box_off[i] + 64ull * i + 8;
        CK(ctx, cudaMemcpyAsync(box, boxes[i], box_len[i], cudaMemcpyHostToDevice, st));
        msg_len[i] = box_len[i] >= (uint64_t)kBoxOverhead ? box_len[i] - kBoxOverhead : 0;
        b.h_chunks[i] = BoxChunk{box, d_msg + msg_off[i], msg_len[i]};
        b.h_blk_base[i] = acc;
        acc += box_stream_blocks(msg_len[i]);
    }
    b.h_blk_base[n] = acc;
    CK(ctx, cudaMemcpyAsync(b.d_chunks, b.h_chunks, n * sizeof(BoxChunk), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemcpyAsync(b.d_blk_base, b.h_blk_base, (n + 1) * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaEventRecord(b.ev_open, st));
    sky_box_keys_kernel<<<(n + 63) / 64, 64, 0, st>>>(b.d_chunks, n, ctx->d_key, b.d_sub);
    CK(ctx, cudaGetLastError());
    sky_box_tag_kernel<<<n, kPolyThreads, 0, st>>>(b.d_chunks, b.d_sub, 1, b.d_status);
    CK(ctx, cudaGetLastError());
    sky_box_xor_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(b.d_chunks, b.d_blk_base, n, b.d_sub, 1);
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaMemcpyAsync(b.h_status, b.d_status, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    ctx->launches += 3;
    return SKY_OK;
}

// MD5 lane assignment (sender and receiver): chunk indices longest first, so a warp's 32 lanes carry similar lengths,
// padded with 0xffffffff to whole groups of 32.  Returns the number of groups.
static uint32_t fill_md5_order(uint32_t *order, uint32_t n, const uint64_t *len) {
    const uint32_t ng = (n + 31) / 32;
    std::iota(order, order + n, 0u);
    std::stable_sort(order, order + n, [&](uint32_t a, uint32_t b) { return len[a] > len[b]; });
    std::fill(order + n, order + ng * 32, 0xffffffffu);
    return ng;
}

// SKY_F_HC selects how frames are made, SKY_F_CHECKSUM / SKY_F_BLOCK_CHECKSUM add to the frame and SKY_F_VERIFY checks
// it, so each needs SKY_F_LZ4, or no stage bit at all (= LZ4 + MD5).  A level field needs SKY_F_HC and a level in kHcMinLevel .. kHcMaxLevel.
// SKY_F_LINKED and SKY_F_OPTIMAL need SKY_F_HC: only the high-ratio compressor links blocks and parses optimally.
// SKY_F_PASSTHROUGH chooses between a frame and the chunk, so it needs SKY_F_LZ4 too, and a raw payload cannot carry the
// LZ4 checksums SKY_F_CHECKSUM / SKY_F_BLOCK_CHECKSUM ask for.
static bool frame_flags_valid(uint32_t flags) {
    if ((flags & kHcLevelMask) && (!(flags & SKY_F_HC) || hc_level(flags) < kHcMinLevel || hc_level(flags) > kHcMaxLevel))
        return false;
    if ((flags & (SKY_F_LINKED | SKY_F_OPTIMAL)) && !(flags & SKY_F_HC)) return false;
    if ((flags & SKY_F_PASSTHROUGH) && (flags & (SKY_F_CHECKSUM | SKY_F_BLOCK_CHECKSUM))) return false;
    return !(flags & (SKY_F_HC | SKY_F_CHECKSUM | SKY_F_BLOCK_CHECKSUM | SKY_F_VERIFY | SKY_F_PASSTHROUGH)) ||
           (flags & (SKY_F_LZ4 | SKY_F_MD5)) != SKY_F_MD5;
}
// Bytes a chunk's frame may take: SKY_F_CHECKSUM adds the 4-byte content checksum behind the EndMark,
// SKY_F_BLOCK_CHECKSUM 4 bytes behind every block.
static uint64_t frame_need(uint64_t n, uint32_t flags) {
    return sky_frame_bound(n) + ((flags & SKY_F_CHECKSUM) ? 4 : 0) + ((flags & SKY_F_BLOCK_CHECKSUM) ? 4 * ((n + kBlock - 1) / kBlock) : 0);
}
// No stage bit means LZ4 + MD5.
static uint32_t with_stages(uint32_t flags) { return (flags & (SKY_F_LZ4 | SKY_F_MD5)) ? flags : flags | SKY_F_LZ4 | SKY_F_MD5; }

// Enqueues the frame check (SKY_F_VERIFY, lz4verify.cuh) of the n chunks in the slot's batch metadata (h_desc / d_desc,
// the frame lengths in outlen, the content checksums in xxh under SKY_F_CHECKSUM) on `st`: index, block check, settle.
// flags: what the frames were made with (FLG, checksums); repair: rewrite every failing frame as its stored-block frame.
// The settled statuses land in s.verify.status.
static int launch_verify(sky_ctx *ctx, Slot &s, cudaStream_t st, uint32_t n, uint32_t rows, uint32_t flags, bool repair) {
    int rc = alloc_verify(ctx, s.verify);
    if (rc != SKY_OK) return rc;
    VerifyArrays &v = s.verify;
    BatchMeta &m = s.meta;
    uint64_t nblk_total = 0;
    for (uint32_t i = 0; i < n; i++) {
        v.h_blk_base[i] = nblk_total;
        nblk_total += m.h_desc[i].nblk;
    }
    rc = grow_block_table(ctx, st, v.table, nblk_total + 1);
    if (rc != SKY_OK) return rc;
    CK(ctx, cudaMemcpyAsync(v.d_blk_base, v.h_blk_base, n * sizeof(uint64_t), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemsetAsync(v.d_counter, 0, sizeof(uint32_t), st));
    VerifyParams p;
    p.chunks = m.d_desc;
    p.frame_len = m.outlen.d;
    p.xxh = (flags & SKY_F_CHECKSUM) ? (const uint32_t *)m.xxh : nullptr;
    p.blk_base = v.d_blk_base;
    p.blocks = v.table.blocks;
    p.status = v.d_status;
    p.status_out = v.status.d;
    p.counter = v.d_counter;
    p.n_chunks = n;
    p.rows = rows;
    p.flags = flags;
    p.repair = repair ? 1u : 0u;
    const bool linked = (flags & SKY_F_LINKED) != 0;
    (linked ? sky_verify_linked_index_kernel : sky_verify_index_kernel)<<<(n + 127) / 128, 128, 0, st>>>(p);
    CK(ctx, cudaGetLastError());
    (linked ? sky_verify_linked_kernel : sky_verify_kernel)<<<ctx->sm_count * 2, kVerifyThreads, 0, st>>>(p);
    CK(ctx, cudaGetLastError());
    (linked ? sky_verify_linked_settle_kernel : sky_verify_settle_kernel)<<<n, kRepairWarps * 32, 0, st>>>(p);
    CK(ctx, cudaGetLastError());
    ctx->launches += 3;
    return SKY_OK;
}

// Fills the slot's metadata for a batch and enqueues: meta H2D, counter reset, fused kernel, results D2H.
// `meta_st`: stream the three small metadata copies ride on (the H2D stream on the host path, so they are
// never queued behind another batch's frame copies); `st`: the stream the kernel runs on.  `flags` has a stage bit
// (with_stages).
static int launch_batch(sky_ctx *ctx, Slot &s, cudaStream_t st, cudaStream_t meta_st, uint32_t n, const uint8_t *d_src,
                        const uint64_t *src_off, const uint64_t *src_len, uint8_t *d_dst, const uint64_t *dst_off, uint32_t flags) {
    if (flags & SKY_F_CHECKSUM) flags |= SKY_F_MD5;  // the content checksum comes from the MD5 lanes
    const bool xxh = (flags & SKY_F_CHECKSUM) != 0, bc = (flags & SKY_F_BLOCK_CHECKSUM) != 0;
    if (flags & SKY_F_HC) {
        const int hrc = alloc_hc(ctx, s.hc);
        if (hrc != SKY_OK) return hrc;
    }
    BatchMeta &m = s.meta;
    uint32_t rows;
    int rc = batch_geometry(n, src_len, rows, [&](uint32_t i, uint32_t nblk) {
        m.h_desc[i] = ChunkDesc{d_src + src_off[i], d_dst + dst_off[i], src_len[i], nblk};
        m.h_chain[i] = kFrameHeaderBytes;  // OFF word: block 0 starts right after the frame header
    });
    if (rc != SKY_OK) return rc;
    const uint32_t ng = fill_md5_order(m.h_order, n, src_len);

    CK(ctx, cudaMemcpyAsync(m.d_desc, m.h_desc, n * sizeof(ChunkDesc), cudaMemcpyHostToDevice, meta_st));
    CK(ctx, cudaMemcpyAsync(m.d_order, m.h_order, ng * 32 * sizeof(uint32_t), cudaMemcpyHostToDevice, meta_st));
    CK(ctx, cudaMemcpyAsync(m.d_chain, m.h_chain, n * sizeof(uint64_t), cudaMemcpyHostToDevice, meta_st));
    if (meta_st != st) {
        CK(ctx, cudaEventRecord(s.ev_h2d, meta_st));  // input (enqueued earlier on meta_st) + metadata have landed
        CK(ctx, cudaStreamWaitEvent(st, s.ev_h2d, 0));
    }
    CK(ctx, cudaMemsetAsync(m.counters, 0, kCountersBytes, st));  // the claim counter and the per-SM chain words
    memset(m.outlen.h, 0, n * sizeof(uint64_t));  // host-side clear (mapped memory; the slot is idle here)
    memset(m.md5.h, 0, (size_t)n * 16);

    Params p;
    p.chunks = m.d_desc;
    p.md5_order = m.d_order;
    p.chain = m.d_chain;
    p.out_len = m.outlen.d;
    p.md5_out = m.md5.d;
    p.counters = m.counters;
    p.scratch = m.scratch;
    p.n_chunks = n;
    p.n_groups = ng;
    const uint32_t grid = (uint32_t)ctx->sm_count * kCtasPerSm;
    // digest CTAs: 4 groups (one per SM sub-partition) each; with few groups spread them one per CTA first.  (Whole digest
    // SMs -- 4 or 8 MD5 warps on a few SMs, nothing else there -- would leave fewer block buffers idle, but with 8 or 16 MiB
    // chunks such packed MD5 warps ran at about half their chain rate, so the spread-out arrangement stays.)
    p.n_md5_ctas = (flags & SKY_F_MD5) ? std::min(grid, std::max((ng + kMd5WarpsPerCta - 1) / kMd5WarpsPerCta,
                                                                 std::min(ng, (uint32_t)ctx->sm_count / 4))) : 0;
    p.rows = rows;
    p.flags = flags;
    p.xxh_out = m.xxh;
    CK(ctx, cudaEventRecord(s.ev_k0, st));
    if (flags & SKY_F_HC) {
        // high-ratio frames from sky_hc_kernel; the digests from the fused kernel's MD5-only mode on a forked stream, so
        // the two run side by side (the HC kernel's CTAs take the SMs as the digest CTAs leave them)
        HcArrays &h = s.hc;
        const bool md5 = (flags & SKY_F_MD5) != 0;
        if (md5) {
            CK(ctx, cudaEventRecord(h.ev_fork, st));
            CK(ctx, cudaStreamWaitEvent(h.md5_stream, h.ev_fork, 0));
            Params pm = p;
            pm.flags = SKY_F_MD5;
            kFusedKernels[xxh][false]<<<grid, kThreads, kSmemBytes, h.md5_stream>>>(pm);
            CK(ctx, cudaGetLastError());
            CK(ctx, cudaEventRecord(h.ev_join, h.md5_stream));
            ctx->launches++;
        }
        p.scratch = h.scratch;
        const HcKernel &k = hc_kernel(flags);
        k.kernel<<<ctx->sm_count, kHcThreads, k.smem, st>>>(p);
        CK(ctx, cudaGetLastError());
        if (md5) CK(ctx, cudaStreamWaitEvent(st, h.ev_join, 0));
    } else {
        kFusedKernels[xxh][bc]<<<grid, kThreads, kSmemBytes, st>>>(p);
        CK(ctx, cudaGetLastError());
    }
    ctx->launches++;
    if (xxh) {  // the content checksum behind every frame's EndMark
        sky_checksum_kernel<<<(n + 127) / 128, 128, 0, st>>>(m.d_desc, m.xxh, m.outlen.d, n);
        CK(ctx, cudaGetLastError());
        ctx->launches++;
    }
    if (flags & SKY_F_VERIFY) {  // every frame is final here: check it, and repair it before it is sealed or copied out
        rc = launch_verify(ctx, s, st, n, rows, flags, true);
        if (rc != SKY_OK) return rc;
    }
    CK(ctx, cudaEventRecord(s.ev_k1, st));
    if (flags & SKY_F_E2EE) {
        rc = launch_seal(ctx, s, st, n, d_dst, flags);
        if (rc != SKY_OK) return rc;
    } else if (flags & SKY_F_PASSTHROUGH) {  // every frame is final: mark the chunks that go as themselves
        sky_passthrough_kernel<<<(n + 127) / 128, 128, 0, st>>>(m.d_desc, m.outlen.d, m.pass.d, n);
        CK(ctx, cudaGetLastError());
        ctx->launches++;
    }
    CK(ctx, cudaEventRecord(s.ev_res, st));  // kernel(s) done => sizes + digests are in host memory
    return SKY_OK;
}

// Frame copies need the compressed sizes, which only exist after the kernel.  Every host-path entry point
// calls this: for each in-flight slot whose sizes have reached the host (ev_res done) it enqueues the exact-length
// D2H copies on the ctx's D2H stream, so batch k's D2H overlaps batch k+1's H2D and kernel without a helper thread.
static int issue_d2h(sky_ctx *ctx, Slot &s) {
    Ticket &t = s.ticket;
    CK(ctx, cudaStreamWaitEvent(ctx->st_d2h, s.ev_res, 0));
    for (uint32_t i = 0; i < t.n; i++) {
        if (s.meta.outlen.h[i] == 0) continue;  // MD5-only batch without E2EE: nothing comes back but the digests
        const uint8_t *from = (t.flags & SKY_F_E2EE) ? s.box.d_box + t.out_off[i] + 64ull * i + 8 : s.d_out + t.out_off[i];
        CK(ctx, cudaMemcpyAsync(t.dst[i], from, s.meta.outlen.h[i], cudaMemcpyDeviceToHost, ctx->st_d2h));
    }
    CK(ctx, cudaEventRecord(s.ev_d2h, ctx->st_d2h));
    t.d2h_issued = true;
    return SKY_OK;
}
static int progress(sky_ctx *ctx) {
    for (Slot &s : ctx->slots) {
        if (!s.ticket.busy || s.ticket.d2h_issued) continue;
        cudaError_t q = cudaEventQuery(s.ev_res);
        if (q == cudaErrorNotReady) continue;
        CK(ctx, q);
        int rc = issue_d2h(ctx, s);
        if (rc != SKY_OK) return rc;
    }
    return SKY_OK;
}

// The synchronous calls run on slot 0 (its metadata, and its slabs for sky_decode): take_slot0 selects the device and
// the stream (the caller's, or the slot's when NULL) and refuses while the slot holds a ticket; finish_sync waits for
// the stream and reads kernel_ms (optional) from `start` (the slot's ev_k0 when NULL) to ev_k1.
static int take_slot0(sky_ctx *ctx, void *stream, cudaStream_t &st) {
    CK(ctx, cudaSetDevice(ctx->device));
    Slot &s = ctx->slots[0];
    if (s.ticket.busy) return SKY_E_BUSY;
    st = stream ? (cudaStream_t)stream : s.stream;
    return SKY_OK;
}
static int finish_sync(sky_ctx *ctx, cudaStream_t st, float *kernel_ms, cudaEvent_t start = nullptr) {
    const Slot &s = ctx->slots[0];
    CK(ctx, cudaStreamSynchronize(st));
    if (kernel_ms) CK(ctx, cudaEventElapsedTime(kernel_ms, start ? start : (cudaEvent_t)s.ev_k0, s.ev_k1));
    return SKY_OK;
}
// Device chunk base + off is 16-byte aligned (base and off both are): the kernels move 16 bytes at a time.
static bool aligned16(const void *base, uint64_t off) { return ((reinterpret_cast<uintptr_t>(base) | off) & 15) == 0; }

int sky_process_device(sky_ctx *ctx, uint32_t n, const void *d_src, const uint64_t *src_off, const uint64_t *src_len,
                       void *d_dst, const uint64_t *dst_off, const uint64_t *dst_cap, uint32_t flags, void *stream,
                       uint64_t *out_len, uint8_t *md5, float *kernel_ms) {
    if (!ctx || n == 0 || !src_off || !src_len || !dst_off || !dst_cap || !d_dst) return SKY_E_INVALID;
    if (flags & (SKY_F_E2EE | SKY_F_VERIFY | SKY_F_PASSTHROUGH)) return SKY_E_INVALID;  // host-path features (sky_submit; sky_verify_device checks)
    if (!frame_flags_valid(flags)) return SKY_E_INVALID;
    if (n > ctx->max_chunks) return SKY_E_CAPACITY;
    for (uint32_t i = 0; i < n; i++) {
        if (!aligned16(d_src, src_off[i]) || !aligned16(d_dst, dst_off[i])) return SKY_E_INVALID;
        if (dst_cap[i] < frame_need(src_len[i], flags)) return SKY_E_CAPACITY;
        if (src_len[i] && !d_src) return SKY_E_INVALID;
    }
    cudaStream_t st;
    int rc = take_slot0(ctx, stream, st);
    if (rc != SKY_OK) return rc;
    Slot &s = ctx->slots[0];
    rc = launch_batch(ctx, s, st, st, n, (const uint8_t *)d_src, src_off, src_len, (uint8_t *)d_dst, dst_off, with_stages(flags));
    if (rc == SKY_OK) rc = finish_sync(ctx, st, kernel_ms);
    if (rc != SKY_OK) return rc;
    if (out_len) memcpy(out_len, s.meta.outlen.h, n * sizeof(uint64_t));
    if (md5) memcpy(md5, s.meta.md5.h, (size_t)n * 16);
    return SKY_OK;
}

int sky_submit(sky_ctx *ctx, uint32_t n, const void *const *src, const uint64_t *src_len, void *const *dst,
               const uint64_t *dst_cap, uint32_t flags, const uint8_t *nonces, uint64_t *ticket) {
    if (!ctx || n == 0 || !src || !src_len || !ticket || !frame_flags_valid(flags)) return SKY_E_INVALID;
    flags = with_stages(flags);
    const bool e2ee = (flags & SKY_F_E2EE) != 0, frames = (flags & SKY_F_LZ4) != 0;
    const bool returns_data = frames || e2ee;  // MD5-only without E2EE: only digests come back
    if (returns_data && (!dst || !dst_cap)) return SKY_E_INVALID;
    if (e2ee && (!ctx->d_key || !nonces)) return SKY_E_NOKEY;
    if (n > ctx->max_chunks) return SKY_E_CAPACITY;
    Slot *sp = nullptr;
    for (Slot &s : ctx->slots)
        if (!s.ticket.busy && s.d_in) { sp = &s; break; }
    if (!sp) return ctx->slots[0].d_in ? SKY_E_BUSY : SKY_E_INVALID;
    Slot &s = *sp;
    CK(ctx, cudaSetDevice(ctx->device));
    { int prc = progress(ctx); if (prc != SKY_OK) return prc; }
    std::vector<uint64_t> in_off(n), out_off(n);
    uint64_t ip = 0, op = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (src_len[i] && !src[i]) return SKY_E_INVALID;
        if (returns_data) {
            const uint64_t need = (frames ? frame_need(src_len[i], flags) : src_len[i]) + (e2ee ? kBoxOverhead : 0);
            if (!dst[i] || dst_cap[i] < need) return SKY_E_CAPACITY;
        }
        in_off[i] = ip;
        out_off[i] = op;
        ip += round16(src_len[i]);
        op += round16(frame_need(src_len[i], flags));
    }
    if (ip > ctx->in_cap || op > ctx->out_cap) return SKY_E_CAPACITY;
    for (uint32_t i = 0; i < n; i++)
        if (src_len[i]) CK(ctx, cudaMemcpyAsync(s.d_in + in_off[i], src[i], src_len[i], cudaMemcpyHostToDevice, ctx->st_h2d));
    if (e2ee) {
        memcpy(s.box.h_nonce, nonces, 24ull * n);
        CK(ctx, cudaMemcpyAsync(s.box.d_nonce, s.box.h_nonce, 24ull * n, cudaMemcpyHostToDevice, ctx->st_h2d));
    }
    int rc = launch_batch(ctx, s, s.stream, ctx->st_h2d, n, s.d_in, in_off.data(), src_len, s.d_out, out_off.data(), flags);
    if (rc != SKY_OK) return rc;
    s.ticket = Ticket{true, false, ctx->next_ticket++, n, flags,
                      returns_data ? std::vector<void *>(dst, dst + n) : std::vector<void *>(n), std::move(out_off)};
    *ticket = s.ticket.id;
    return SKY_OK;
}

int sky_wait(sky_ctx *ctx, uint64_t ticket, uint64_t *out_len, uint8_t *md5, int32_t *verify, uint8_t *compressed, float *kernel_ms) {
    if (!ctx) return SKY_E_INVALID;
    Slot *sp = nullptr;
    for (Slot &s : ctx->slots)
        if (s.ticket.busy && s.ticket.id == ticket) { sp = &s; break; }
    if (!sp) return SKY_E_TICKET;
    Slot &s = *sp;
    if (verify && !(s.ticket.flags & SKY_F_VERIFY)) return SKY_E_INVALID;  // (the ticket stays valid)
    if (!compressed && (s.ticket.flags & SKY_F_PASSTHROUGH)) return SKY_E_INVALID;  // (likewise)
    CK(ctx, cudaSetDevice(ctx->device));
    { int prc = progress(ctx); if (prc != SKY_OK) return prc; }
    if (!s.ticket.d2h_issued) {
        CK(ctx, cudaEventSynchronize(s.ev_res));  // sizes + digests are on the host now
        int rc = issue_d2h(ctx, s);
        if (rc != SKY_OK) return rc;
    }
    { int prc = progress(ctx); if (prc != SKY_OK) return prc; }  // let later batches' copies queue up behind ours
    CK(ctx, cudaEventSynchronize(s.ev_d2h));
    if (out_len) memcpy(out_len, s.meta.outlen.h, s.ticket.n * sizeof(uint64_t));
    if (md5) memcpy(md5, s.meta.md5.h, (size_t)s.ticket.n * 16);
    if (verify) memcpy(verify, s.verify.status.h, s.ticket.n * sizeof(int32_t));
    if (compressed) {
        if (s.ticket.flags & SKY_F_PASSTHROUGH)
            for (uint32_t i = 0; i < s.ticket.n; i++) compressed[i] = s.meta.pass.h[i] ? 0 : 1;
        else
            memset(compressed, (s.ticket.flags & SKY_F_LZ4) ? 1 : 0, s.ticket.n);
    }
    if (kernel_ms) CK(ctx, cudaEventElapsedTime(kernel_ms, s.ev_k0, s.ev_k1));
    s.ticket.busy = false;
    return SKY_OK;
}

int sky_verify_device(sky_ctx *ctx, uint32_t n, const void *d_src, const uint64_t *src_off, const uint64_t *src_len, void *d_frames,
                      const uint64_t *frame_off, uint64_t *frame_len, const uint64_t *frame_cap, const uint32_t *content_xxh,
                      uint32_t flags, void *stream, int32_t *status, float *kernel_ms) {
    if (!ctx || n == 0 || !src_off || !src_len || !d_frames || !frame_off || !frame_len) return SKY_E_INVALID;
    if ((flags & (SKY_F_E2EE | SKY_F_PASSTHROUGH)) || !frame_flags_valid(flags) || (flags & (SKY_F_LZ4 | SKY_F_MD5)) == SKY_F_MD5)
        return SKY_E_INVALID;
    if (((flags & SKY_F_CHECKSUM) != 0) != (content_xxh != nullptr)) return SKY_E_INVALID;
    if (n > ctx->max_chunks) return SKY_E_CAPACITY;
    for (uint32_t i = 0; i < n; i++) {
        if (!aligned16(d_src, src_off[i])) return SKY_E_INVALID;
        if (src_len[i] && !d_src) return SKY_E_INVALID;
        if (frame_cap && frame_cap[i] < frame_need(src_len[i], flags)) return SKY_E_CAPACITY;
    }
    cudaStream_t st;
    int rc = take_slot0(ctx, stream, st);
    if (rc != SKY_OK) return rc;
    Slot &s = ctx->slots[0];
    BatchMeta &m = s.meta;
    uint32_t rows;
    rc = batch_geometry(n, src_len, rows, [&](uint32_t i, uint32_t nblk) {
        m.h_desc[i] = ChunkDesc{(const uint8_t *)d_src + src_off[i], (uint8_t *)d_frames + frame_off[i], src_len[i], nblk};
    });
    if (rc != SKY_OK) return rc;
    CK(ctx, cudaStreamSynchronize(st));  // (slot 0's metadata is free: nothing earlier on this stream still reads it)
    memcpy(m.outlen.h, frame_len, n * sizeof(uint64_t));
    CK(ctx, cudaMemcpyAsync(m.d_desc, m.h_desc, n * sizeof(ChunkDesc), cudaMemcpyHostToDevice, st));
    if (content_xxh) CK(ctx, cudaMemcpyAsync(m.xxh, content_xxh, n * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaEventRecord(s.ev_k0, st));
    rc = launch_verify(ctx, s, st, n, rows, flags, frame_cap != nullptr);
    if (rc != SKY_OK) return rc;
    CK(ctx, cudaEventRecord(s.ev_k1, st));
    rc = finish_sync(ctx, st, kernel_ms);
    if (rc != SKY_OK) return rc;
    if (status) memcpy(status, s.verify.status.h, n * sizeof(int32_t));
    memcpy(frame_len, m.outlen.h, n * sizeof(uint64_t));
    return SKY_OK;
}

int sky_device_alloc(sky_ctx *ctx, uint64_t bytes, void **dptr) {
    if (!ctx || !dptr) return SKY_E_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    cudaError_t e = cudaMalloc(dptr, bytes ? bytes : 16);
    if (e != cudaSuccess) { ctx->err = cudaGetErrorString(e); return SKY_E_NOMEM; }
    return SKY_OK;
}
int sky_device_free(sky_ctx *ctx, void *dptr) {
    if (!ctx) return SKY_E_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaFree(dptr));
    return SKY_OK;
}
int sky_memcpy_h2d(sky_ctx *ctx, void *dptr, const void *host, uint64_t bytes) {
    if (!ctx) return SKY_E_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaMemcpy(dptr, host, bytes, cudaMemcpyHostToDevice));
    return SKY_OK;
}
int sky_memcpy_d2h(sky_ctx *ctx, void *host, const void *dptr, uint64_t bytes) {
    if (!ctx) return SKY_E_INVALID;
    CK(ctx, cudaSetDevice(ctx->device));
    CK(ctx, cudaMemcpy(host, dptr, bytes, cudaMemcpyDeviceToHost));
    return SKY_OK;
}


// ---------------------------------------------------------------------------------- receiver side
// Enqueues index + decode (+ MD5 of the decoded bytes through the fused kernel's MD5 role) on `st`.
static int launch_decode(sky_ctx *ctx, Slot &s, cudaStream_t st, uint32_t n, const uint8_t *d_frames, const uint64_t *frame_off,
                         const uint64_t *frame_len, uint8_t *d_out, const uint64_t *out_off, const uint64_t *raw_len) {
    int rc = alloc_dec(ctx, s.dec);
    if (rc != SKY_OK) return rc;
    DecodeArrays &d = s.dec;
    uint64_t nblk_total = 0;
    uint32_t rows;
    rc = batch_geometry(n, raw_len, rows, [&](uint32_t i, uint32_t nblk) {
        d.h_chunks[i] = DecChunk{d_frames + frame_off[i], d_out + out_off[i], frame_len[i], raw_len[i], nblk_total, nblk, 0};
        nblk_total += nblk;
    });
    if (rc == SKY_OK) rc = grow_block_table(ctx, st, d.table, nblk_total + 1);
    if (rc != SKY_OK) return rc;
    BatchMeta &m = s.meta;
    CK(ctx, cudaMemcpyAsync(d.d_chunks, d.h_chunks, n * sizeof(DecChunk), cudaMemcpyHostToDevice, st));
    CK(ctx, cudaMemsetAsync(m.counters, 0, 64, st));
    CK(ctx, cudaMemsetAsync(d.d_dec_done, 0, n * sizeof(uint32_t), st));
    CK(ctx, cudaMemsetAsync(d.d_status, 0, n * sizeof(int32_t), st));
    CK(ctx, cudaMemsetAsync(d.table.done, 0, (nblk_total + 1) * sizeof(uint32_t), st));
    const uint32_t ng = fill_md5_order(m.h_order, n, raw_len);
    CK(ctx, cudaMemcpyAsync(m.d_order, m.h_order, ng * 32 * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    memset(m.md5.h, 0, (size_t)n * 16);
    DecParams p;
    p.chunks = d.d_chunks;
    p.blocks = d.table.blocks;
    p.status = d.d_status;
    p.dec_done = d.d_dec_done;
    p.counter = m.counters;
    p.blk_done = d.table.done;
    p.md5_order = m.d_order;
    p.md5_out = m.md5.d;
    p.n_chunks = n;
    p.n_groups = ng;
    p.rows = rows;
    CK(ctx, cudaEventRecord(s.ev_k0, st));
    sky_frame_index_kernel<<<(n + 127) / 128, 128, 0, st>>>(p);
    CK(ctx, cudaGetLastError());
    sky_decode_kernel<<<ctx->sm_count, 512, kMd5WarpsPerCta * kDecRingBytes, st>>>(p);
    CK(ctx, cudaGetLastError());
    CK(ctx, cudaEventRecord(s.ev_k1, st));
    ctx->launches += 2;
    CK(ctx, cudaMemcpyAsync(d.h_status, d.d_status, n * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    return SKY_OK;
}

int sky_decode_device(sky_ctx *ctx, uint32_t n, const void *d_frames, const uint64_t *frame_off, const uint64_t *frame_len,
                      void *d_out, const uint64_t *out_off, const uint64_t *raw_len, void *stream, int32_t *status, uint8_t *md5,
                      float *kernel_ms) {
    if (!ctx || n == 0 || !d_frames || !frame_off || !frame_len || !out_off || !raw_len) return SKY_E_INVALID;
    if (n > ctx->max_chunks) return SKY_E_CAPACITY;
    for (uint32_t i = 0; i < n; i++) {
        if (!aligned16(d_out, out_off[i])) return SKY_E_INVALID;
        if (raw_len[i] && !d_out) return SKY_E_INVALID;
    }
    cudaStream_t st;
    int rc = take_slot0(ctx, stream, st);
    if (rc != SKY_OK) return rc;
    Slot &s = ctx->slots[0];
    rc = launch_decode(ctx, s, st, n, (const uint8_t *)d_frames, frame_off, frame_len, (uint8_t *)d_out, out_off, raw_len);
    if (rc == SKY_OK) rc = finish_sync(ctx, st, kernel_ms);  // index + decode + MD5
    if (rc != SKY_OK) return rc;
    if (status) memcpy(status, s.dec.h_status, n * sizeof(int32_t));
    if (md5) memcpy(md5, s.meta.md5.h, (size_t)n * 16);
    return SKY_OK;
}

// sky_decode of payloads that are the chunks themselves (SKY_F_MD5 alone: the sender's `compress: false`), sealed or not.
// The chunk bytes go into the slot's INPUT slab -- copied there, or opened there from their boxes -- and are digested by
// the launch sky_submit(SKY_F_MD5) makes.  A chunk of the wrong size is left out of that launch (length 0), and the digest of a
// chunk that fails is reported as 16 zero bytes.  Only opened chunks are copied back: an unsealed one the caller already holds.
static int decode_raw(sky_ctx *ctx, Slot &s, uint32_t n, const void *const *payload, const uint64_t *payload_len, void *const *dst,
                      const uint64_t *raw_len, bool e2ee, int32_t *status, uint8_t *md5, float *kernel_ms) {
    std::vector<uint64_t> off(n), box_off(n), msg_len(payload_len, payload_len + n), md5_len(n);
    uint64_t ip = 0, bp = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (payload_len[i] && !payload[i]) return SKY_E_INVALID;
        if (e2ee && raw_len[i] && !dst[i]) return SKY_E_INVALID;
        if (e2ee) msg_len[i] = payload_len[i] >= (uint64_t)kBoxOverhead ? payload_len[i] - kBoxOverhead : 0;
        md5_len[i] = msg_len[i] == raw_len[i] ? raw_len[i] : 0;
        off[i] = ip;
        box_off[i] = bp;
        ip += round16(e2ee ? msg_len[i] : md5_len[i]);  // (an opened chunk lands whole, whatever size was expected)
        bp += round16(payload_len[i]);
    }
    if (ip > ctx->in_cap || (e2ee && bp > ctx->out_cap)) return SKY_E_CAPACITY;
    if (e2ee) {
        const int rc = launch_open(ctx, s, n, payload, payload_len, box_off.data(), s.d_in, off.data(), msg_len.data());
        if (rc != SKY_OK) return rc;
    } else {
        for (uint32_t i = 0; i < n; i++)
            if (md5_len[i]) CK(ctx, cudaMemcpyAsync(s.d_in + off[i], payload[i], md5_len[i], cudaMemcpyHostToDevice, s.stream));
    }
    // (no frames are written without SKY_F_LZ4: the frame slab only lends the descriptors an address)
    int rc = launch_batch(ctx, s, s.stream, s.stream, n, s.d_in, off.data(), md5_len.data(), s.d_out, off.data(), SKY_F_MD5);
    if (rc == SKY_OK) rc = finish_sync(ctx, s.stream, kernel_ms, e2ee ? (cudaEvent_t)s.box.ev_open : nullptr);  // open + digest
    if (rc != SKY_OK) return rc;
    for (uint32_t i = 0; i < n; i++) {
        int32_t st = msg_len[i] == raw_len[i] ? SKY_D_OK : SKY_D_SIZE;
        if (e2ee && (s.box.h_status[i] != 0 || payload_len[i] < (uint64_t)kBoxOverhead)) st = SKY_D_AUTH;  // never hand its bytes out
        if (status) status[i] = st;
        if (md5) {
            if (st == SKY_D_OK) memcpy(md5 + 16ull * i, s.meta.md5.h + 16ull * i, 16);
            else memset(md5 + 16ull * i, 0, 16);
        }
        if (e2ee && st == SKY_D_OK && raw_len[i])
            CK(ctx, cudaMemcpyAsync(dst[i], s.d_in + off[i], raw_len[i], cudaMemcpyDeviceToHost, s.stream));
    }
    if (e2ee) CK(ctx, cudaStreamSynchronize(s.stream));
    return SKY_OK;
}

int sky_decode(sky_ctx *ctx, uint32_t n, const void *const *frames, const uint64_t *frame_len, void *const *dst,
               const uint64_t *raw_len, uint32_t flags, int32_t *status, uint8_t *md5, float *kernel_ms) {
    if (flags & ~(SKY_F_LZ4 | SKY_F_MD5 | SKY_F_E2EE)) return SKY_E_INVALID;  // a receiver takes what it is sent: no frame options
    const bool e2ee = (flags & SKY_F_E2EE) != 0, raw = (flags & (SKY_F_LZ4 | SKY_F_MD5)) == SKY_F_MD5;
    const bool returns_data = !raw || e2ee;  // an unsealed raw chunk is only digested: the caller holds its bytes
    if (!ctx || n == 0 || !frames || !frame_len || (returns_data && !dst) || !raw_len) return SKY_E_INVALID;
    if (n > ctx->max_chunks) return SKY_E_CAPACITY;
    cudaStream_t st;
    int rc = take_slot0(ctx, nullptr, st);
    if (rc != SKY_OK) return rc;
    Slot &s = ctx->slots[0];
    if (!s.d_in) return SKY_E_INVALID;  // ctx created without slabs
    if (e2ee && !ctx->d_key) return SKY_E_NOKEY;
    if (raw) return decode_raw(ctx, s, n, frames, frame_len, dst, raw_len, e2ee, status, md5, kernel_ms);
    // roles swap on the way back: frames (<= bound) go into the frame slab, decoded bytes into the input slab
    std::vector<uint64_t> f_off(n), o_off(n), f_len(frame_len, frame_len + n);
    uint64_t fp = 0, op = 0;
    for (uint32_t i = 0; i < n; i++) {
        if (!frames[i] || (raw_len[i] && !dst[i])) return SKY_E_INVALID;
        f_off[i] = fp;
        o_off[i] = op;
        fp += round16(frame_len[i]);
        op += round16(raw_len[i]);
    }
    if (fp > ctx->out_cap || op > ctx->in_cap) return SKY_E_CAPACITY;
    if (e2ee) {
        // the payloads are boxes (nonce | tag | ciphertext): check the tags, decrypt into the frame slab, then decode as usual
        rc = launch_open(ctx, s, n, frames, frame_len, f_off.data(), s.d_out, f_off.data(), f_len.data());
        if (rc != SKY_OK) return rc;
    } else {
        for (uint32_t i = 0; i < n; i++)
            CK(ctx, cudaMemcpyAsync(s.d_out + f_off[i], frames[i], frame_len[i], cudaMemcpyHostToDevice, st));
    }
    rc = launch_decode(ctx, s, st, n, s.d_out, f_off.data(), f_len.data(), s.d_in, o_off.data(), raw_len);
    if (rc == SKY_OK) rc = finish_sync(ctx, st, kernel_ms);  // index + decode + MD5, without the box open
    if (rc != SKY_OK) return rc;
    for (uint32_t i = 0; i < n; i++) {
        if (e2ee && (s.box.h_status[i] != 0 || frame_len[i] < (uint64_t)kBoxOverhead))  // forged or truncated box: never hand its bytes out
            s.dec.h_status[i] = SKY_D_AUTH;
        if (raw_len[i] && s.dec.h_status[i] == 0)
            CK(ctx, cudaMemcpyAsync(dst[i], s.d_in + o_off[i], raw_len[i], cudaMemcpyDeviceToHost, st));
    }
    if (status) memcpy(status, s.dec.h_status, n * sizeof(int32_t));
    if (md5) memcpy(md5, s.meta.md5.h, (size_t)n * 16);
    CK(ctx, cudaStreamSynchronize(st));
    return SKY_OK;
}

uint64_t sky_launch_count(const sky_ctx *ctx) { return ctx ? ctx->launches : 0; }

#ifdef SKY_MD5_TRACE
// Diagnostic build only, not part of the ABI: copies the trace records of the last fused launches on `device` to the host
// (sizes in bytes, as tools/md5_trace.py lays them out) and clears them.
SKY_API int sky_md5_trace_fetch(int device, void *md5, uint64_t md5_bytes, void *ctas, uint64_t cta_bytes) {
    if (md5_bytes != sizeof(sky::g_md5_trace) || cta_bytes != sizeof(sky::g_cta_trace)) return SKY_E_INVALID;
    if (cudaSetDevice(device) != cudaSuccess || cudaDeviceSynchronize() != cudaSuccess ||
        cudaMemcpyFromSymbol(md5, sky::g_md5_trace, md5_bytes) != cudaSuccess ||
        cudaMemcpyFromSymbol(ctas, sky::g_cta_trace, cta_bytes) != cudaSuccess)
        return SKY_E_CUDA;
    static const char zero[sizeof(sky::g_md5_trace)] = {};
    static_assert(sizeof(sky::g_md5_trace) >= sizeof(sky::g_cta_trace), "one zero buffer clears both");
    if (cudaMemcpyToSymbol(sky::g_md5_trace, zero, md5_bytes) != cudaSuccess ||
        cudaMemcpyToSymbol(sky::g_cta_trace, zero, cta_bytes) != cudaSuccess)
        return SKY_E_CUDA;
    return SKY_OK;
}
#endif

}  // extern "C"

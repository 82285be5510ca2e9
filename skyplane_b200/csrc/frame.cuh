// frame.cuh -- the sender's batch and frame contract, shared by both block compressors (sky_fused_kernel in skychunk.cu,
// sky_hc_kernel in lz4hc.cuh) and the frame check's repair: the batch descriptors, the final frame header (the one place
// that maps the batch's flags to FLG bits), the block claim, the block load into shared memory, the block's placement in
// its frame through the OFF chain, the per-warp write-out, and the block and content checksums.
//
// OFF chain (one word per chunk): OFF = (next block index << 40) | frame offset of that block, a prefix sum handed from
// block j-1 to block j as soon as j-1 knows its compressed size -- before it has written a byte, so offsets race down the
// chain.  The host starts every chunk's word at (0 << 40) | kFrameHeaderBytes.  Waiting is deadlock-free: a CTA only waits
// on lower-numbered work items, all of which were claimed earlier by running CTAs.
#pragma once
#include "../../include/skychunk.h"
#include "lz4.cuh"
#include "xxh32.cuh"

namespace sky {

constexpr uint32_t kFrameHeaderBytes = 15;  // frame header with content size: magic, FLG, BD, 8-byte content size, header checksum

// Frame header bytes of an n-byte chunk: the content size is omitted for an empty chunk (0 means "unknown" to LZ4F).
__device__ __forceinline__ uint32_t frame_header_bytes(uint64_t n) { return n ? kFrameHeaderBytes : 7u; }

// The FLG bits a batch's flags set: C.Checksum (0x04) with SKY_F_CHECKSUM, B.Checksum (0x10) with SKY_F_BLOCK_CHECKSUM.
__device__ __forceinline__ uint32_t frame_flg(uint32_t flags) {
    return ((flags & SKY_F_CHECKSUM) ? 0x04u : 0u) | ((flags & SKY_F_BLOCK_CHECKSUM) ? 0x10u : 0u);
}
// FLG's B.Indep (0x20) for an n-byte chunk: set, unless SKY_F_LINKED links the blocks of a chunk of more than one block
// (liblz4 declares a frame of at most one block independent whatever blockMode asks for).  kLinkable: the caller may see
// SKY_F_LINKED (the linked compressor and frame check); every other caller writes independent frames only.
template <bool kLinkable>
__device__ __forceinline__ uint32_t frame_indep(uint32_t flags, uint64_t n) {
    return (kLinkable && (flags & SKY_F_LINKED) && n > kBlock) ? 0u : 0x20u;
}

__device__ __forceinline__ void st_u32le(uint8_t *p, uint32_t v) {
    p[0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[2] = (uint8_t)(v >> 16); p[3] = (uint8_t)(v >> 24);
}

// Single thread: writes the final frame header of an n-byte chunk made with the batch's `flags`; returns its size.
template <bool kLinkable = false>
__device__ __forceinline__ uint32_t write_frame_header(uint8_t *dst, uint64_t n, uint32_t flags) {
    uint8_t d[10];
    d[1] = 0x40;  // BD: 64 KiB blocks
    st_u32le(dst, 0x184D2204u);  // magic
    if (n == 0) {
        d[0] = (uint8_t)(0x40u | frame_indep<kLinkable>(flags, n) | frame_flg(flags));  // v01 | B.Indep
        dst[4] = d[0]; dst[5] = d[1];
        dst[6] = (uint8_t)(xxh32_small(d, 2) >> 8);
        return 7;
    }
    d[0] = (uint8_t)(0x48u | frame_indep<kLinkable>(flags, n) | frame_flg(flags));  // v01 | B.Indep | C.Size
#pragma unroll
    for (int i = 0; i < 8; i++) d[2 + i] = (uint8_t)(n >> (8 * i));
#pragma unroll
    for (int i = 0; i < 10; i++) dst[4 + i] = d[i];
    dst[kFrameHeaderBytes - 1] = (uint8_t)(xxh32_small(d, 10) >> 8);
    return kFrameHeaderBytes;
}

constexpr uint32_t kInBytes = kBlock + 128;  // a block buffer in shared memory, + slack: unaligned 4-byte reads may touch the word after the last byte
constexpr uint32_t kLoadPiece = 8192;        // bytes per bulk copy of the block load
constexpr int kOffBits = 40;
constexpr uint64_t kOffMask = (1ull << kOffBits) - 1;

struct ChunkDesc {
    const uint8_t *src;  // 16-byte aligned
    uint8_t *dst;        // 16-byte aligned
    uint64_t len;
    uint32_t nblk;
};

struct Params {
    const ChunkDesc *chunks;
    const uint32_t *md5_order;  // chunk indices, longest first, padded with 0xffffffff to 32*n_groups
    uint64_t *chain;            // per chunk OFF word: (next block index << 40) | frame offset of that block
    uint64_t *out_len;          // per chunk frame length
    uint8_t *md5_out;           // 16 bytes per chunk
    uint32_t *counters;         // [0] = LZ4 work counter
    uint8_t *scratch;           // per CTA: where a block is compressed before its frame offset is known
    uint32_t n_chunks;
    uint32_t n_groups;
    uint32_t n_md5_ctas;        // CTAs 0..n_md5_ctas-1 digest (4 groups each at a time) before they compress
    uint32_t rows;  // max(1, max nblk)
    uint32_t flags;
    uint32_t *xxh_out;          // per chunk XXH32 of the input (sky_fused_xxh_kernel only)
};

struct BlockDesc {            // written by the claiming thread, read by every warp after the block-start barrier
    const uint8_t *src;       // block start in the chunk (16-byte aligned)
    uint8_t *dst;             // chunk's frame region
    uint32_t c, j, L, last;   // chunk, block index, block length, 1 = last block of the chunk
    uint32_t valid, pad;
};

__device__ __forceinline__ uint64_t ld_acquire(const uint64_t *p) {
    uint64_t v;
    asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_acquire32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint32_t ld_relaxed32(const uint32_t *p) {
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release(uint64_t *p, uint64_t v) {
    asm volatile("st.release.gpu.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_release32(uint32_t *p, uint32_t v) {
    asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// One thread: claim the next block that has LZ4 work (empty chunks are finished on the spot) and describe it to the CTA.
// Block 0's claim writes the frame header (kLinkable: write_frame_header's).
template <bool kLinkable = false>
__device__ __forceinline__ void claim_block(const Params &p, BlockDesc *d) {
    const uint32_t total = p.rows * p.n_chunks;
    // read per claim: hoisted out of the kernel's block loop, the FLG bits would hold a register there (sky_fused_kernel spills)
    uint32_t flags = p.flags;
    asm volatile("" : "+r"(flags));
    for (;;) {
        const uint32_t w = atomicAdd(p.counters, 1u);
        if (w >= total) {
            d->valid = 0;
            return;
        }
        const uint32_t c = w % p.n_chunks, j = w / p.n_chunks;  // row-major: block row j of every chunk, then row j+1
        const ChunkDesc cd = p.chunks[c];
        if (cd.nblk == 0) {
            if (j == 0) {  // empty chunk: 7-byte header + EndMark
                const uint32_t h = write_frame_header<kLinkable>(cd.dst, 0, flags);
                st_u32le(cd.dst + h, 0);
                p.out_len[c] = h + 4;
            }
            continue;
        }
        if (j >= cd.nblk) continue;
        const uint64_t boff = (uint64_t)j * kBlock;
        d->src = cd.src + boff;
        d->dst = cd.dst;
        d->c = c;
        d->j = j;
        d->L = (uint32_t)min((uint64_t)kBlock, cd.len - boff);
        d->last = (j + 1 == cd.nblk);
        d->valid = 1;
        if (j == 0) write_frame_header<kLinkable>(cd.dst, cd.len, flags);
        return;
    }
}

// One thread: bring the block's L bytes from src into the shared-memory buffer `in` (kInBytes); completes on `bar`.
__device__ __forceinline__ void load_block(uint8_t *in, const uint8_t *src, uint32_t L, uint64_t *bar) {
    const uint32_t bytes = (L + 15u) & ~15u;  // (the input slab is readable up to the next multiple of 16)
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic reads of the old block before the async write
    mbar_arrive_expect_tx(bar, bytes);
    for (uint32_t o = 0; o < bytes; o += kLoadPiece)  // several copies in flight: the pieces stream in parallel
        bulk_load(in + o, src + o, min(kLoadPiece, bytes - o), bar);
}

struct BlockPlace {
    uint64_t data;  // frame offset of the block's first data byte
    bool raw;       // stored: the block's L input bytes go to `data`, not its csize compressed ones
};
// One thread, once the block's compressed size is known: wait for the block's frame offset on the OFF chain, hand block
// j+1 its offset at once, write the block header and, on the chunk's last block, the EndMark and the frame length.
// kBlkChk (SKY_F_BLOCK_CHECKSUM): 4 more bytes follow the block's data for its checksum (block_checksum writes them), so
// the next offset is known before any hashing.
template <bool kBlkChk = false>
__device__ __forceinline__ BlockPlace place_block(const Params &p, const BlockDesc &d, uint32_t csize, uint32_t L) {
    const bool raw = csize > L - 1;  // LZ4F_makeBlock: a block that does not shrink is stored
    uint64_t *cw = p.chain + d.c;
    uint64_t st;
    unsigned ns = 128;
    while (((st = ld_acquire(cw)) >> kOffBits) != d.j) {
        __nanosleep(ns);
        if (ns < 2048) ns <<= 1;
    }
    const uint64_t off = st & kOffMask;
    const uint64_t end = off + 4 + (raw ? L : csize) + (kBlkChk ? 4 : 0);
    if (!d.last) st_release(cw, ((uint64_t)(d.j + 1) << kOffBits) | end);
    st_u32le(d.dst + off, raw ? (L | 0x80000000u) : csize);
    if (d.last) {
        st_u32le(d.dst + end, 0);  // EndMark
        p.out_len[d.c] = end + 4;
    }
    return BlockPlace{off + 4, raw};
}

// Every warp of the CTA: copy n bytes from src (16-byte aligned) to out, one 16-byte-aligned slice per warp.
// kReadOnly: src is the kernel's read-only input, else scratch this CTA wrote (see warp_copy_stream).
template <int kNumWarps, bool kReadOnly>
__device__ __forceinline__ void copy_block(uint8_t *out, const uint8_t *src, uint32_t n, unsigned warp, unsigned lane) {
    const uint32_t per = (((n + kNumWarps - 1) / kNumWarps) + 15u) & ~15u;
    const uint32_t lo = warp * per;
    if (lo < n) warp_copy_stream<kReadOnly>(out + lo, src + lo, min(per, n - lo), lane);
}

// SKY_F_BLOCK_CHECKSUM, one warp: the block checksum -- XXH32 (seed 0) of the block's n data bytes as stored in the frame:
// the compressed bytes, or the raw bytes of a stored block -- read from `src` and written as u32le at `at`, right behind
// the data.  place_block<true> has passed the next offset on before any of this, so the hash is never on the OFF chain.
__device__ __forceinline__ void block_checksum(const uint8_t *src, uint32_t n, uint8_t *at, unsigned lane) {
    const uint32_t x = xxh32_warp(src, n, lane);
    if (lane == 0) st_u32le(at, x);
}
// A block whose checksum is hashed later from its bytes in the frame, by one warp of the CTA that wrote them, after a CTA
// barrier has ordered those writes before its reads: the warp runs it where it would otherwise wait, off the CTA's next
// block (sky_fused_kernel and sky_hc_kernel say where).  It lives in shared memory (a register copy would stay live across
// the whole block loop), and only the hashing warp reads or writes it once the kernel has cleared it.
struct PendingChecksum {
    uint8_t *data;  // the block's first data byte in the frame; null: nothing pending
    uint32_t n;
};
// The hashing warp: hash the pending block, if there is one, and clear it.
__device__ __forceinline__ void run_pending(PendingChecksum *pc, unsigned lane) {
    uint8_t *const d = pc->data;
    const uint32_t n = pc->n;
    if (!d) return;
    __syncwarp();  // every lane has read it
    if (lane == 0) pc->data = nullptr;
    block_checksum(d, n, d + n, lane);
}
__device__ __forceinline__ void set_pending(PendingChecksum *pc, uint8_t *data, uint32_t n, unsigned lane) {
    __syncwarp();
    if (lane == 0) {
        pc->data = data;
        pc->n = n;
    }
}

// SKY_F_CHECKSUM, one thread, on a finished frame of *len bytes (its header already carries C.Checksum): the content
// checksum `xxh`, the XXH32 of the chunk, goes behind the EndMark and *len grows by 4.
__device__ __forceinline__ void finish_frame(uint8_t *frame, uint64_t *len, uint32_t xxh) {
    const uint64_t end = *len;
    st_u32le(frame + end, xxh);
    *len = end + 4;
}

}  // namespace sky

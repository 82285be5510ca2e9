// frame.cuh -- the sender's batch and frame contract, shared by both block compressors (sky_fused_kernel in skychunk.cu,
// sky_hc_kernel in lz4hc.cuh): the batch descriptors, the block claim, the block load into shared memory, the block's
// placement in its frame through the OFF chain, and the per-warp write-out.
//
// OFF chain (one word per chunk): OFF = (next block index << 40) | frame offset of that block, a prefix sum handed from
// block j-1 to block j as soon as j-1 knows its compressed size -- before it has written a byte, so offsets race down the
// chain.  The host starts every chunk's word at (0 << 40) | kFrameHeaderBytes.  Waiting is deadlock-free: a CTA only waits
// on lower-numbered work items, all of which were claimed earlier by running CTAs.
#pragma once
#include "lz4.cuh"
#include "xxh32.cuh"

namespace sky {

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
__device__ __forceinline__ void claim_block(const Params &p, BlockDesc *d) {
    const uint32_t total = p.rows * p.n_chunks;
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
                const uint32_t h = write_frame_header(cd.dst, 0);
                cd.dst[h] = cd.dst[h + 1] = cd.dst[h + 2] = cd.dst[h + 3] = 0;
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
        if (j == 0) write_frame_header(cd.dst, cd.len);
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
    uint8_t *hdr = d.dst + off;
    const uint32_t hword = raw ? (L | 0x80000000u) : csize;
    hdr[0] = (uint8_t)hword; hdr[1] = (uint8_t)(hword >> 8); hdr[2] = (uint8_t)(hword >> 16); hdr[3] = (uint8_t)(hword >> 24);
    if (d.last) {
        uint8_t *e = d.dst + end;
        e[0] = e[1] = e[2] = e[3] = 0;  // EndMark
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
    if (lane == 0) { at[0] = (uint8_t)x; at[1] = (uint8_t)(x >> 8); at[2] = (uint8_t)(x >> 16); at[3] = (uint8_t)(x >> 24); }
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

// Frame-descriptor epilogue of chunk c's finished frame, one thread: FLG gains `flg` (SKY_F_CHECKSUM: C.Checksum 0x04,
// SKY_F_BLOCK_CHECKSUM: B.Checksum 0x10; 0x68 -> 0x6C / 0x78 / 0x7C, 0x60 -> 0x64 / 0x70 / 0x74 for an empty chunk) and
// the header checksum byte follows.  With the content checksum (xxh != null) xxh[c], the XXH32 of the chunk, goes behind
// the EndMark at out_len[c], which grows by 4.
__device__ __forceinline__ void finish_frame(const ChunkDesc *chunks, const uint32_t *xxh, uint64_t *out_len, uint32_t c, uint32_t flg) {
    const ChunkDesc cd = chunks[c];
    uint8_t *f = cd.dst;
    const uint32_t dlen = cd.len ? 10u : 2u;  // FLG, BD (+ content size)
    f[4] |= (uint8_t)flg;
    uint8_t d[10];
    for (uint32_t i = 0; i < dlen; i++) d[i] = f[4 + i];
    f[4 + dlen] = (uint8_t)(xxh32_small(d, dlen) >> 8);
    if (!xxh) return;
    const uint64_t end = out_len[c];
    const uint32_t x = xxh[c];
    f[end] = (uint8_t)x; f[end + 1] = (uint8_t)(x >> 8); f[end + 2] = (uint8_t)(x >> 16); f[end + 3] = (uint8_t)(x >> 24);
    out_len[c] = end + 4;
}

}  // namespace sky

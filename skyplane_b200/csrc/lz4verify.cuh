// lz4verify.cuh -- the sender's frame check (SKY_F_VERIFY), sm_90a: does every finished frame restore its chunk under any
// LZ4 decoder?  Where one does not, the chunk's stored-block frame takes its place before anything is sealed or sent.
//
// Three launches on the batch's stream, after the frame epilogue (finish_frame) and before the seal:
//   sky_verify_index_kernel  : one thread per chunk.  FLG and BD must be exactly what write_frame_header (frame.cuh) writes
//                              for the chunk and the batch's flags, then frame_index (lz4dec.cuh) checks magic, content
//                              size and HC byte and walks the block words with nblk taken from the chunk's length; the
//                              EndMark must follow the last block, the frame must end right behind it (and its content
//                              checksum), and the content checksum must be the XXH32 the MD5 lanes computed from the chunk.
//   sky_verify_kernel        : one warp per 64 KiB block, claimed row-major (claim_row_major, lz4dec.cuh).  The block
//                              checksum over the block's stored bytes, then a stored block's bytes against the chunk, or a
//                              compare-decode of a compressed block against the chunk.
//   sky_verify_settle_kernel : one CTA per chunk.  The chunk's status (settle_status), and for a failing chunk with repair
//                              on, its frame rewritten in place as the stored-block frame through frame.cuh's writers.
// Compare-decode.  An independent block decodes to the source block iff every literal byte equals the source at its output
// position q and every match byte satisfies src[q] == src[q - off]: by induction over q, once every output byte before q
// equals the source, a match copies source bytes.  So no output buffer and no digest are needed, and every block checks
// on its own.  The walk also enforces what liblz4 enforces and the GPU receiver does not (DESIGN §9): off >= 1,
// q - off >= the block start, no overrun of the block or of the block's bytes, a decoded length of exactly
// min(64 KiB, n - block start), the last 5 bytes literals and the last match starting >= 12 bytes before the block end.
// Status 0 therefore means liblz4 decodes the frame to the chunk.
// Linked frames (SKY_F_LINKED, the sky_verify_linked_* kernels): a match may reach back across its block's start, up to
// the chunk's first byte (off <= block start + q; the 16-bit field caps it at 65535).  The induction still holds per block,
// since a chunk passes only when every block passes and the earliest failing block's code wins, so the blocks are checked
// in parallel; the end-of-block rules stay per block.  A failure is reported in the receiver's codes, plus
// kVerifyMismatch: well formed, but other bytes; within a chunk the earliest failing block's code wins (block_fail, the
// receiver's per-block status protocol in lz4dec.cuh).
#pragma once
#include <stdint.h>

#include "../../include/skychunk.h"
#include "frame.cuh"
#include "lz4dec.cuh"

namespace sky {

constexpr int32_t kVerifyMismatch = -9;  // SKY_D_MISMATCH
static_assert(kVerifyMismatch == SKY_D_MISMATCH, "include/skychunk.h");
constexpr int kVerifyThreads = 512;      // sky_verify_kernel: 16 warps per CTA, one block per warp at a time
constexpr int kRepairWarps = 8;          // sky_verify_settle_kernel: warps per chunk

struct VerifyParams {
    const ChunkDesc *chunks;   // src = the chunk (16-byte aligned), dst = its frame, len, nblk
    uint64_t *frame_len;       // per chunk: the frame's length; the stored-block frame's once repaired
    const uint32_t *xxh;       // per chunk XXH32 of the chunk (SKY_F_CHECKSUM), else null
    const uint64_t *blk_base;  // per chunk: its first entry in `blocks`
    DecBlock *blocks;          // the block table frame_index fills
    int32_t *status;           // per chunk: 0, a frame-level code, kDecChecksum (content), or block_fail(j, code)
    int32_t *status_out;       // per chunk, the settled code (mapped host memory)
    uint32_t *counter;         // work counter of sky_verify_kernel
    uint32_t n_chunks;
    uint32_t rows;             // max(1, max nblk)
    uint32_t flags;            // the batch's SKY_F_* (checksum bits)
    uint32_t repair;           // 1: rewrite failing frames
};

// One thread per chunk: the frame-level checks.  -> kDecOk, kDecChecksum (content checksum: the blocks are still checked,
// and a block failure takes precedence) or a frame-level code (the blocks are not checked).  kLinked: the batch's flags
// may hold SKY_F_LINKED.
template <bool kLinked>
__device__ __forceinline__ int32_t verify_frame(const VerifyParams &p, uint32_t c) {
    const ChunkDesc cd = p.chunks[c];
    DecChunk d{cd.dst, nullptr, p.frame_len[c], cd.len, p.blk_base[c], cd.nblk, 0, 0, 0};
    const uint8_t *f = cd.dst;
    uint8_t want[kFrameHeaderBytes];  // the header the stage writes for this chunk
    write_frame_header<kLinked>(want, cd.len, p.flags);
    if (d.frame_len >= 11 && (f[4] != want[4] || f[5] != want[5])) return kDecBadHeader;
    int32_t st = kDecOk;
    frame_index(d, p.blocks + d.blk_base, &st);
    if (st != kDecOk) return st;
    // frame_index has found the EndMark behind block nblk - 1 (and room for the content checksum): the frame ends there
    const uint32_t bc = (p.flags & SKY_F_BLOCK_CHECKSUM) ? 4u : 0u;
    uint64_t end = frame_header_bytes(cd.len);
    if (cd.nblk) {
        const DecBlock last = p.blocks[d.blk_base + cd.nblk - 1];
        end = last.off + (last.word & 0x7FFFFFFFu) + bc;
    }
    end += 4 + ((p.flags & SKY_F_CHECKSUM) ? 4u : 0u);
    if (d.frame_len != end) return kDecSize;  // bytes behind the frame
    if ((p.flags & SKY_F_CHECKSUM) && d.content_xxh != p.xxh[c]) return kDecChecksum;
    return kDecOk;
}

// Whole warp: a[0, n) == s[0, n)?  a any alignment (read in aligned 4-byte words), s 16-byte aligned.  Every lane returns
// the same answer.
__device__ __forceinline__ bool warp_equal(const uint8_t *a, const uint8_t *s, uint32_t n, unsigned lane) {
    bool ok = true;
    const uint32_t sh = (uint32_t)(reinterpret_cast<uintptr_t>(a) & 3u) * 8u;
    const uint32_t *aw = reinterpret_cast<const uint32_t *>(reinterpret_cast<uintptr_t>(a) & ~(uintptr_t)3);
    const uint4 *sv = reinterpret_cast<const uint4 *>(s);
    const uint32_t nvec = n >> 4;
    for (uint32_t k = lane; k < nvec; k += 32) {
        const uint4 v = __ldg(sv + k);
        const uint32_t *q = aw + 4 * (size_t)k;
        const uint32_t w0 = q[0], w1 = q[1], w2 = q[2], w3 = q[3];
        const uint32_t w4 = sh ? q[4] : 0u;  // (the word holding a[16k + 15]: no read past it)
        ok &= __funnelshift_r(w0, w1, sh) == v.x && __funnelshift_r(w1, w2, sh) == v.y && __funnelshift_r(w2, w3, sh) == v.z &&
              __funnelshift_r(w3, w4, sh) == v.w;
    }
    for (uint32_t k = (nvec << 4) + lane; k < n; k += 32) ok &= a[k] == s[k];
    return __all_sync(kFull, ok);
}

// Whole warp, warp-uniform arguments: compare-decode of the compressed block blk[0, slen) against its source block
// src[0, want) (16-byte aligned).  Every lane walks the same tokens; the lanes compare 32 bytes per round.  A structural
// failure returns at once; a byte mismatch is only reported once the whole block is known to be well formed.  kLinked:
// the block starts `pos` bytes into its chunk, whose bytes before src a match may reach.
template <bool kLinked>
__device__ __forceinline__ int32_t compare_decode(const uint8_t *blk, uint32_t slen, const uint8_t *src, uint32_t want, uint64_t pos,
                                                  unsigned lane) {
    bool ok = true;
    uint32_t ip = 0, q = 0;  // q: output position inside the block
    if (slen == 0) return kDecCorrupt;
    for (;;) {
        if (ip >= slen) return kDecCorrupt;
        const uint32_t token = blk[ip++];
        uint32_t ll = token >> 4;
        if (ll == 15 && !read_ext(blk, slen, ip, ll)) return kDecCorrupt;
        if (ll > slen - ip || ll > want - q) return kDecCorrupt;
        for (uint32_t k = lane; k < ll; k += 32) ok &= blk[ip + k] == __ldg(src + q + k);
        ip += ll;
        q += ll;
        if (ip == slen) break;  // last sequence: literals only
        if (slen - ip < 2) return kDecCorrupt;
        const uint32_t off = blk[ip] | (blk[ip + 1] << 8);
        ip += 2;
        if (off == 0 || (kLinked ? off > pos + q : off > q)) return kDecCorrupt;  // q - off before the block (chunk) start
        uint32_t ml = token & 15;
        if (ml == 15 && !read_ext(blk, slen, ip, ml)) return kDecCorrupt;
        ml += kMinMatch;
        // end-of-block rules: the match starts >= kMfLimit bytes before the block end and leaves kLastLiterals literals
        if (q + kMfLimit > want || ml > want - q - kLastLiterals) return kDecCorrupt;
        for (uint32_t k = lane; k < ml; k += 32) ok &= __ldg(src + q + k) == __ldg(src + q + k - off);
        q += ml;
    }
    if (q != want) return kDecLayout;
    return __all_sync(kFull, ok) ? kDecOk : kVerifyMismatch;
}

// Whole warp: block j of chunk cd as frame_index found it.  -> kDecOk or the block's code.
template <bool kLinked>
__device__ __forceinline__ int32_t verify_block(const ChunkDesc &cd, const DecBlock &b, uint32_t j, bool bc, unsigned lane) {
    const uint8_t *blk = cd.dst + b.off;
    const uint32_t sz = b.word & 0x7FFFFFFFu;
    const uint64_t pos = (uint64_t)j * kBlock;
    const uint32_t want = (uint32_t)min((uint64_t)kBlock, cd.len - pos);
    if (bc && xxh32_warp(blk, sz, lane) != b.chk) return kDecChecksum;
    if (b.word & 0x80000000u) {
        if (sz != want) return kDecLayout;
        return warp_equal(blk, cd.src + pos, sz, lane) ? kDecOk : kVerifyMismatch;
    }
    return compare_decode<kLinked>(blk, sz, cd.src + pos, want, pos, lane);
}

template <bool kLinked>
__device__ __forceinline__ void verify_index(const VerifyParams &p) {
    const uint32_t c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c < p.n_chunks) p.status[c] = verify_frame<kLinked>(p, c);
}

// Persistent, one warp per block (work item w = row * n + chunk).  A block is skipped once the frame or an earlier block
// of its chunk has failed.
template <bool kLinked>
__device__ __forceinline__ void verify_blocks(const VerifyParams &p) {
    const unsigned lane = threadIdx.x & 31;
    const bool bc = (p.flags & SKY_F_BLOCK_CHECKSUM) != 0;
    for (uint32_t c, j; claim_row_major(p.counter, p.n_chunks, p.rows, lane, c, j);) {
        const ChunkDesc cd = p.chunks[c];
        if (j >= cd.nblk) continue;
        if (!block_may_run(*reinterpret_cast<volatile int32_t *>(p.status + c), j)) continue;
        const int32_t r = verify_block<kLinked>(cd, p.blocks[p.blk_base[c] + j], j, bc, lane);
        if (r != kDecOk && lane == 0) atomicMin(p.status + c, block_fail(j, r));
    }
}

// One CTA per chunk: settle the status; with repair, rewrite a failing frame in place as the chunk's stored-block frame --
// the stage's header (write_frame_header), every block stored raw from the chunk (with its block checksum under
// SKY_F_BLOCK_CHECKSUM), the EndMark and the content checksum (finish_frame) -- frame_need(n, flags) bytes, which the
// frame's capacity holds.
template <bool kLinked>
__device__ __forceinline__ void verify_settle(const VerifyParams &p) {
    __shared__ int32_t code;
    const uint32_t c = blockIdx.x;
    const unsigned warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        code = settle_status(p.status[c]);
        p.status_out[c] = code;
    }
    __syncthreads();
    if (code == kDecOk || !p.repair) return;
    const ChunkDesc cd = p.chunks[c];
    const uint32_t bc = (p.flags & SKY_F_BLOCK_CHECKSUM) ? 4u : 0u;
    const uint64_t hdr = frame_header_bytes(cd.len);
    for (uint32_t j = 0; j < cd.nblk; j++) {
        const uint64_t pos = (uint64_t)j * kBlock;
        const uint32_t L = (uint32_t)min((uint64_t)kBlock, cd.len - pos);
        uint8_t *w = cd.dst + hdr + (uint64_t)j * (4 + kBlock + bc);
        if (threadIdx.x == 0) st_u32le(w, L | 0x80000000u);
        copy_block<kRepairWarps, true>(w + 4, cd.src + pos, L, warp, lane);
        if (bc && warp == j % kRepairWarps) block_checksum(cd.src + pos, L, w + 4 + L, lane);  // (the same bytes, from the chunk)
    }
    if (threadIdx.x == 0) {
        write_frame_header<kLinked>(cd.dst, cd.len, p.flags);
        uint8_t *e = cd.dst + hdr + (uint64_t)cd.nblk * (4 + bc) + cd.len;
        st_u32le(e, 0);  // EndMark
        p.frame_len[c] = (uint64_t)(e - cd.dst) + 4;
        if (p.flags & SKY_F_CHECKSUM) finish_frame(cd.dst, p.frame_len + c, p.xxh[c]);
    }
}

__global__ void sky_verify_index_kernel(const VerifyParams p) { verify_index<false>(p); }
__global__ void __launch_bounds__(kVerifyThreads, 2) sky_verify_kernel(const VerifyParams p) { verify_blocks<false>(p); }
__global__ void __launch_bounds__(kRepairWarps * 32) sky_verify_settle_kernel(const VerifyParams p) { verify_settle<false>(p); }
// SKY_F_LINKED: the same three for linked frames
__global__ void sky_verify_linked_index_kernel(const VerifyParams p) { verify_index<true>(p); }
__global__ void __launch_bounds__(kVerifyThreads, 2) sky_verify_linked_kernel(const VerifyParams p) { verify_blocks<true>(p); }
__global__ void __launch_bounds__(kRepairWarps * 32) sky_verify_linked_settle_kernel(const VerifyParams p) { verify_settle<true>(p); }

}  // namespace sky

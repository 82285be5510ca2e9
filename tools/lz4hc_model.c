/*
 * lz4hc_model.c -- sequential CPU twin of the high-ratio (SKY_F_HC) block compressor (skyplane_b200/csrc/lz4hc.cuh).
 *
 * NOT product code: the specification of the HC parse.  The kernel's frames are byte-identical to the ones built from
 * this program (tests/test_gpu_hc.py), and this program's frames decode with liblz4, pyarrow and the strict oracle
 * decoder (tests/test_hc_model.py).
 *
 * Per 64 KiB block of length L (independent blocks: nothing is shared between blocks):
 *   positions  p = 0 .. mflimit (= L - 12) may start a match; a match ends at or before matchlimit (= L - 5).
 *   hash       h(p) = (le32(src + p) * 2654435761) >> (32 - hash_bits)       (4 bytes: the minimum match)
 *   chains     inserting p = 0, 1, ... in order: chain[p] = the latest earlier position with hash h(p) (none if there is
 *              none), then head[h(p)] = p.
 *   best match for every p: walk chain[p], chain[chain[p]], ... at most `depth` candidates, nearest first.  A candidate's
 *              length is the common prefix of src+p and src+cand, at most cap(p) = min(nice, matchlimit - p).  The
 *              longest wins; on a tie the nearer (earlier walked) one stays.  The walk stops when a length reaches
 *              cap(p).  Lengths below 4 count as no match.
 *   lazy parse from the cursor (initially 0): the first p >= cursor with len(p) >= 4 and not len(p + 1) > len(p)
 *              (len(mflimit + 1) = 0) starts the next match.  A match of length `nice` is extended byte by byte with the
 *              same candidate up to matchlimit.  Emit literals [anchor, p) + the match; cursor = anchor = match end.
 *   emit       standard LZ4 sequences; the final literals [anchor, L).  A block whose compressed size would exceed
 *              L - 1 is stored raw (return 0), as LZ4F_makeBlock does.
 *   linked     (SKY_F_LINKED, hc_compress_block_linked) the hist source bytes before src are visible: 0 for a chunk's
 *              first block, 65536 for every later one (FLG B.Indep clear when the chunk has more than one block).  The
 *              chains are exact sequential insertion over p = -hist .. mflimit, the window's positions first; only the
 *              block's positions start matches.  A walk stops at the first candidate more than 65535 bytes back, and that
 *              candidate uses no depth.  Candidates are compared against the chunk's source bytes, so a match may run
 *              from the previous block into this one.  Block j depends on source bytes only, never on block j-1's output.
 *              With hist = 0 it is hc_compress_block, byte for byte.
 *
 * Build: gcc -O2 -shared -fPIC -o tools/bin/liblz4hc.so tools/lz4hc_model.c
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define MINMATCH 4
#define MFLIMIT 12
#define LASTLITERALS 5

typedef struct {
    int depth;      /* chain candidates walked per position (kernel: sky_kernel_config(4)) */
    int hash_bits;  /* log2 of the head table's entries (kernel: sky_kernel_config(5)) */
    int nice;       /* length at which a position's search stops; the parse extends such matches (sky_kernel_config(6)) */
} hc_opts;

static uint32_t rd32(const uint8_t *p) { uint32_t v; memcpy(&v, p, 4); return v; }

static uint32_t emit(uint8_t *out, uint32_t op, const uint8_t *src, uint32_t anchor, uint32_t ll, uint32_t ml, uint32_t off) {
    uint32_t mcode = ml ? ml - MINMATCH : 0;
    out[op++] = (uint8_t)(((ll < 15 ? ll : 15) << 4) | (mcode < 15 ? mcode : 15));
    if (ll >= 15) { uint32_t r = ll - 15; for (; r >= 255; r -= 255) out[op++] = 255; out[op++] = (uint8_t)r; }
    memcpy(out + op, src + anchor, ll); op += ll;
    if (ml) {
        out[op++] = (uint8_t)off; out[op++] = (uint8_t)(off >> 8);
        if (mcode >= 15) { uint32_t r = mcode - 15; for (; r >= 255; r -= 255) out[op++] = 255; out[op++] = (uint8_t)r; }
    }
    return op;
}

#define WINDOW 65535  /* the largest offset */

/* returns the compressed size, or 0 if the block does not shrink (store raw); out capacity >= L + 2048.
   src[-hist .. -1] are visible (linked blocks); hist = 0: an independent block. */
static uint32_t compress_block(const uint8_t *src, uint32_t L, uint32_t hist, uint8_t *out, const hc_opts *o) {
    uint32_t op = 0, anchor = 0;
    if (L >= MFLIMIT + 1) {
        const uint32_t mflimit = L - MFLIMIT, matchlimit = L - LASTLITERALS;
        const uint32_t nh = 1u << o->hash_bits, nice = (uint32_t)o->nice;
        const int64_t none = INT64_MIN;
        int64_t *head = malloc(nh * sizeof(int64_t));
        int64_t *chain = (int64_t *)malloc((hist + mflimit + 1) * sizeof(int64_t)) + hist;  /* chain[p], p = -hist .. mflimit */
        uint32_t *blen = calloc(mflimit + 2, sizeof(uint32_t)), *boff = calloc(mflimit + 2, sizeof(uint32_t));
        for (uint32_t h = 0; h < nh; h++) head[h] = none;
        for (int64_t p = -(int64_t)hist; p <= (int64_t)mflimit; p++) {
            const uint32_t h = (rd32(src + p) * 2654435761u) >> (32 - o->hash_bits);
            chain[p] = head[h];
            head[h] = p;
        }
        for (uint32_t p = 0; p <= mflimit; p++) {
            const uint32_t cap = matchlimit - p < nice ? matchlimit - p : nice;
            uint32_t best = 0, bo = 0;
            int64_t c = chain[p];
            for (int k = 0; k < o->depth && c != none && (int64_t)p - c <= WINDOW; k++, c = chain[c]) {
                uint32_t len = 0;
                while (len < cap && src[p + len] == src[c + len]) len++;
                if (len > best) { best = len; bo = (uint32_t)(p - c); }
                if (best == cap) break;
            }
            if (best >= MINMATCH) { blen[p] = best; boff[p] = bo; }
        }
        uint32_t p = 0;
        while (p <= mflimit) {
            const uint32_t ml0 = blen[p];
            if (ml0 < MINMATCH || blen[p + 1] > ml0) { p++; continue; }  /* (blen[mflimit + 1] = 0) */
            uint32_t ml = ml0;
            const uint32_t off = boff[p];
            if (ml == nice) while (p + ml < matchlimit && src[p + ml] == src[(int64_t)p - off + ml]) ml++;
            op = emit(out, op, src, anchor, p - anchor, ml, off);
            p += ml;
            anchor = p;
        }
        free(head); free(chain - hist); free(blen); free(boff);
    }
    op = emit(out, op, src, anchor, L - anchor, 0, 0);
    return op <= L - 1 ? op : 0;
}

uint32_t hc_compress_block(const uint8_t *src, uint32_t L, uint8_t *out, const hc_opts *o) {
    return compress_block(src, L, 0, out, o);
}

/* a block of a linked chunk: src[-hist .. -1] are the chunk's bytes before it (hist = 0 for block 0, else 65536) */
uint32_t hc_compress_block_linked(const uint8_t *src, uint32_t L, uint32_t hist, uint8_t *out, const hc_opts *o) {
    return compress_block(src, L, hist, out, o);
}

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
 *   optimal    (SKY_F_OPTIMAL, hc_compress_block_opt) the same chains and search (blen, boff); only the parse differs.
 *              It picks the sequences of least byte cost among these candidates, independent or linked:
 *     segments   positions split into segments of `seg` bytes [s0, s1) (seg = 0: one segment per block).  No match
 *                crosses its segment's end, and a segment's parse depends on nothing before it: it starts closed (no
 *                open literal run) at s0, which is what lets the kernel parse the segments in parallel.
 *     long       a position p <= mflimit with blen(p) = nice and s1 - p >= nice is long.  The first long position e at or
 *                after the window start a ends the window [a, e]: the parse reaches e by the cheapest path from a and
 *                takes the match at e extended with the same candidate up to min(matchlimit, s1), as the lazy parse
 *                extends it (liblz4's optimal parse takes a match past its sufficient length the same way).  The next
 *                window starts closed at its end.  Without a long position the window is [a, s1].
 *     candidates from p in a window [a, e]: the literal p -> p + 1, and a match of every length ml = 4 .. min(blen(p), e - p)
 *                at boff(p) (so lengths up to nice - 1: no long position lies inside a window).
 *     cost       the bytes a sequence takes: 1 + litext(ll) + ll + 2 + mlext(ml - 4), where a length field's extension
 *                bytes are litext(x) = mlext(x) = x >= 15 ? 1 + (x - 15) / 255 : 0 (the final literals' token is the same
 *                in every parse).  A literal run is carried as liblz4 carries it: each position keeps one state (cost,
 *                run, last) -- cost of the cheapest path to it including its open run's literal bytes, that run's length,
 *                and the length of the match that ends there (0: reached by a literal).  A literal adds
 *                lit(run + 1) - lit(run), lit(x) = x + litext(x); a match adds 3 + mlext(ml - 4) and closes the run.
 *                One kept run per position is what makes this an approximation: two paths of equal cost with different
 *                runs may differ by one extension byte later.
 *     ties       positions are relaxed in order, each one's state final before it is relaxed; a state is replaced only
 *                by a lexicographically smaller (cost, run, last).  The order of relaxation therefore does not matter.
 *     backtrace  from e (or s1) back to a through `last`; the matches it passes, and the long match, are the window's.
 *     emission   the chosen matches in position order across all segments with one anchor, so a literal run that
 *                crosses a segment's start becomes one sequence; the final literals [anchor, L).  Stored raw as above.
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

/* literal run ll: its bytes plus its length field's extension bytes (the token is counted with the sequence) */
static uint32_t lit_price(uint32_t ll) { return ll + (ll >= 15 ? 1 + (ll - 15) / 255 : 0); }
/* a match of ml bytes after its literal run: token, offset, match length extension bytes */
static uint32_t match_price(uint32_t ml) { return 3 + (ml - MINMATCH >= 15 ? 1 + (ml - MINMATCH - 15) / 255 : 0); }

/* Optimal parse (hc_compress_block_opt): writes sel[p] = the length of the match the parse starts at p, 0 elsewhere.
   See the header comment for the rule; blen / boff are the search's (blen[p] = 0 below 4, p > mflimit: 0). */
static void opt_parse(const uint8_t *src, uint32_t L, uint32_t seg, uint32_t nice, const uint32_t *blen, const uint32_t *boff,
                      uint32_t *sel) {
    const uint32_t mflimit = L - MFLIMIT, matchlimit = L - LASTLITERALS;
    uint32_t *price = malloc((L + 1) * sizeof(uint32_t)), *run = malloc((L + 1) * sizeof(uint32_t)),
             *last = malloc((L + 1) * sizeof(uint32_t));
    if (seg == 0) seg = L;
    for (uint32_t s0 = 0; s0 < L; s0 += seg) {
        const uint32_t s1 = L - s0 < seg ? L : s0 + seg;  /* the segment's end: no match crosses it */
        uint32_t a = s0;
        while (a < s1) {
            uint32_t e = a;  /* the window ends at the first long position, else at the segment's end */
            while (e < s1 && !(e <= mflimit && blen[e] == nice && s1 - e >= nice)) e++;
            price[a] = 0; run[a] = 0; last[a] = 0;
            for (uint32_t q = a + 1; q <= e; q++) price[q] = UINT32_MAX;
            for (uint32_t p = a; p < e; p++) {  /* p's state is final: relax the literal and every match from p */
                const uint32_t ll = run[p] + 1, lp = price[p] - lit_price(run[p]) + lit_price(ll);
                uint32_t cp = lp, cr = ll, cm = 0;
                /* (cost, run, last) is compared lexicographically; the smaller replaces */
                if (cp < price[p + 1] || (cp == price[p + 1] && (cr < run[p + 1] || (cr == run[p + 1] && cm < last[p + 1])))) {
                    price[p + 1] = cp; run[p + 1] = cr; last[p + 1] = cm;
                }
                const uint32_t maxml = blen[p] < e - p ? blen[p] : e - p;
                for (uint32_t ml = MINMATCH; ml <= maxml; ml++) {
                    const uint32_t q = p + ml;
                    cp = price[p] + match_price(ml); cr = 0; cm = ml;
                    if (cp < price[q] || (cp == price[q] && (cr < run[q] || (cr == run[q] && cm < last[q])))) {
                        price[q] = cp; run[q] = cr; last[q] = cm;
                    }
                }
            }
            for (uint32_t q = a; q < e; q++) sel[q] = 0;
            for (uint32_t q = e; q > a;) {  /* backtrace */
                const uint32_t m = last[q];
                if (m) { q -= m; sel[q] = m; } else q--;
            }
            if (e == s1) break;
            uint32_t ml = nice;  /* the long match at e, extended with the same candidate, clipped to the segment */
            const uint32_t lim = (matchlimit < s1 ? matchlimit : s1) - e;
            while (ml < lim && src[e + ml] == src[(int64_t)e - boff[e] + ml]) ml++;
            sel[e] = ml;
            a = e + ml;
        }
    }
    free(price); free(run); free(last);
}

/* returns the compressed size, or 0 if the block does not shrink (store raw); out capacity >= L + 2048.
   src[-hist .. -1] are visible (linked blocks); hist = 0: an independent block.  opt: the optimal parse with segments of
   `seg` bytes (0: one segment), else the lazy parse. */
static uint32_t compress_block(const uint8_t *src, uint32_t L, uint32_t hist, int opt, uint32_t seg, uint8_t *out, const hc_opts *o) {
    uint32_t op = 0, anchor = 0;
    if (L >= MFLIMIT + 1) {
        const uint32_t mflimit = L - MFLIMIT, matchlimit = L - LASTLITERALS;
        const uint32_t nh = 1u << o->hash_bits, nice = (uint32_t)o->nice;
        const int64_t none = INT64_MIN;
        int64_t *head = malloc(nh * sizeof(int64_t));
        int64_t *chain = (int64_t *)malloc((hist + mflimit + 1) * sizeof(int64_t)) + hist;  /* chain[p], p = -hist .. mflimit */
        uint32_t *blen = calloc(L + 1, sizeof(uint32_t)), *boff = calloc(L + 1, sizeof(uint32_t));
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
        if (opt) {
            uint32_t *sel = calloc(L + 1, sizeof(uint32_t));
            opt_parse(src, L, seg, nice, blen, boff, sel);
            for (uint32_t p = 0; p <= mflimit;) {
                if (!sel[p]) { p++; continue; }
                op = emit(out, op, src, anchor, p - anchor, sel[p], boff[p]);
                p += sel[p];
                anchor = p;
            }
            free(sel);
        } else {
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
        }
        free(head); free(chain - hist); free(blen); free(boff);
    }
    op = emit(out, op, src, anchor, L - anchor, 0, 0);
    return op <= L - 1 ? op : 0;
}

uint32_t hc_compress_block(const uint8_t *src, uint32_t L, uint8_t *out, const hc_opts *o) {
    return compress_block(src, L, 0, 0, 0, out, o);
}

/* a block of a linked chunk: src[-hist .. -1] are the chunk's bytes before it (hist = 0 for block 0, else 65536) */
uint32_t hc_compress_block_linked(const uint8_t *src, uint32_t L, uint32_t hist, uint8_t *out, const hc_opts *o) {
    return compress_block(src, L, hist, 0, 0, out, o);
}

/* the optimal parse (SKY_F_OPTIMAL) of an independent (hist = 0) or linked block, with parse segments of `seg` bytes
   (0: the whole block is one segment) */
uint32_t hc_compress_block_opt(const uint8_t *src, uint32_t L, uint32_t hist, uint32_t seg, uint8_t *out, const hc_opts *o) {
    return compress_block(src, L, hist, 1, seg, out, o);
}

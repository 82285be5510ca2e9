// md5_chain_bench.cu -- measures the dependent-chain latency of one MD5 block per lane on sm_90a
// for several instruction selections of the on-chain add.  Not product code: a measurement tool.  (md5.cuh's own
// selection -- a + M[g] as an IMAD off the chain, an all-ALU chain -- is measured by the in-situ mode below.)
//   V0: plain C (ptxas picks IMAD.IADD for the on-chain add: alu -> fma -> alu)
//   V1: on-chain add forced onto the ALU pipe by consuming its carry (IADD3 with carry-out)
//   V2: 3-input on-chain add (a, m+K, f) kept separate via carry trick on the inner add
// and, next to them, the product loop itself ("in-situ"): sky::md5_warp from md5.cuh in the flagship's arrangement --
// one MD5 warp per CTA, 32 CTAs, each lane streaming its own 8 MiB region of one device buffer through the staging ring
// in dynamic shared memory -- so the gap between the register-only chain and the real loop is measured, not inferred.
// Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 -std=c++17 -I skyplane_b200/csrc \
//            -o tools/bin/md5_chain_bench tools/md5_chain_bench.cu
// (-I another directory holding an md5.cuh measures that version of md5_warp; the first argument labels the lines.)
#include <cstdint>
#include <cstdio>
#include <cuda_runtime.h>

#include "md5.cuh"

#define F_(b, c, d) ((d) ^ ((b) & ((c) ^ (d))))
#define G_(b, c, d) ((c) ^ ((d) & ((b) ^ (c))))
#define H_(b, c, d) ((b) ^ (c) ^ (d))
#define I_(b, c, d) ((c) ^ ((b) | ~(d)))

__device__ __forceinline__ uint32_t mk_add(uint32_t m, uint32_t k) {
    uint32_t r;
    asm("add.u32 %0, %1, %2;" : "=r"(r) : "r"(m), "r"(k));
    return r;
}

template <int V>
struct Step {
    static __device__ __forceinline__ void run(uint32_t &a, uint32_t b, uint32_t f, uint32_t m, uint32_t k, int s,
                                               uint32_t &dummy) {
        if (V == 0) {
            uint32_t t = a + mk_add(m, k) + f;
            a = b + __funnelshift_l(t, t, s);
        } else if (V == 1) {
            uint32_t amk = a + mk_add(m, k);
            uint32_t t;
            asm("{add.cc.u32 %0, %2, %3;\n\t addc.u32 %1, %1, 0;}" : "=r"(t), "+r"(dummy) : "r"(amk), "r"(f));
            a = b + __funnelshift_l(t, t, s);
        } else {
            uint32_t t = a + m + k + f;  // whatever ptxas likes (re-associates K onto the chain)
            a = b + __funnelshift_l(t, t, s);
        }
    }
};

#define ST(FN, a, b, c, d, mi, k, s) Step<V>::run(a, b, FN(b, c, d), w[mi], k, s, dummy);

template <int V>
__device__ __forceinline__ void md5_block(uint32_t (&st)[4], const uint32_t (&w)[16], uint32_t &dummy) {
    uint32_t a = st[0], b = st[1], c = st[2], d = st[3];
    ST(F_, a, b, c, d, 0, 0xd76aa478, 7) ST(F_, d, a, b, c, 1, 0xe8c7b756, 12) ST(F_, c, d, a, b, 2, 0x242070db, 17) ST(F_, b, c, d, a, 3, 0xc1bdceee, 22)
    ST(F_, a, b, c, d, 4, 0xf57c0faf, 7) ST(F_, d, a, b, c, 5, 0x4787c62a, 12) ST(F_, c, d, a, b, 6, 0xa8304613, 17) ST(F_, b, c, d, a, 7, 0xfd469501, 22)
    ST(F_, a, b, c, d, 8, 0x698098d8, 7) ST(F_, d, a, b, c, 9, 0x8b44f7af, 12) ST(F_, c, d, a, b, 10, 0xffff5bb1, 17) ST(F_, b, c, d, a, 11, 0x895cd7be, 22)
    ST(F_, a, b, c, d, 12, 0x6b901122, 7) ST(F_, d, a, b, c, 13, 0xfd987193, 12) ST(F_, c, d, a, b, 14, 0xa679438e, 17) ST(F_, b, c, d, a, 15, 0x49b40821, 22)
    ST(G_, a, b, c, d, 1, 0xf61e2562, 5) ST(G_, d, a, b, c, 6, 0xc040b340, 9) ST(G_, c, d, a, b, 11, 0x265e5a51, 14) ST(G_, b, c, d, a, 0, 0xe9b6c7aa, 20)
    ST(G_, a, b, c, d, 5, 0xd62f105d, 5) ST(G_, d, a, b, c, 10, 0x02441453, 9) ST(G_, c, d, a, b, 15, 0xd8a1e681, 14) ST(G_, b, c, d, a, 4, 0xe7d3fbc8, 20)
    ST(G_, a, b, c, d, 9, 0x21e1cde6, 5) ST(G_, d, a, b, c, 14, 0xc33707d6, 9) ST(G_, c, d, a, b, 3, 0xf4d50d87, 14) ST(G_, b, c, d, a, 8, 0x455a14ed, 20)
    ST(G_, a, b, c, d, 13, 0xa9e3e905, 5) ST(G_, d, a, b, c, 2, 0xfcefa3f8, 9) ST(G_, c, d, a, b, 7, 0x676f02d9, 14) ST(G_, b, c, d, a, 12, 0x8d2a4c8a, 20)
    ST(H_, a, b, c, d, 5, 0xfffa3942, 4) ST(H_, d, a, b, c, 8, 0x8771f681, 11) ST(H_, c, d, a, b, 11, 0x6d9d6122, 16) ST(H_, b, c, d, a, 14, 0xfde5380c, 23)
    ST(H_, a, b, c, d, 1, 0xa4beea44, 4) ST(H_, d, a, b, c, 4, 0x4bdecfa9, 11) ST(H_, c, d, a, b, 7, 0xf6bb4b60, 16) ST(H_, b, c, d, a, 10, 0xbebfbc70, 23)
    ST(H_, a, b, c, d, 13, 0x289b7ec6, 4) ST(H_, d, a, b, c, 0, 0xeaa127fa, 11) ST(H_, c, d, a, b, 3, 0xd4ef3085, 16) ST(H_, b, c, d, a, 6, 0x04881d05, 23)
    ST(H_, a, b, c, d, 9, 0xd9d4d039, 4) ST(H_, d, a, b, c, 12, 0xe6db99e5, 11) ST(H_, c, d, a, b, 15, 0x1fa27cf8, 16) ST(H_, b, c, d, a, 2, 0xc4ac5665, 23)
    ST(I_, a, b, c, d, 0, 0xf4292244, 6) ST(I_, d, a, b, c, 7, 0x432aff97, 10) ST(I_, c, d, a, b, 14, 0xab9423a7, 15) ST(I_, b, c, d, a, 5, 0xfc93a039, 21)
    ST(I_, a, b, c, d, 12, 0x655b59c3, 6) ST(I_, d, a, b, c, 3, 0x8f0ccc92, 10) ST(I_, c, d, a, b, 10, 0xffeff47d, 15) ST(I_, b, c, d, a, 1, 0x85845dd1, 21)
    ST(I_, a, b, c, d, 8, 0x6fa87e4f, 6) ST(I_, d, a, b, c, 15, 0xfe2ce6e0, 10) ST(I_, c, d, a, b, 6, 0xa3014314, 15) ST(I_, b, c, d, a, 13, 0x4e0811a1, 21)
    ST(I_, a, b, c, d, 4, 0xf7537e82, 6) ST(I_, d, a, b, c, 11, 0xbd3af235, 10) ST(I_, c, d, a, b, 2, 0x2ad7d2bb, 15) ST(I_, b, c, d, a, 9, 0xeb86d391, 21)
    st[0] += a; st[1] += b; st[2] += c; st[3] += d;
}

template <int V>
__global__ void chain(uint32_t *out, int nblocks, long long *cycles) {
    uint32_t st[4] = {0x67452301u, 0xefcdab89u, 0x98badcfeu, 0x10325476u};
    uint32_t w[16];
    for (int i = 0; i < 16; i++) w[i] = threadIdx.x * 2654435761u + i * 40503u + blockIdx.x;
    uint32_t dummy = 0;
    long long t0 = clock64();
    for (int i = 0; i < nblocks; i++) {
        md5_block<V>(st, w, dummy);
        w[i & 15] += st[0];  // keep the message changing without memory traffic
    }
    long long t1 = clock64();
    out[blockIdx.x * blockDim.x + threadIdx.x] = st[0] ^ st[1] ^ st[2] ^ st[3] ^ dummy;
    if (threadIdx.x == 0) cycles[blockIdx.x] = t1 - t0;
}

template <int V>
void run(const char *name, int warps_per_cta, int ctas) {
    uint32_t *out;
    long long *cyc;
    cudaMalloc(&out, sizeof(uint32_t) * ctas * warps_per_cta * 32);
    cudaMalloc(&cyc, sizeof(long long) * ctas);
    const int nb = 20000;
    chain<V><<<ctas, warps_per_cta * 32>>>(out, 1000, cyc);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    cudaEventRecord(e0);
    chain<V><<<ctas, warps_per_cta * 32>>>(out, nb, cyc);
    cudaEventRecord(e1);
    cudaDeviceSynchronize();
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    long long c0;
    cudaMemcpy(&c0, cyc, sizeof c0, cudaMemcpyDeviceToHost);
    double cpb = (double)c0 / nb;
    printf("%-28s warps/cta=%2d ctas=%3d  cycles/block=%8.1f  cycles/step=%6.2f  per-stream=%.4f GB/s  agg=%.1f GB/s (%.3f ms)\n", name,
           warps_per_cta, ctas, cpb, cpb / 64, 64.0 * nb / (ms * 1e-3) / 1e9, 64.0 * nb * ctas * warps_per_cta * 32 / (ms * 1e-3) / 1e9, ms);
    cudaFree(out);
    cudaFree(cyc);
}

// ---- in-situ: the product's md5_warp ------------------------------------------------------------------------
constexpr int kInsituCtas = 32;                 // 1024 chunks = 32 MD5 groups, one per digest CTA
constexpr uint64_t kInsituLaneBytes = 8 << 20;  // 8 MiB per lane (chunk)
constexpr uint32_t kInsituRingBytes = SKY_MD5_SLOTS * 2048;

__global__ void fill(uint64_t *p, uint64_t n, uint64_t seed) {
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t z = seed + (i + 1) * 0x9e3779b97f4a7c15ull;  // splitmix64
        z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
        z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
        p[i] = z ^ (z >> 31);
    }
}

// __launch_bounds__ as sky_fused_kernel's, so md5_warp is compiled under the same register budget.
// Lengths and `active` come from device memory, as the fused kernel reads them from its chunk table: constants here
// let ptxas compile a different loop (without the per-lane branches the fused kernel's copy has).
__global__ void __launch_bounds__(448, 2) insitu(const uint8_t *buf, const uint64_t *lens, uint8_t *digests, long long *cycles) {
    extern __shared__ __align__(128) uint8_t smem[];
    const unsigned lane = threadIdx.x & 31;
    const uint64_t c = (uint64_t)blockIdx.x * 32 + lane;
    const uint64_t len = lens[c];
    __syncwarp();
    const long long t0 = clock64();
    sky::md5_warp(reinterpret_cast<uint32_t *>(smem), buf + c * kInsituLaneBytes, len, len != 0, digests + c * 16, lane);
    __syncwarp();
    const long long t1 = clock64();
    if (lane == 0) cycles[blockIdx.x] = t1 - t0;
}

void run_insitu(const char *label) {
    const uint64_t bytes = kInsituLaneBytes * 32 * kInsituCtas;
    uint8_t *buf, *dg;
    uint64_t *lens;
    long long *cyc;
    cudaMalloc(&buf, bytes);
    cudaMalloc(&lens, sizeof(uint64_t) * 32 * kInsituCtas);
    uint64_t h_lens[32 * kInsituCtas];
    for (uint64_t &l : h_lens) l = kInsituLaneBytes;
    cudaMemcpy(lens, h_lens, sizeof h_lens, cudaMemcpyHostToDevice);
    cudaMalloc(&dg, 16 * 32 * kInsituCtas);
    cudaMalloc(&cyc, sizeof(long long) * kInsituCtas);
    fill<<<1024, 256>>>(reinterpret_cast<uint64_t *>(buf), bytes / 8, 1);
    cudaEvent_t e0, e1;
    cudaEventCreate(&e0);
    cudaEventCreate(&e1);
    const double nblocks = (double)(kInsituLaneBytes / 64);
    insitu<<<kInsituCtas, 32, kInsituRingBytes>>>(buf, lens, dg, cyc);  // warm-up
    for (int rep = 0; rep < 5; rep++) {
        cudaEventRecord(e0);
        insitu<<<kInsituCtas, 32, kInsituRingBytes>>>(buf, lens, dg, cyc);
        cudaEventRecord(e1);
        cudaError_t err = cudaDeviceSynchronize();
        if (err != cudaSuccess) {
            printf("in-situ: %s\n", cudaGetErrorString(err));
            return;
        }
        float ms;
        cudaEventElapsedTime(&ms, e0, e1);
        long long c[kInsituCtas];
        cudaMemcpy(c, cyc, sizeof c, cudaMemcpyDeviceToHost);
        long long lo = c[0], hi = c[0];
        for (long long v : c) lo = v < lo ? v : lo, hi = v > hi ? v : hi;
        printf("in-situ md5_warp [%s] rep %d  ctas=%d lanes=32 MiB/lane=%d  cycles/block=%8.1f (fastest CTA %.1f)  "
               "cycles/step=%6.2f  per-stream=%.4f GB/s  (%.3f ms)\n",
               label, rep, kInsituCtas, (int)(kInsituLaneBytes >> 20), hi / nblocks, lo / nblocks, hi / nblocks / 64,
               kInsituLaneBytes / (ms * 1e-3) / 1e9, ms);
    }
    cudaFree(buf);
    cudaFree(lens);
    cudaFree(dg);
    cudaFree(cyc);
}

int main(int argc, char **argv) {
    const char *label = argc > 1 ? argv[1] : "md5.cuh";
    int sms = 0;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
    printf("SMs=%d\n", sms);
    for (int wpc : {1, 4, 8, 16}) {
        run<0>("V0 imad-on-chain", wpc, sms);
        run<1>("V1 iadd3-carry-on-chain", wpc, sms);
        run<2>("V2 ptxas-free-form", wpc, sms);
    }
    run_insitu(label);
    return 0;
}

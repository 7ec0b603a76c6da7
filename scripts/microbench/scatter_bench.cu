// scatter_bench.cu -- microbenchmark behind DESIGN.md 6.1: what bounds scattered record stores on the GPU?
//
// Every CTA appends records to S private streams, picking the stream of each record pseudo-randomly (like the level-A partition
// kernel: a shared-memory cursor per stream, slot = atomicAdd). Knobs:
//   -s S        streams per CTA                       (open 128-byte lines per CTA; 2 CTAs of 512 threads per SM)
//   -w 16|32    bytes per store                       (32 = two records of a stream written back to back by one thread)
//   -l cta|part layout: CTA-major (a CTA's streams are adjacent: its stores stay inside total/G bytes) or partition-major
//               (stream p of every CTA adjacent: a CTA's stores spread over the whole buffer)
//   -g GB       total bytes written
// Prints GB/s for each configuration so that "streams per CTA", "store width" and "layout" can be separated. Build + run:
//   nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o scatter_bench scatter_bench.cu && ./scatter_bench
//
// Page-locality mode (-c MB): every CTA writes C MB of 16-byte records into S streams (-S, default 640), CTA-major, either into
// one region of C MB (today's level-A staging: the stores of a CTA hit all of its region's pages for the whole launch) or in
// consecutive slices of R MB each (-r, repeatable): the cursors restart in a fresh sub-region of R MB at every slice, so only the
// current slice's pages take stores. Same bytes, same streams per slice, same instructions; only the live footprint differs.
//   ./scatter_bench -c 57 -S 640 -r 57 -r 16 -r 4 -r 2
//
// Refinement mode (-b 1): the write pattern of refine_k's scatter sweep. One CTA per SM of 1024 threads (or two of 512), 1024 or
// 2048 bins per CTA, each bin a contiguous child region of its CTA, records to pseudo-random bins. Three ways to write them:
//   lone   one 16-byte store per record as it takes its slot (shared-memory atomic cursor)
//   pair   32-byte pairs: two records of a bin written back to back by one thread (an idealised sector mailbox)
//   batch  N records per CTA per batch: rank in the bin (one shared-memory atomic), block scan of the batch counts, the owner of a
//          bin claims its run, permute into bin order in shared memory, flush with consecutive threads on consecutive addresses
//   ./scatter_bench -b 1 -g 8
//
// Level-A mode (-a 1): the same lone and batched writes at level A's shape: 640 and 2560 streams per CTA, 16- and 32-byte
// records, two CTAs of 512 or one of 1024 threads per SM, and only the batch sizes that fit next to the shared memory the
// partition kernel's roll state takes.
//   ./scatter_bench -a 1 -g 8
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <vector>

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_)); exit(1); } } while (0)

__device__ __forceinline__ uint32_t mix(uint32_t x) { x ^= x >> 16; x *= 0x7feb352dU; x ^= x >> 15; x *= 0x846ca68bU; x ^= x >> 16; return x; }

template <int WIDTH>
__global__ void __launch_bounds__(512, 2) scatter_k(uint64_t *out, const uint64_t *stream_base /*[G][S] in 16-byte records*/, int S, uint32_t per_stream,
                                                   uint32_t records_per_cta) {
    extern __shared__ uint32_t cur[];          // S cursors
    for (int i = threadIdx.x; i < S; i += blockDim.x) cur[i] = 0;
    __syncthreads();
    const uint64_t *mybase = stream_base + (size_t)blockIdx.x * S;
    constexpr uint32_t RPS = WIDTH / 16;        // records per store
    for (uint32_t i = threadIdx.x; i < records_per_cta / RPS; i += blockDim.x) {
        const uint32_t h = mix(i * 2654435761u + blockIdx.x * 40503u);
        const uint32_t s = h % (uint32_t)S;
        const uint32_t slot = atomicAdd(&cur[s], RPS);
        if (slot + RPS > per_stream) continue;                   // stream full (the random pick is only balanced on average)
        uint64_t *dst = out + (mybase[s] + slot) * 2;
        const uint64_t a = h, b = ~(uint64_t)h;
        if (WIDTH == 16) asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"(a), "l"(b) : "memory");
        else asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};\n\tst.global.L1::no_allocate.v2.u64 [%3], {%4, %5};" ::"l"(dst), "l"(a), "l"(b),
                          "l"(dst + 2), "l"(a + 1), "l"(b + 1) : "memory");
    }
}

// CTA g writes nslice slices of recs_per_slice records; slice s owns the sub-region [(g * nslice + s) * S * per_stream, +S * per_stream)
__global__ void __launch_bounds__(512, 2) slice_k(uint64_t *out, int S, uint32_t per_stream, uint32_t recs_per_slice, int nslice) {
    extern __shared__ uint32_t cur[];
    for (int sl = 0; sl < nslice; ++sl) {
        for (int i = threadIdx.x; i < S; i += blockDim.x) cur[i] = 0;
        __syncthreads();
        const uint64_t region = ((uint64_t)blockIdx.x * nslice + sl) * S * per_stream;
        for (uint32_t i = threadIdx.x; i < recs_per_slice; i += blockDim.x) {
            const uint32_t h = mix(i * 2654435761u + (blockIdx.x * nslice + sl) * 40503u);
            const uint32_t s = h % (uint32_t)S;
            const uint32_t slot = atomicAdd(&cur[s], 1u);
            if (slot >= per_stream) continue;
            uint64_t *dst = out + (region + (uint64_t)s * per_stream + slot) * 2;
            asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"((uint64_t)h), "l"(~(uint64_t)h) : "memory");
        }
        __syncthreads();
    }
}

// ---- refinement mode ------------------------------------------------------------------------------------------------------
// CTA g owns bins [g * B, (g + 1) * B), bin b's region starts at b * per_bin records of W bytes. PAIR: two records per store.
template <int T, int W, bool PAIR>
__global__ void __launch_bounds__(T) rlone_k(uint64_t *out, int B, uint32_t per_bin, uint32_t records_per_cta) {
    extern __shared__ uint32_t cur[];
    for (int i = threadIdx.x; i < B; i += T) cur[i] = 0;
    __syncthreads();
    constexpr uint32_t RPS = PAIR ? 2 : 1;
    for (uint32_t i = threadIdx.x; i < records_per_cta / RPS; i += T) {
        const uint32_t h = mix(i * 2654435761u + blockIdx.x * 40503u);
        const uint32_t b = h % (uint32_t)B;
        const uint32_t slot = atomicAdd(&cur[b], RPS);
        if (slot + RPS > per_bin) continue;
        uint64_t *dst = out + ((uint64_t)blockIdx.x * B + b) * per_bin * 2 + (uint64_t)slot * 2;
        asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst), "l"((uint64_t)h), "l"(~(uint64_t)h) : "memory");
        if (PAIR) asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst + 2), "l"((uint64_t)h + 1), "l"(~(uint64_t)h) : "memory");
    }
}

// records of W bytes (8, 16, 32) in batches of N per CTA, up to MAXB bins (tag = rank << log2(MAXB) | bin)
template <int T, int W, int N, int MAXB = 2048>
__global__ void __launch_bounds__(T) rbatch_k(uint64_t *out, int B, uint32_t per_bin, uint32_t records_per_cta) {
    constexpr int NW = W / 8, RPT = N / T, BPT = MAXB / T;       // records and bins per thread
    constexpr int TB = MAXB == 2048 ? 11 : 12;
    static_assert(MAXB == 2048 || MAXB == 4096, "tag layout");
    extern __shared__ uint64_t sm[];
    uint64_t *stage = sm;                                                         // [N][NW]
    uint32_t *sslot = reinterpret_cast<uint32_t *>(stage + (size_t)N * NW);       // [N] global record index
    uint32_t *cnt = sslot + N, *roff = cnt + B, *rbase = roff + B;                // [B] each
    __shared__ uint32_t wtot[T / 32];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t cur[BPT];
    for (int q = 0; q < BPT; ++q) {
        const uint32_t b = threadIdx.x * BPT + q;
        cur[q] = 0;
        if (b < (uint32_t)B) cnt[b] = 0;
    }
    __syncthreads();
    for (uint32_t b0 = 0; b0 < records_per_cta; b0 += N) {
        uint32_t tag[RPT];
        uint64_t v[RPT];
#pragma unroll
        for (int j = 0; j < RPT; ++j) {
            const uint32_t i = b0 + threadIdx.x + T * j;
            const uint32_t h = mix(i * 2654435761u + blockIdx.x * 40503u);
            const uint32_t b = h % (uint32_t)B;
            v[j] = h;
            tag[j] = i < records_per_cta ? (atomicAdd(&cnt[b], 1u) << TB) | b : ~0u;
        }
        __syncthreads();
        uint32_t c[BPT], tsum = 0;
        for (int q = 0; q < BPT; ++q) {
            const uint32_t b = threadIdx.x * BPT + q;
            c[q] = b < (uint32_t)B ? cnt[b] : 0u;
            tsum += c[q];
        }
        uint32_t inc = tsum;
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, inc, o); if (lane >= o) inc += t; }
        if (lane == 31) wtot[warp] = inc;
        __syncthreads();
        uint32_t w = lane < T / 32 ? wtot[lane] : 0u, winc = w;
        for (int o = 1; o < 32; o <<= 1) { uint32_t t = __shfl_up_sync(0xffffffffu, winc, o); if (lane >= o) winc += t; }
        const uint32_t total = __shfl_sync(0xffffffffu, winc, 31);
        uint32_t off = __shfl_sync(0xffffffffu, winc - w, warp) + inc - tsum;
        for (int q = 0; q < BPT; ++q) {
            const uint32_t b = threadIdx.x * BPT + q;
            if (b < (uint32_t)B) { roff[b] = off; rbase[b] = b * per_bin + cur[q]; cnt[b] = 0; }
            off += c[q]; cur[q] += c[q];
        }
        __syncthreads();
#pragma unroll
        for (int j = 0; j < RPT; ++j) {
            if (tag[j] == ~0u) continue;
            const uint32_t b = tag[j] & (MAXB - 1u), rank = tag[j] >> TB;
            const uint32_t p = roff[b] + rank;
            for (int k = 0; k < NW; ++k) stage[(size_t)p * NW + k] = v[j] + k;
            sslot[p] = rank + rbase[b];
        }
        __syncthreads();
        uint64_t *cta_out = out + (uint64_t)blockIdx.x * B * per_bin * NW;
        for (uint32_t p = threadIdx.x; p < total; p += T) {
            uint64_t *dst = cta_out + (uint64_t)sslot[p] * NW;
            if (NW == 1) asm volatile("st.global.L1::no_allocate.u64 [%0], %1;" ::"l"(dst), "l"(stage[p]) : "memory");
            for (int k = 0; k + 1 < NW; k += 2)
                asm volatile("st.global.L1::no_allocate.v2.u64 [%0], {%1, %2};" ::"l"(dst + k), "l"(stage[(size_t)p * NW + k]), "l"(stage[(size_t)p * NW + k + 1]) : "memory");
        }
    }
}

// GB/s of record bytes, best of 3 (per_bin leaves 25 % slack over the mean: far more than the spread of the pseudo-random bins)
template <class F>
static float rtime(F launch, double bytes) {
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e30f;
    for (int rep = 0; rep < 3; ++rep) {
        CK(cudaEventRecord(e0));
        launch();
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
    }
    CK(cudaGetLastError());
    return (float)(bytes / 1e9 / (best / 1e3));
}

template <int T>
static void refine_row(int B, double gb, int SMs, uint64_t *d_out, size_t out_bytes) {
    const int G = SMs * (1024 / T);
    auto lone = [&](bool pair) {
        const uint32_t per_cta = (uint32_t)(gb * 1e9 / 16 / G), per_bin = (uint32_t)((uint64_t)per_cta * 5 / 4 / B + 8) & ~1u;
        if ((uint64_t)per_bin * B * G * 16 > out_bytes) { fprintf(stderr, "buffer too small\n"); exit(1); }
        auto k = pair ? rlone_k<T, 16, true> : rlone_k<T, 16, false>;
        return rtime([&] { k<<<G, T, B * 4>>>(d_out, B, per_bin, per_cta); }, (double)per_cta * G * 16);
    };
    auto batch = [&](auto kern, int W, int N) {
        const uint32_t per_cta = (uint32_t)(gb * 1e9 / W / G), per_bin = (uint32_t)((uint64_t)per_cta * 5 / 4 / B + 8) & ~1u;
        if ((uint64_t)per_bin * B * G * W > out_bytes) { fprintf(stderr, "buffer too small\n"); exit(1); }
        const size_t sm = (size_t)N * (W + 4) + 3 * (size_t)B * 4;
        if (sm > 220u << 10 || (1024 / T) * sm > 226u << 10) return -1.f;          // does not fit (1024 / T) CTAs per SM
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        return rtime([&] { kern<<<G, T, sm>>>(d_out, B, per_bin, per_cta); }, (double)per_cta * G * W);
    };
    printf("%5d x %4d | %5d | %6.0f %6.0f | %6.0f %6.0f %6.0f | %6.0f %6.0f | %6.0f\n", 1024 / T, T, B, lone(false), lone(true),
           batch(rbatch_k<T, 16, 2048>, 16, 2048), batch(rbatch_k<T, 16, 4096>, 16, 4096), batch(rbatch_k<T, 16, 8192>, 16, 8192),
           batch(rbatch_k<T, 8, 8192>, 8, 8192), batch(rbatch_k<T, 8, 16384>, 8, 16384), batch(rbatch_k<T, 32, 4096>, 32, 4096));
    fflush(stdout);
}

// Level-A mode (-a 1): the write pattern of levelA_scatter_roll_k -- S = 640 or 2560 partition streams per CTA, CTA-major
// regions, 16- or 32-byte records -- at two CTAs of 512 threads or one of 1024 per SM. Every CTA also holds the shared memory of
// the roll kernel's warp slices (2952 bytes per warp), so a batch only gets what is left next to them and the batch tables
// (3 x 4 bytes per stream); "-" marks a batch that does not fit that room.
template <int T>
static void levela_row(int S, int W, double gb, int SMs, uint64_t *d_out, size_t out_bytes) {
    const int G = SMs * (1024 / T);
    const size_t roll = (size_t)(T / 32) * 2952;
    const size_t room = T == 1024 ? 232448 - 128 : 115584 - 128;        // opt-in limit per CTA; half an SM minus the reservation
    const uint32_t per_cta = (uint32_t)(gb * 1e9 / W / G), per_bin = (uint32_t)((uint64_t)per_cta * 5 / 4 / S + 8) & ~1u;
    if ((uint64_t)per_bin * S * G * W > out_bytes) { fprintf(stderr, "buffer too small\n"); exit(1); }
    auto lone = [&]() {
        auto k = W == 16 ? rlone_k<T, 16, false> : rlone_k<T, 16, true>;
        const size_t sm = roll + (size_t)S * 4;
        CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        const uint32_t pc = W == 16 ? per_cta : 2 * per_cta, pb = W == 16 ? per_bin : 2 * per_bin;    // 16-byte units
        return rtime([&] { k<<<G, T, sm>>>(d_out, S, pb, pc); }, (double)per_cta * G * W);
    };
    auto batch = [&](auto kern, int N) {
        const size_t sm = (size_t)N * (W + 4) + 3 * (size_t)S * 4 + roll;
        if (N % T || sm > room) return -1.f;
        CK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        return rtime([&] { kern<<<G, T, sm>>>(d_out, S, per_bin, per_cta); }, (double)per_cta * G * W);
    };
    printf("%5d x %4d | %5d | %3d | %6.0f", 1024 / T, T, S, W, lone());
    if (W == 16)
        printf(" | %6.0f %6.0f %6.0f %6.0f %6.0f %6.0f\n", batch(rbatch_k<T, 16, 1024, 4096>, 1024), batch(rbatch_k<T, 16, 2048, 4096>, 2048),
               batch(rbatch_k<T, 16, 3072, 4096>, 3072), batch(rbatch_k<T, 16, 4096, 4096>, 4096), batch(rbatch_k<T, 16, 5120, 4096>, 5120),
               batch(rbatch_k<T, 16, 6144, 4096>, 6144));
    else
        printf(" | %6.0f %6.0f %6.0f %6.0f %6.0f %6.0f\n", batch(rbatch_k<T, 32, 1024, 4096>, 1024), batch(rbatch_k<T, 32, 2048, 4096>, 2048),
               batch(rbatch_k<T, 32, 3072, 4096>, 3072), batch(rbatch_k<T, 32, 4096, 4096>, 4096), batch(rbatch_k<T, 32, 5120, 4096>, 5120),
               batch(rbatch_k<T, 32, 6144, 4096>, 6144));
    fflush(stdout);
}

// GB/s of record bytes, best of `reps`, for C MB per CTA written in slices of R MB
static float run_slices(double cta_mb, double slice_mb, int S, int G, uint64_t *d_out, size_t out_bytes, int reps) {
    int nslice = (int)(cta_mb / slice_mb + 0.5);
    if (nslice < 1) nslice = 1;
    const uint64_t per_cta = (uint64_t)(cta_mb * 1e6 / 16);
    const uint32_t per_slice = (uint32_t)(per_cta / nslice);
    const uint32_t per_stream = (uint32_t)((uint64_t)per_slice * 5 / 4 / S + 8) & ~1u;
    if ((uint64_t)per_stream * S * nslice * G * 16 > out_bytes) { fprintf(stderr, "buffer too small\n"); exit(1); }
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e30f;
    for (int rep = 0; rep < reps; ++rep) {
        CK(cudaEventRecord(e0));
        slice_k<<<G, 512, S * 4>>>(d_out, S, per_stream, per_slice, nslice);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
    }
    CK(cudaGetLastError());
    return (float)((double)per_slice * nslice * G * 16 / 1e9 / (best / 1e3));
}

static float run(int width, int S, bool cta_major, double gb, int G, uint64_t *d_out, size_t out_bytes) {
    const uint64_t total_rec = (uint64_t)(gb * 1e9 / 16);
    const uint32_t per_cta = (uint32_t)(total_rec / G);
    uint32_t per_stream = (uint32_t)((uint64_t)per_cta * 5 / 4 / S + 8) & ~1u;      // 25 % slack, even (32-byte alignment of every stream)
    if ((uint64_t)per_stream * S * G * 16 > out_bytes) { fprintf(stderr, "buffer too small\n"); exit(1); }
    std::vector<uint64_t> base((size_t)G * S);
    for (int g = 0; g < G; ++g)
        for (int s = 0; s < S; ++s) base[(size_t)g * S + s] = cta_major ? ((uint64_t)g * S + s) * per_stream : ((uint64_t)s * G + g) * per_stream;
    uint64_t *d_base;
    CK(cudaMalloc(&d_base, base.size() * 8));
    CK(cudaMemcpy(d_base, base.data(), base.size() * 8, cudaMemcpyHostToDevice));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    float best = 1e30f;
    for (int rep = 0; rep < 3; ++rep) {
        CK(cudaEventRecord(e0));
        if (width == 16) scatter_k<16><<<G, 512, S * 4>>>(d_out, d_base, S, per_stream, per_cta);
        else scatter_k<32><<<G, 512, S * 4>>>(d_out, d_base, S, per_stream, per_cta);
        CK(cudaEventRecord(e1));
        CK(cudaEventSynchronize(e1));
        float ms; CK(cudaEventElapsedTime(&ms, e0, e1));
        if (ms < best) best = ms;
    }
    CK(cudaGetLastError());
    CK(cudaFree(d_base));
    return (float)((double)per_cta * G * 16 / 1e9 / (best / 1e3));
}

int main(int argc, char **argv) {
    double gb = 8.0, cta_mb = 0;
    int S = 640, refine_mode = 0, levela_mode = 0;
    std::vector<double> slice_mb;
    for (int i = 1; i + 1 < argc; i += 2) {
        if (!strcmp(argv[i], "-g")) gb = atof(argv[i + 1]);
        else if (!strcmp(argv[i], "-c")) cta_mb = atof(argv[i + 1]);
        else if (!strcmp(argv[i], "-S")) S = atoi(argv[i + 1]);
        else if (!strcmp(argv[i], "-r")) slice_mb.push_back(atof(argv[i + 1]));
        else if (!strcmp(argv[i], "-b")) refine_mode = atoi(argv[i + 1]);
        else if (!strcmp(argv[i], "-a")) levela_mode = atoi(argv[i + 1]);
    }
    cudaDeviceProp p; CK(cudaGetDeviceProperties(&p, 0));
    const int G = p.multiProcessorCount * 2;
    if (levela_mode) {
        const size_t out_bytes = (size_t)(gb * 1.4e9) + (64u << 20);
        uint64_t *d_out;
        CK(cudaMalloc(&d_out, out_bytes));
        CK(cudaMemset(d_out, 0, out_bytes));
        printf("%s, level-A write pattern next to the roll kernel's warp slices, %.1f GB per run; GB/s of record bytes, best of 3 "
               "(-: does not fit)\n", p.name, gb);
        printf("%12s | %5s | %3s | %6s | %6s %6s %6s %6s %6s %6s\n", "CTAs x thr", "strms", "W", "lone", "b/1k", "b/2k", "b/3k", "b/4k",
               "b/5k", "b/6k");
        for (int S2 : {640, 2560})
            for (int W : {16, 32}) {
                levela_row<512>(S2, W, gb, p.multiProcessorCount, d_out, out_bytes);
                levela_row<1024>(S2, W, gb, p.multiProcessorCount, d_out, out_bytes);
            }
        CK(cudaFree(d_out));
        return 0;
    }
    if (refine_mode) {
        const size_t out_bytes = (size_t)(gb * 1.4e9) + (64u << 20);
        uint64_t *d_out;
        CK(cudaMalloc(&d_out, out_bytes));
        CK(cudaMemset(d_out, 0, out_bytes));
        printf("%s, refinement write pattern, %.1f GB per run; GB/s of record bytes, best of 3 (-: does not fit shared memory)\n", p.name, gb);
        printf("%12s | %5s | %6s %6s | %6s %6s %6s | %6s %6s | %6s\n", "CTAs x thr", "bins", "lone16", "pair32", "b16/2k", "b16/4k",
               "b16/8k", "b8/8k", "b8/16k", "b32/4k");
        for (int B : {1024, 2048}) {
            refine_row<1024>(B, gb, p.multiProcessorCount, d_out, out_bytes);
            refine_row<512>(B, gb, p.multiProcessorCount, d_out, out_bytes);
        }
        CK(cudaFree(d_out));
        return 0;
    }
    if (cta_mb > 0) {
        if (slice_mb.empty()) slice_mb.push_back(cta_mb);
        const size_t out_bytes = (size_t)(cta_mb * 1e6 * G * 1.3) + (64u << 20);
        uint64_t *d_out;
        CK(cudaMalloc(&d_out, out_bytes));
        CK(cudaMemset(d_out, 0, out_bytes));
        CK(cudaFuncSetAttribute(slice_k, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 << 10));
        printf("%s, %d CTAs x 512 threads, %d streams, %.1f MB per CTA (%.1f GB per run); GB/s of record bytes, best of 3\n", p.name, G, S, cta_mb,
               cta_mb * G / 1e3);
        for (int round = 0; round < 3; ++round)      // alternating: every slice size once per round
            for (double r : slice_mb) {
                printf("round %d  slice %6.1f MB  %8.0f GB/s\n", round, r, run_slices(cta_mb, r, S, G, d_out, out_bytes, 3));
                fflush(stdout);
            }
        CK(cudaFree(d_out));
        return 0;
    }
    const size_t out_bytes = (size_t)(gb * 1.4e9) + (64u << 20);
    uint64_t *d_out;
    CK(cudaMalloc(&d_out, out_bytes));
    CK(cudaMemset(d_out, 0, out_bytes));
    CK(cudaFuncSetAttribute(scatter_k<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 << 10));
    CK(cudaFuncSetAttribute(scatter_k<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 << 10));
    printf("%s, %d CTAs x 512 threads, %.1f GB per run; GB/s of record bytes\n", p.name, G, gb);
    printf("%8s | %12s %12s | %12s %12s\n", "streams", "16B cta-maj", "32B cta-maj", "16B part-maj", "32B part-maj");
    const int Ss[] = {32, 64, 128, 256, 512, 1024, 2048, 4096, 8192};
    for (int S : Ss) {
        printf("%8d | %12.0f %12.0f | %12.0f %12.0f\n", S, run(16, S, true, gb, G, d_out, out_bytes), run(32, S, true, gb, G, d_out, out_bytes),
               run(16, S, false, gb, G, d_out, out_bytes), run(32, S, false, gb, G, d_out, out_bytes));
        fflush(stdout);
    }
    CK(cudaFree(d_out));
    return 0;
}

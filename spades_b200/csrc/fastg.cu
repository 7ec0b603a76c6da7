// fastg.cu -- the graph as FASTG (io::FastgWriter) and the unitigs as spades-gbuilder's FASTA, formatted on the device.
//   FastgWriter::WriteSegmentsAndLinks (src/common/io/graph/fastg_writer.cpp:21-46): one record per edge of graph_.edges(), i.e. edge
//   3 + 2i, then its conjugate 4 + 2i unless the edge is self-conjugate; header = name(e) [':' names of the end vertex's outgoing
//   edges] ';'; body = the sequence wrapped at 60 (FastaWriter, io/reads/osequencestream.hpp:113-117).
//   gbuilder's unitig mode (projects/spades_tools/gbuilder.cpp:191-200): ">EDGE_<n>_length_<bases>", then the sequence wrapped at 60.
// The vertex structure comes from the GFA writer's host code (graph_vertices); the text is built here: a size kernel, scans, then per
// run of whole records a header kernel (one thread per record) and a body kernel over tiles of output bytes (a megabase edge spreads
// over many blocks). A run's buffer goes to pinned host memory on the copy stream while the next run is formatted.
#include <algorithm>

#include "fastg_fmt.cuh"
#include "graph.h"

namespace sg {

namespace {

const uint64_t kTile = (uint64_t)(kWrap + 1) * 64;     // body bytes per block of the body kernel: 64 lines
const size_t kRunCap = (size_t)128 << 20;              // largest run buffer: beyond it, longer runs gain nothing on the copies

struct Tables {
    const uint32_t *len, *raw;
    const uint64_t *eoff;       // edge text offsets in the graph's sequence
    const uint8_t *selfc;
    const uint64_t *lst_off, *lst, *end_slot;
    const uint64_t *rec;        // record r: 2i + (conjugate strand)
    int k;
    bool fastg;
};

__device__ __forceinline__ int record_header(const Tables &t, uint64_t r, char *d) {
    const uint64_t c = t.rec[r], i = c >> 1;
    if (!t.fastg) return fmt_unitig_header(d, i, t.len[i]);
    const uint64_t slot = t.end_slot[c];
    const uint64_t a = t.lst_off[slot], b = t.lst_off[slot + 1];
    uint64_t succ[kMaxSucc];
    int ns = 0;
    for (uint64_t j = a; j < b && ns < kMaxSucc; ++j) succ[ns++] = t.lst[j];
    return fmt_fastg_header(d, 3 + 2 * i + (c & 1), succ, ns, t.len, t.raw, t.selfc, t.k);
}

__global__ void fmt_size_k(Tables t, uint64_t R, uint32_t *hdr, uint64_t *size, uint64_t *ntile) {
    const uint64_t r = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= R) return;
    const uint32_t h = (uint32_t)record_header(t, r, nullptr);
    const uint64_t body = fmt_body_len(t.len[t.rec[r] >> 1]);
    hdr[r] = h;
    size[r] = h + body;
    ntile[r] = (body + kTile - 1) / kTile;
}

__global__ void fmt_header_k(Tables t, uint64_t r0, uint64_t r1, const uint64_t *off, char *out) {
    const uint64_t r = r0 + (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= r1) return;
    record_header(t, r, out + (off[r] - off[r0]));
}

// block b writes body tile tile0 + b; text holds the run's edges from graph offset text0
__global__ void fmt_body_k(Tables t, uint64_t r0, uint64_t r1, uint64_t tile0, const uint64_t *off, const uint64_t *tstart, const uint32_t *hdr,
                           const char *text, uint64_t text0, char *out) {
    __shared__ uint64_t s_r;
    const uint64_t tile = tile0 + blockIdx.x;
    if (threadIdx.x == 0) {
        uint64_t lo = r0, hi = r1;                   // the last record whose first tile is <= tile
        while (hi - lo > 1) {
            const uint64_t mid = lo + (hi - lo) / 2;
            if (tstart[mid] <= tile) lo = mid; else hi = mid;
        }
        s_r = lo;
    }
    __syncthreads();
    const uint64_t r = s_r, c = t.rec[r], i = c >> 1, n = t.len[i];
    const uint64_t body = fmt_body_len(n), q0 = (tile - tstart[r]) * kTile, q1 = min(q0 + kTile, body);
    const char *s = text + (t.eoff[i] - text0);
    char *d = out + (off[r] - off[r0]) + hdr[r];
    for (uint64_t q = q0 + threadIdx.x; q < q1; q += blockDim.x) d[q] = fmt_body_byte(s, n, c & 1, q);
}

template <class T>
void upload(Ctx *ctx, DArr<T> &d, const T *h, size_t n) {
    d.alloc(ctx, n);
    if (n) SG_CUDA(cudaMemcpyAsync(d.p, h, n * sizeof(T), cudaMemcpyHostToDevice, ctx->stream));
}

struct Events {
    cudaEvent_t e[8] = {};
    Events() { for (auto &x : e) SG_CUDA(cudaEventCreate(&x)); }
    ~Events() { for (auto &x : e) if (x) cudaEventDestroy(x); }
};

}  // namespace

uint64_t graph_format(Ctx *ctx, const Graph *g, bool fastg, uint64_t cap, const std::function<void(const char *, size_t)> &sink) {
    FormatStats &st = g->fmt;
    st = FormatStats();
    const size_t E = g->edge_len.size();
    if (E == 0) return 0;
    Trace tr(fastg ? "sgpu fastg" : "sgpu unitigs fasta", ctx->stream);
    const Stopwatch host_clock;
    GraphVertices gv;
    if (fastg) gv = graph_vertices(g, tr, true);
    else gv.selfc.assign(E, 1);                           // one record per edge
    std::vector<uint64_t> rec;
    rec.reserve(2 * E);
    for (size_t i = 0; i < E; ++i) {
        rec.push_back(2 * i);
        if (!gv.selfc[i]) rec.push_back(2 * i + 1);
    }
    const uint64_t R = rec.size();
    if (fastg) {
        for (uint64_t c : rec)
            SG_CHECK(gv.end_slot[c] != ~0ull, 2, "inconsistent link records: an edge end belongs to no vertex");
    } else {
        gv.lst_off.assign(2, 0);
        gv.lst.assign(1, 0);
        gv.end_slot.assign(1, 0);
    }
    for (size_t i = 0; i < E; ++i) SG_CHECK(g->edge_len[i] > (uint32_t)g->k, 2, "an edge shorter than k + 1 bases");
    st.records = R;
    st.vertices_ms = host_clock.ms();

    DArr<uint32_t> d_len, d_raw;
    DArr<uint64_t> d_eoff, d_lst_off, d_lst, d_end, d_rec;
    DArr<uint8_t> d_selfc;
    upload(ctx, d_len, g->edge_len.data(), E);
    upload(ctx, d_raw, g->raw_cov.data(), E);
    upload(ctx, d_eoff, g->edge_off.data(), E);
    upload(ctx, d_selfc, gv.selfc.data(), E);
    upload(ctx, d_lst_off, gv.lst_off.data(), gv.lst_off.size());
    upload(ctx, d_lst, gv.lst.data(), gv.lst.size());
    upload(ctx, d_end, gv.end_slot.data(), gv.end_slot.size());
    upload(ctx, d_rec, rec.data(), R);
    const Tables t{d_len.p, d_raw.p, d_eoff.p, d_selfc.p, d_lst_off.p, d_lst.p, d_end.p, d_rec.p, g->k, fastg};

    DArr<uint32_t> d_hdr;
    DArr<uint64_t> d_size, d_off, d_ntile, d_tstart;
    d_hdr.alloc(ctx, R);
    d_size.alloc(ctx, R + 1);
    d_ntile.alloc(ctx, R + 1);
    SG_CUDA(cudaMemsetAsync(d_size.p + R, 0, 8, ctx->stream));
    SG_CUDA(cudaMemsetAsync(d_ntile.p + R, 0, 8, ctx->stream));
    fmt_size_k<<<div_up((int64_t)R, 256), 256, 0, ctx->stream>>>(t, R, d_hdr.p, d_size.p, d_ntile.p);
    ctx->launches++;
    SG_CUDA(cudaGetLastError());
    d_off.alloc(ctx, R + 1);
    d_tstart.alloc(ctx, R + 1);
    exclusive_scan_u64(ctx, d_size.p, d_off.p, R + 1);
    exclusive_scan_u64(ctx, d_ntile.p, d_tstart.p, R + 1);
    d_size.release();
    d_ntile.release();
    std::vector<uint64_t> off(R + 1), tstart(R + 1);
    SG_CUDA(cudaMemcpyAsync(off.data(), d_off.p, (R + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaMemcpyAsync(tstart.data(), d_tstart.p, (R + 1) * 8, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
    tr.mark("record sizes");
    const uint64_t total = off[R];
    st.bytes = total;
    st.sizes_ms = host_clock.ms() - st.vertices_ms;
    if (total > cap) return total;

    uint64_t largest = 0;
    for (uint64_t r = 0; r < R; ++r) largest = std::max(largest, off[r + 1] - off[r]);
    // two output buffers (one being formatted, one being copied out) and one for the run's edge text, which is never longer than
    // the run's bodies: each takes a third of the memory left, at most kRunCap unless the largest record needs more
    const size_t third = ctx->budget_left() / 3;
    if (third < largest) {
        char m[256];
        snprintf(m, sizeof m, "the device memory left (%zu bytes) holds no three buffers of the largest record (%llu bytes)", ctx->budget_left(),
                 (unsigned long long)largest);
        throw Error(4, m);
    }
    const size_t buf = std::min<size_t>(std::max<size_t>(largest, std::min(third, kRunCap)), total);
    DArr<char> d_out[2], d_text;
    d_out[0].alloc(ctx, buf);
    d_out[1].alloc(ctx, buf);
    d_text.alloc(ctx, buf);
    HostArr<char> h_out[2];
    h_out[0].alloc(buf);
    h_out[1].alloc(buf);
    cudaStream_t cs = ctx->copy_stream();
    Events ev[2];                                         // per buffer: format start/end, copy start/end, copied
    uint64_t run_bytes[2] = {0, 0};
    float write_ms = 0;
    auto drain = [&](int b) {
        SG_CUDA(cudaEventSynchronize(ev[b].e[3]));
        float f = 0, c = 0;
        SG_CUDA(cudaEventElapsedTime(&f, ev[b].e[0], ev[b].e[1]));
        SG_CUDA(cudaEventElapsedTime(&c, ev[b].e[2], ev[b].e[3]));
        st.format_ms += f; st.d2h_ms += c;
        const Stopwatch w;
        sink(h_out[b].p, run_bytes[b]);
        write_ms += w.ms();
    };
    uint64_t r0 = 0;
    int j = 0;
    while (r0 < R) {
        const uint64_t r1 = (uint64_t)(std::upper_bound(off.begin() + r0 + 1, off.end(), off[r0] + buf) - off.begin()) - 1;
        const int b = j & 1;
        const uint64_t e0 = rec[r0] >> 1, e1 = rec[r1 - 1] >> 1;
        const uint64_t text0 = g->edge_off[e0], text_n = g->edge_off[e1] + g->edge_len[e1] - text0;
        SG_CHECK(text_n <= buf, 6, "a run's edge text is longer than its records: edges not laid end to end");
        SG_CUDA(cudaMemcpyAsync(d_text.p, g->seq.data() + text0, text_n, cudaMemcpyHostToDevice, ctx->stream));
        if (j >= 2) SG_CUDA(cudaStreamWaitEvent(ctx->stream, ev[b].e[3], 0));   // the copy out of this buffer's previous run is done
        SG_CUDA(cudaEventRecord(ev[b].e[0], ctx->stream));
        fmt_header_k<<<div_up((int64_t)(r1 - r0), 256), 256, 0, ctx->stream>>>(t, r0, r1, d_off.p, d_out[b].p);
        const uint64_t tiles = tstart[r1] - tstart[r0];
        if (tiles)
            fmt_body_k<<<(unsigned)tiles, 256, 0, ctx->stream>>>(t, r0, r1, tstart[r0], d_off.p, d_tstart.p, d_hdr.p, d_text.p, text0, d_out[b].p);
        ctx->launches += tiles ? 2 : 1;
        SG_CUDA(cudaGetLastError());
        SG_CUDA(cudaEventRecord(ev[b].e[1], ctx->stream));
        SG_CUDA(cudaStreamWaitEvent(cs, ev[b].e[1], 0));
        SG_CUDA(cudaEventRecord(ev[b].e[2], cs));
        run_bytes[b] = off[r1] - off[r0];
        SG_CUDA(cudaMemcpyAsync(h_out[b].p, d_out[b].p, run_bytes[b], cudaMemcpyDeviceToHost, cs));
        SG_CUDA(cudaEventRecord(ev[b].e[3], cs));
        if (j >= 1) drain(b ^ 1);
        r0 = r1;
        ++j;
    }
    drain((j - 1) & 1);
    st.runs = (uint64_t)j;
    st.write_ms = write_ms;
    tr.mark("formatted and written");
    return total;
}

// ---- the coverage text on host and device (tests compare both with printf's "%f") ---------------------------------------------------
namespace {
__global__ void fmt_cov_k(const uint32_t *raw, const uint32_t *den, int64_t n, char *out) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    char *d = out + i * 32;
    d[fmt_cov(d, raw[i], den[i])] = 0;
}
}  // namespace

void format_cov(Ctx *ctx, bool on_device, const uint32_t *raw, const uint32_t *den, int64_t n, char *out) {
    for (int64_t i = 0; i < n; ++i) SG_CHECK(den[i] != 0, 2, "a zero divisor");
    if (!on_device) {
        for (int64_t i = 0; i < n; ++i) out[i * 32 + fmt_cov(out + i * 32, raw[i], den[i])] = 0;
        return;
    }
    if (!n) return;
    DArr<uint32_t> d_raw, d_den;
    DArr<char> d_out;
    upload(ctx, d_raw, raw, (size_t)n);
    upload(ctx, d_den, den, (size_t)n);
    d_out.alloc(ctx, (size_t)n * 32);
    fmt_cov_k<<<div_up(n, 256), 256, 0, ctx->stream>>>(d_raw.p, d_den.p, n, d_out.p);
    ctx->launches++;
    SG_CUDA(cudaGetLastError());
    SG_CUDA(cudaMemcpyAsync(out, d_out.p, (size_t)n * 32, cudaMemcpyDeviceToHost, ctx->stream));
    SG_CUDA(cudaStreamSynchronize(ctx->stream));
}

}  // namespace sg

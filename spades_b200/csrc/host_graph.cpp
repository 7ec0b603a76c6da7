// host_graph.cpp -- graph linking and GFA text on the host (string-heavy, a few million records).
//   FastGraphFromSequencesConstructor::ConstructGraph (src/common/assembly_graph/construction/debruijn_graph_constructor.hpp:506-567)
//   ids: GraphCore ID_BIAS=3 (assembly_graph/core/graph_core.hpp:233), edge i -> 3+2i, conjugate +1 (:514-531), vertex v -> 3+2v (:459-479)
//   PairedVertex::AddOutgoingEdge keeps outgoing edges sorted by id (graph_core.hpp:206-209)
//   GFAWriter::WriteSegments / WriteLinks / WriteVertexLinks (src/common/io/graph/gfa_writer.cpp:19-116)
// Inputs are the per-edge link records and raw coverages computed on the GPU (graph.cu).
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <string>
#include <thread>
#include <vector>

#include "graph.h"
#include "host_par.h"

namespace sg {

namespace {
struct Rec {
    uint64_t hm;     // hash_and_mask_
    uint64_t edge;   // EdgeId
    uint64_t edge_and_mask() const { return (edge << 2) | (hm & 3); }
};
const uint64_t kMinId = 3;

inline void put_u(std::string &s, uint64_t v) {
    char tmp[24];
    int n = 0;
    do { tmp[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    while (n) s.push_back(tmp[--n]);
}

}  // namespace

GraphVertices graph_vertices(const Graph *g, Trace &tr, bool end_slots) {
    const size_t E = g->edge_len.size();
    GraphVertices gv;
    std::vector<uint8_t> &selfc = gv.selfc;
    selfc.assign(E ? E : 1, 0);
    raw_vector<Rec> recs(2 * E);
    par_chunks(E, host_threads_for(E), [&](int, size_t lo, size_t hi) {
        for (size_t i = lo; i < hi; ++i) {
            const uint64_t e = kMinId + 2 * i;
            recs[2 * i] = Rec{g->link_start[i], e};
            if (g->link_end[i] == ~0ull) { selfc[i] = 1; recs[2 * i + 1] = Rec{~0ull, 0}; }      // LinkRecord() of a self-conjugate edge
            else recs[2 * i + 1] = Rec{g->link_end[i], e};
        }
    });
    par_sort(recs, [](const Rec &a, const Rec &b) {                                        // CompareByVertexKMerEdgeIdAndMask
        const uint64_t ha = a.hm >> 2, hb = b.hm >> 2;
        if (ha != hb) return ha < hb;
        return a.edge_and_mask() < b.edge_and_mask();
    });
    tr.mark("link records sorted");
    // a vertex = a run of records with one k-mer index; the placeholder records of self-conjugate edges form no vertex
    auto group_start = [&](size_t i) {
        if (i != 0 && (recs[i].hm >> 2) == (recs[i - 1].hm >> 2)) return false;
        return !((recs[i].hm + 1 == 0) && recs[i].edge == 0);
    };
    raw_vector<size_t> groups;
    {
        const int TG = host_threads_for(recs.size());
        std::vector<size_t> cnt((size_t)TG + 1, 0);
        par_chunks(recs.size(), TG, [&](int c, size_t lo, size_t hi) {
            size_t n = 0;
            for (size_t i = lo; i < hi; ++i) n += group_start(i);
            cnt[(size_t)c + 1] = n;
        });
        for (int c = 0; c < TG; ++c) cnt[(size_t)c + 1] += cnt[(size_t)c];
        groups.resize(cnt[(size_t)TG]);
        par_chunks(recs.size(), TG, [&](int c, size_t lo, size_t hi) {
            size_t o = cnt[(size_t)c];
            for (size_t i = lo; i < hi; ++i) if (group_start(i)) groups[o++] = i;
        });
    }
    {
        // vertex order = order of the first record's (edge, mask): sort (key, group) pairs so that the compare touches no other array
        struct KG { uint64_t key; size_t grp; };
        raw_vector<KG> kg(groups.size());
        par_chunks(groups.size(), host_threads_for(groups.size()), [&](int, size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) kg[i] = KG{recs[groups[i]].edge_and_mask(), groups[i]};
        });
        par_sort(kg, [](const KG &a, const KG &b) { return a.key < b.key; });
        par_chunks(groups.size(), host_threads_for(groups.size()), [&](int, size_t lo, size_t hi) {
            for (size_t i = lo; i < hi; ++i) groups[i] = kg[i].grp;
        });
    }
    const size_t V = groups.size();
    gv.V = V;
    // outgoing edge lists of vertex v (slot 2v) and of its conjugate (slot 2v+1), CSR: a vertex group has at most 8 records
    std::vector<uint64_t> &lst_off = gv.lst_off;
    lst_off.assign(2 * V + 1, 0);
    const int TV = host_threads_for(V);
    par_chunks(V, TV, [&](int, size_t lo, size_t hi) {
        for (size_t vn = lo; vn < hi; ++vn) {
            const size_t i = groups[vn];
            uint64_t c0 = 0, c1 = 0;
            for (size_t j = i; j < recs.size() && (recs[j].hm >> 2) == (recs[i].hm >> 2); ++j) {
                const bool is_start = recs[j].hm & 1, is_rc = recs[j].hm & 2;
                const int side = (is_rc ? 1 : 0) ^ (is_start ? 0 : 1);
                if (side) ++c1; else ++c0;
            }
            lst_off[2 * vn + 1] = c0; lst_off[2 * vn + 2] = c1;
        }
    });
    for (size_t i = 1; i <= 2 * V; ++i) lst_off[i] += lst_off[i - 1];
    raw_vector<uint64_t> &lst = gv.lst;
    lst.resize(lst_off[2 * V] + 1);
    if (end_slots) gv.end_slot.assign(2 * E, ~0ull);
    par_chunks(V, TV, [&](int, size_t lo, size_t hi) {
        for (size_t vn = lo; vn < hi; ++vn) {
            const size_t i = groups[vn];
            uint64_t p0 = lst_off[2 * vn], p1 = lst_off[2 * vn + 1];
            for (size_t j = i; j < recs.size() && (recs[j].hm >> 2) == (recs[i].hm >> 2); ++j) {
                const bool is_start = recs[j].hm & 1, is_rc = recs[j].hm & 2;
                const uint64_t e = recs[j].edge;
                const size_t ei = (size_t)((e - kMinId) / 2);
                const uint64_t ce = selfc[ei] ? e : e + 1;
                const int side = is_rc ? 1 : 0;                                     // LinkEdge: v1 = is_rc ? conjugate(v) : v
                // LinkOutgoingEdge(v1, e)  /  LinkIncomingEdge(v1, e): cvertex(v1) gets conjugate(e)
                const int slot = is_start ? side : (side ^ 1);
                const uint64_t val = is_start ? e : ce;
                if (slot) lst[p1++] = val; else lst[p0++] = val;
                // the end vertex of e is v1 when this record is e's end; when it is e's start, the end of conjugate(e) is conjugate(v1)
                if (!end_slots) continue;
                if (!is_start) gv.end_slot[2 * ei] = 2 * vn + side;
                else gv.end_slot[2 * ei + (selfc[ei] ? 0 : 1)] = 2 * vn + (side ^ 1);
            }
            std::sort(lst.begin() + lst_off[2 * vn], lst.begin() + lst_off[2 * vn + 1]);
            std::sort(lst.begin() + lst_off[2 * vn + 1], lst.begin() + lst_off[2 * vn + 2]);
        }
    });
    tr.mark("vertices + edge lists");
    return gv;
}

std::vector<std::string> graph_gfa_chunks(const Graph *g, const char *version) {
    const size_t E = g->edge_len.size();
    const int K = g->k;
    Trace tr("sgpu gfa");
    const GraphVertices gv = graph_vertices(g, tr, false);
    const std::vector<uint8_t> &selfc = gv.selfc;
    const std::vector<uint64_t> &lst_off = gv.lst_off;
    const raw_vector<uint64_t> &lst = gv.lst;
    const size_t V = gv.V;
    const int TV = host_threads_for(V);
    const int TE = host_threads_for(E);
    std::vector<std::string> chunks(1 + (size_t)TE + (size_t)TV);
    chunks[0] = std::string("H\tsp:Z:") + version + "\n";
    par_chunks(E, TE, [&](int c, size_t lo, size_t hi) {
        std::string &t = chunks[1 + (size_t)c];
        size_t bases = 0;
        for (size_t i = lo; i < hi; ++i) bases += g->edge_len[i];
        t.reserve(bases + 64 * (hi - lo) + 64);
        for (size_t i = lo; i < hi; ++i) {
            t += "S\t"; put_u(t, kMinId + 2 * i); t += "\t";
            t.append(g->seq, g->edge_off[i], g->edge_len[i]);
            const uint32_t raw = g->raw_cov[i];
            const double cv = (double)raw / (double)(g->edge_len[i] - K);          // CoverageIndex::coverage, core/coverage.hpp:59-61
            char tmp[64];
            int n = snprintf(tmp, sizeof tmp, "\tDP:f:%g\tKC:i:%u\n", (double)(float)cv, raw);   // `os << float(cov)`, gfa_writer.cpp:24
            t.append(tmp, n);
        }
    });
    char ktail[32];
    const int ktail_n = snprintf(ktail, sizeof ktail, "\t%dM\n", K);
    par_chunks(V, TV, [&](int c, size_t lo, size_t hi) {
        std::string &t = chunks[1 + (size_t)TE + (size_t)c];
        t.reserve(40 * (hi - lo) * 2 + 64);
        for (size_t vn = lo; vn < hi; ++vn) {
            for (uint64_t a = lst_off[2 * vn + 1]; a < lst_off[2 * vn + 2]; ++a) {   // IncomingEdges(v) = conjugates of OutgoingEdges(conj v)
                const uint64_t x = lst[a];
                const size_t xi = (size_t)((x - kMinId) / 2);
                const uint64_t inc = selfc[xi] ? x : (((x - kMinId) & 1) ? x - 1 : x + 1);
                for (uint64_t b = lst_off[2 * vn]; b < lst_off[2 * vn + 1]; ++b) {
                    const uint64_t ends[2] = {inc, lst[b]};
                    t += "L";
                    for (int q = 0; q < 2; ++q) {
                        const uint64_t e = ends[q];
                        const size_t ei = (size_t)((e - kMinId) / 2);
                        const bool canon = selfc[ei] || (((e - kMinId) & 1) == 0);
                        t += "\t"; put_u(t, kMinId + 2 * ei); t += canon ? "\t+" : "\t-";
                    }
                    t.append(ktail, ktail_n);
                }
            }
        }
    });
    tr.mark("S and L lines");
    return chunks;
}

std::string graph_gfa(const Graph *g, const char *version) {
    std::vector<std::string> ch = graph_gfa_chunks(g, version);
    size_t total = 0;
    for (const auto &c : ch) total += c.size();
    std::string t;
    t.reserve(total);
    for (auto &c : ch) { t += c; std::string().swap(c); }
    return t;
}

}  // namespace sg

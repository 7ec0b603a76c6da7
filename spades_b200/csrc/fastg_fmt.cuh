// fastg_fmt.cuh -- the text pieces of the FASTG and unitig FASTA records, for the device formatter (fastg.cu) and its host tests.
//   FastgWriter::WriteSegmentsAndLinks (src/common/io/graph/fastg_writer.cpp:21-46), BasicNamingF + CanonicalEdgeHelper
//   (io/utils/edge_namer.hpp:31-35,56-93), MakeContigId (io/reads/header_naming.hpp:23-25), WriteWrapped (io/reads/osequencestream.hpp:24-30)
#pragma once
#include <stdint.h>

namespace sg {

static const int kWrap = 60;            // bases per body line
static const int kCovChars = 24;        // the longest cov text: 10 integer digits, '.', 6 digits
static const int kNameChars = 80;       // "EDGE_" u64 "_length_" u32 "_cov_" cov "'"
static const int kMaxSucc = 4;          // outgoing edges of a vertex

// body bytes of an edge of n bases: n bases plus a '\n' after every 60 of them and after the last partial line
__host__ __device__ inline uint64_t fmt_body_len(uint64_t n) { return n + (n + kWrap - 1) / kWrap; }

__host__ __device__ inline int fmt_u64(char *d, uint64_t v) {
    char t[20];
    int n = 0;
    do { t[n++] = (char)('0' + v % 10); v /= 10; } while (v);
    for (int i = 0; i < n; ++i) d[i] = t[n - 1 - i];
    return n;
}

// std::to_string(raw / den) for raw < 2^32 and 1 <= den < 2^32: printf's "%f", exact. v = m 2^-s with m < 2^53; since v < 2^32 and
// v >= 2^-32, 21 <= s <= 84, so m 10^6 < 2^73 fits 128 bits; it is shifted right by s and rounded half to even on the exact remainder.
__host__ __device__ inline int fmt_cov(char *d, uint32_t raw, uint32_t den) {
    const double v = (double)raw / (double)den;
    uint64_t ip = 0;
    uint32_t fr = 0;
    if (raw) {
        union { double f; uint64_t u; } b;
        b.f = v;
        const int ex = (int)((b.u >> 52) & 0x7ff);
        const uint64_t m = (b.u & ((1ull << 52) - 1)) | (1ull << 52);
        const int s = 1075 - ex;
        const unsigned __int128 x = (unsigned __int128)m * 1000000u;
        unsigned __int128 q = x >> s;
        const unsigned __int128 rem = x - (q << s), half = (unsigned __int128)1 << (s - 1);
        if (rem > half || (rem == half && (q & 1))) ++q;
        ip = (uint64_t)(q / 1000000u);
        fr = (uint32_t)(q % 1000000u);
    }
    int n = fmt_u64(d, ip);
    d[n++] = '.';
    for (int i = 5; i >= 0; --i) { d[n + i] = (char)('0' + fr % 10); fr /= 10; }
    return n + 6;
}

// name(e) of the edge with GFA id x (3 + 2i, or 4 + 2i for the conjugate of a non-self-conjugate edge i)
__host__ __device__ inline int fmt_edge_name(char *d, uint64_t x, const uint32_t *len, const uint32_t *raw, const uint8_t *selfc, int k) {
    const uint64_t i = (x - 3) / 2;
    const bool canon = selfc[i] || ((x - 3) & 1) == 0;
    const char *p0 = "EDGE_", *p1 = "_length_", *p2 = "_cov_";
    int n = 0;
    for (const char *p = p0; *p; ++p) d[n++] = *p;
    n += fmt_u64(d + n, 3 + 2 * i);
    for (const char *p = p1; *p; ++p) d[n++] = *p;
    n += fmt_u64(d + n, len[i]);
    for (const char *p = p2; *p; ++p) d[n++] = *p;
    n += fmt_cov(d + n, raw[i], len[i] - (uint32_t)k);
    if (!canon) d[n++] = '\'';
    return n;
}

__host__ __device__ inline int fmt_cmp(const char *a, int na, const char *b, int nb) {
    const int n = na < nb ? na : nb;
    for (int i = 0; i < n; ++i)
        if (a[i] != b[i]) return (unsigned char)a[i] < (unsigned char)b[i] ? -1 : 1;
    return na < nb ? -1 : (na > nb ? 1 : 0);
}

// The FASTG header of the edge with GFA id x, whose end vertex has the outgoing edges succ[0..ns): '>' name [':' names in byte
// order, duplicates once, ','-separated] ";\n". Writes to d when d is not null; returns its length either way.
__host__ __device__ inline int fmt_fastg_header(char *d, uint64_t x, const uint64_t *succ, int ns, const uint32_t *len, const uint32_t *raw,
                                                const uint8_t *selfc, int k) {
    char nm[kMaxSucc][kNameChars];
    int nl[kMaxSucc], ord[kMaxSucc];
    for (int j = 0; j < ns; ++j) {
        nl[j] = fmt_edge_name(nm[j], succ[j], len, raw, selfc, k);
        int p = j;                                           // insertion sort of the names (std::set<std::string>)
        while (p > 0 && fmt_cmp(nm[ord[p - 1]], nl[ord[p - 1]], nm[j], nl[j]) > 0) { ord[p] = ord[p - 1]; --p; }
        ord[p] = j;
    }
    char own[kNameChars];
    const int no = fmt_edge_name(own, x, len, raw, selfc, k);
    int n = 1 + no;
    if (d) { d[0] = '>'; for (int i = 0; i < no; ++i) d[1 + i] = own[i]; }
    for (int j = 0; j < ns; ++j) {
        const int a = ord[j];
        if (j > 0 && fmt_cmp(nm[ord[j - 1]], nl[ord[j - 1]], nm[a], nl[a]) == 0) continue;
        if (d) { d[n] = j == 0 ? ':' : ','; for (int i = 0; i < nl[a]; ++i) d[n + 1 + i] = nm[a][i]; }
        n += 1 + nl[a];
    }
    if (d) { d[n] = ';'; d[n + 1] = '\n'; }
    return n + 2;
}

// gbuilder's unitig header: ">EDGE_<index + 1>_length_<bases>\n"
__host__ __device__ inline int fmt_unitig_header(char *d, uint64_t i, uint32_t bases) {
    char t[64];
    const char *p0 = ">EDGE_", *p1 = "_length_";
    int n = 0;
    for (const char *p = p0; *p; ++p) t[n++] = *p;
    n += fmt_u64(t + n, i + 1);
    for (const char *p = p1; *p; ++p) t[n++] = *p;
    n += fmt_u64(t + n, bases);
    t[n++] = '\n';
    if (d) for (int j = 0; j < n; ++j) d[j] = t[j];
    return n;
}

__host__ __device__ inline char fmt_complement(char c) {
    switch (c) { case 'A': return 'T'; case 'C': return 'G'; case 'G': return 'C'; case 'T': return 'A'; default: return 'N'; }
}

// byte q of the wrapped body of the n bases at s (reverse complement when rc)
__host__ __device__ inline char fmt_body_byte(const char *s, uint64_t n, bool rc, uint64_t q) {
    const uint64_t line = q / (kWrap + 1), col = q % (kWrap + 1), b = line * kWrap + col;
    if (col == kWrap || b == n) return '\n';
    return rc ? fmt_complement(s[n - 1 - b]) : s[b];
}

}  // namespace sg

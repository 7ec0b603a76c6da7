"""FASTG and unitig FASTA restated from a GFA text, independently of the device formatter.

io::FastgWriter::WriteSegmentsAndLinks (io/graph/fastg_writer.cpp:21-46) writes, for every edge in id order (3 + 2i, then its
conjugate 4 + 2i unless the edge is self-conjugate), '>' name(e), then ':' and the names of the end vertex's outgoing edges from a
std::set<std::string> joined by ',', then ';', and the sequence wrapped at 60. name(e) = EDGE_<3+2i>_length_<bases>_cov_<%f of
raw / (bases - k)>, with "'" on a non-canonical edge. The GFA (GFAWriter) has every edge as an S line in id order with its raw
coverage (KC) and every pair (incoming, outgoing) of a vertex as an L line, which is all FASTG needs: the outgoing edges of the end
of x are the b of every "L x b" and the conjugate of the a of every "L a conj(x)". An edge is self-conjugate exactly when its
sequence is its own reverse complement.
"""

_COMP = str.maketrans("ACGT", "TGCA")


def revcomp(s):
    return s.translate(_COMP)[::-1]


def wrapped(seq, width=60):
    return "".join(seq[i:i + width] + "\n" for i in range(0, len(seq), width))


def cov_text(raw, den):
    """std::to_string(double(raw) / den): printf's %f, which Python's % reproduces exactly (correctly rounded, ties to even)"""
    return "%f" % (raw / den)


def fastg_from_gfa(gfa, k, with_coverage=True):
    segs, links = [], []
    for line in gfa.split("\n"):
        f = line.split("\t")
        if f[0] == "S":
            kc = [x for x in f[3:] if x.startswith("KC:i:")]
            segs.append((int(f[1]), f[2], int(kc[0][5:]) if kc else 0))
        elif f[0] == "L":
            links.append(((int(f[1]), f[2]), (int(f[3]), f[4])))
    info = {sid: (seq, raw, seq == revcomp(seq)) for sid, seq, raw in segs}

    def norm(o):
        return (o[0], "+") if info[o[0]][2] else o

    def flip(o):
        return norm((o[0], "-" if o[1] == "+" else "+"))

    def name(o):
        seq, raw, _ = info[o[0]]
        c = cov_text(raw if with_coverage else 0, len(seq) - k)
        return "EDGE_%d_length_%d_cov_%s%s" % (o[0], len(seq), c, "'" if o[1] == "-" else "")

    succ = {}
    for a, b in links:
        a, b = norm(a), norm(b)
        succ.setdefault(a, set()).add(b)
        succ.setdefault(flip(b), set()).add(flip(a))
    out = []
    for sid, seq, _ in segs:
        recs = [((sid, "+"), seq)]
        if not info[sid][2]:
            recs.append(((sid, "-"), revcomp(seq)))
        for o, s in recs:
            nxt = sorted({name(x) for x in succ.get(o, ())})
            out.append(">" + name(o) + (":" + ",".join(nxt) if nxt else "") + ";\n" + wrapped(s))
    return "".join(out)


def unitigs_fasta(seqs):
    """spades-gbuilder's unitig output (gbuilder.cpp:191-200)"""
    return "".join(">EDGE_%d_length_%d\n%s" % (i + 1, len(s), wrapped(s)) for i, s in enumerate(seqs))

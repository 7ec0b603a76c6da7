"""Generates tests/golden/*_fastg.npz: the reference's own FASTG and unitig FASTA for the reads of existing graph fixtures.

spades_gbuilder_gpu --fastg (integration/, compiled against the unmodified reference) builds the reference's graph over the GPU's
arrays and writes it with the reference's io::FastgWriter before (graph_nocov_ref.fastg) and after (graph_ref.fastg) the coverage
fill, and the reference's unitigs with gbuilder's loop (unitigs_ref.fasta). It needs a GPU and the tool built where the reference is:
    python -c "import __graft_entry__ as g; g.build()"     # with the reference present
    python tests/golden/make_golden_fastg.py [OUTDIR]      # on a GPU machine; default OUTDIR is tests/golden
Each fixture holds the reads, k, B, the early tip clipper's bound and the three texts.
"""
import os
import subprocess
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
TOOL = os.path.join(ROOT, "integration", "_build", "spades_gbuilder_gpu")

# one to four words, ids >= 10, self-conjugate edges, perfect loops, up to four successors, a tip-clipped graph
SOURCES = ["ecoli_k21_B40_graph", "ecoli_k55_B16_graph", "dense_k3_B1_graph", "pal_k21_B20_eigraph", "loops_k21_B10_graph",
           "syn_k127_B20_eigraph", "syn_k21_B10_tcgraph"]


def main():
    out_dir = sys.argv[1] if len(sys.argv) > 1 else HERE
    for src in SOURCES:
        z = np.load(os.path.join(HERE, src + ".npz"))
        k, B = int(z["k"][0]), int(z["B"][0])
        tc = int(z["tc_bound"][0]) if "tc_bound" in z.files else 0
        reads = z["reads"].tobytes().decode().split("\n")
        with tempfile.TemporaryDirectory() as d:
            rf = os.path.join(d, "reads.txt")
            with open(rf, "w") as f:
                f.write("\n".join(r for r in reads if r) + "\n")
            w = os.path.join(d, "w")
            p = subprocess.run([TOOL, rf, str(k), w, str(B), str(tc), "--fastg"], capture_output=True, text=True)
            if p.returncode != 0:
                sys.exit("%s: the tool failed (%d)\n%s" % (src, p.returncode, (p.stdout + p.stderr)[-3000:]))
            texts = {}
            for key, fn in (("fastg", "graph_ref.fastg"), ("fastg_nocov", "graph_nocov_ref.fastg"), ("unitigs_fasta", "unitigs_ref.fasta")):
                with open(os.path.join(w, fn), "rb") as f:
                    texts[key] = np.frombuffer(f.read(), np.uint8)
        name = src.rsplit("_", 1)[0] + ("_tc" if tc else "") + "_fastg"
        np.savez_compressed(os.path.join(out_dir, name + ".npz"), reads=z["reads"], k=np.array([k]), B=np.array([B]), tc_bound=np.array([tc]),
                            mode=np.frombuffer(b"fastg", np.uint8), source=np.frombuffer(src.encode(), np.uint8), **texts)
        print(name, {key: len(v) for key, v in texts.items()}, flush=True)


if __name__ == "__main__":
    main()

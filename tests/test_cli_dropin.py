"""Drop-in proof at the reference's own CLI level (CPU; needs the reference package __graft_entry__.build() installs under
oracle/_ref/install, which travels with the built tree):
the UNMODIFIED reference `CRISPResso` main() is run twice on the same FASTQ, once as it is and once with its
module-global `process_fastq` re-bound to crispresso2_b200.core.process_fastq (kernel logic on the CPU warp
emulator build of the engine).  Every file the run writes -- allele frequency table, modification count vectors,
nucleotide tables, quantification, mapping statistics, allele tables around the cut, ... (SURVEY.md Appendix B)
-- must be byte-identical, and the engine's own count block must equal the vectors the reference's
quantification loop built."""
import gzip
import hashlib
import json
import os
import subprocess
import sys
import zipfile

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "install", "CRISPResso2", "CRISPRessoCORE.py"))
pytestmark = pytest.mark.skipif(not HAVE_REF, reason="needs oracle/_ref/install (built by __graft_entry__.build())")

sys.path.insert(0, os.path.join(HERE, "emu"))

VOLATILE = ("CRISPResso_RUNNING_LOG.txt", "CRISPResso2_info.json", "CRISPResso_status.json")


def _run(mode, lib, outdir, argv):
    vec = os.path.join(outdir, "_vectors.json")
    os.makedirs(outdir, exist_ok=True)
    p = subprocess.run([sys.executable, os.path.join(HERE, "cli_dropin_runner.py"), mode, lib, outdir, vec, "--"] + argv,
                       capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-3000:]
    with open(vec) as fh:
        return json.load(fh)


def _snapshot(outdir):
    runs = [d for d in os.listdir(outdir) if d.startswith("CRISPResso_on_")]
    assert len(runs) == 1, runs
    rd = os.path.join(outdir, runs[0])
    snap = {}
    for base, _, files in os.walk(rd):
        for f in files:
            if f in VOLATILE:
                continue
            path = os.path.join(base, f)
            rel = os.path.relpath(path, rd)
            if f.endswith(".zip"):
                with zipfile.ZipFile(path) as z:
                    for n in z.namelist():
                        snap[rel + "!" + n] = hashlib.sha256(z.read(n)).hexdigest()
            elif f.endswith(".gz"):                           # gzip headers carry a timestamp
                try:
                    with gzip.open(path, "rb") as fh:
                        snap[rel] = hashlib.sha256(fh.read()).hexdigest()
                except gzip.BadGzipFile:                      # the paired --fastq_output file: named .gz, written as text (:1542)
                    with open(path, "rb") as fh:
                        snap[rel] = hashlib.sha256(fh.read()).hexdigest()
            else:
                with open(path, "rb") as fh:
                    snap[rel] = hashlib.sha256(fh.read()).hexdigest()
    return snap


def _info_stats(outdir):
    runs = [d for d in os.listdir(outdir) if d.startswith("CRISPResso_on_")]
    with open(os.path.join(outdir, runs[0], "CRISPResso2_info.json")) as fh:
        info = json.load(fh)
    return info["results"]["alignment_stats"]


def _cases(tmp=None):
    with open(os.path.join(HERE, "golden", "gen_golden.py")) as fh:
        src = fh.read()
    ns = {}
    for name in ("FANC", "FANC_HDR"):                         # the two amplicon constants, without importing the shim
        start = src.index(name + " = (")
        end = src.index(")\n", start) + 1
        exec(src[start:end], ns)
    fq = ""
    if tmp is not None:                                       # the reference's test FASTQ, stored as a fixture
        import pe_case
        fq = os.path.join(str(tmp), "FANC.Cas9.fastq")
        with open(fq, "w") as fh:
            fh.write(pe_case.fanc_fastq_text())
    g = "GGAATCCCTTCTGCAGCACC"
    pe = []
    if tmp is not None:
        pe_fq = os.path.join(str(tmp), "pe_scaffold.fastq")
        import pe_case
        ext, scaffold = pe_case.write_fastq(pe_fq, ns["FANC"])
        pe = ["-r1", pe_fq, "-a", ns["FANC"], "--prime_editing_pegRNA_spacer_seq", g, "--prime_editing_pegRNA_extension_seq", ext,
              "--prime_editing_pegRNA_scaffold_seq", scaffold, "--write_detailed_allele_table"]
    paired = []
    if tmp is not None:
        import pe_case
        r1, r2 = os.path.join(str(tmp), "pairs_R1.fastq"), os.path.join(str(tmp), "pairs_R2.fastq")
        pe_case.write_pairs(r1, r2, ns["FANC"])
        paired = ["-r1", r1, "-r2", r2, "-a", ns["FANC"], "-g", g, "--crispresso_merge",
                  "--fastp_command", sys.executable + " " + os.path.join(HERE, "fake_fastp.py")]
    panel, names = allele_panel(ns["FANC"])
    F = ns["FANC"]
    win_fq, hdr_win = "", F[:118] + "TC" + F[118:128] + F[133:]          # 2-bp insertion inside 110-125, 128-132 deleted
    if tmp is not None:
        win_fq = window_fastq(os.path.join(str(tmp), "window_edges.fastq"), F)
    g2 = F[150:170]
    amas = ["-amas", "60,70,65,80,75"]
    return {
        # five allele amplicons plus -e: six references per read, the one-kernel form of the general kernel
        "fanc_panel": ["-r1", fq, "-a", ",".join(panel), "-an", ",".join(names), "-g", g, "-e", ns["FANC_HDR"],
                       "--expand_ambiguous_alignments"] + amas,
        "fanc_panel_fastq_output": ["-r1", fq, "-a", ",".join(panel), "-an", ",".join(names), "-g", g, "-e", ns["FANC_HDR"],
                                    "--fastq_output"] + amas,
        # the coding sequence lies in three of the five alleles: the other two carry a SNP inside it
        "fanc_panel_coding": ["-r1", fq, "-a", ",".join(panel), "-an", ",".join(names), "-g", g,
                              "-c", "GGGCCTTCGCGCACCTCATGGAATCCCTTCTGCAGCACCTGGATCGCTTTT"],
        # SURVEY 8(f) rank 3: --crispresso_merge, process_paired_fastq over one batch of GPU alignments (crispresso2_b200/paired.py)
        "fanc_paired_merge": paired,
        # (with -e the reference's own HDR re-projection fails on the paired entries' five-element ref_aln_details, :4243)
        "fanc_paired_merge_out": paired + ["--fastq_output", "--expand_ambiguous_alignments", "-w", "3"],
        # CRISPRessoCORE.py:789-796: reads with the pegRNA scaffold after the extension move to 'Scaffold-incorporated'
        "fanc_pe_scaffold": pe,
        "fanc_pe_scaffold_discard": pe + ["--discard_indel_reads", "--expand_ambiguous_alignments"],
        "fanc_default": ["-r1", fq, "-a", ns["FANC"], "-g", g, "--write_detailed_allele_table"],
        "fanc_params": ["-r1", fq, "-a", ns["FANC"], "-g", g, "-e", ns["FANC_HDR"],
                        "-c", "GGGCCTTCGCGCACCTCATGGAATCCCTTCTGCAGCACCTGGATCGCTTTT", "--dump", "-qwc", "20-30_45-50",
                        "-q", "30", "--default_min_aln_score", "80", "-an", "FANC", "-n", "params", "--base_editor_output",
                        "-fg", "AGCCTTGCAGTGGGCGCGCTA,CCCACTGAAGGCCC", "--dsODN", "GCTAGATTTCCCAAGAAGA", "-gn", "hi",
                        "-fgn", "dear"],
        "fanc_flags": ["-r1", fq, "-a", ns["FANC"], "-g", g, "--ignore_substitutions", "--discard_indel_reads",
                       "-w", "10", "--exclude_bp_from_left", "5"],
        # SURVEY 8(f) rank 4: process_fastq_write_out (CRISPRessoCORE.py:2283-2348) wraps the module-global process_fastq and
        # annotates every FASTQ record from variantCache / not_aligned -- with the engine's lazy entries behind it
        "fanc_fastq_output": ["-r1", fq, "-a", ns["FANC"], "-g", g, "-e", ns["FANC_HDR"], "--fastq_output"],
        "fanc_legacy": ["-r1", fq, "-a", ns["FANC"], "-g", g, "-e", ns["FANC_HDR"], "--use_legacy_insertion_quantification", "-w", "4"],
        # scoring options: an asymmetric NCBI-format matrix (tests/golden/scoring_nuc.matrix), gap_open == gap_extend, incentive 3
        "fanc_scoring": ["-r1", fq, "-a", ns["FANC"], "-g", g] + SCORING_ARGS,
        # quantification windows (tests/test_window_space.py), reads with edits on every run edge: two guides, one with no
        # window of its own (-w 5,0) and per-guide centres; three -qwc runs touching both ends, under legacy; -w 0; and -e
        # with an HDR amplicon whose indels lie inside -qwc runs, so its cloned window differs from reference 0's
        "window_two_guides": ["-r1", win_fq, "-a", F, "-g", g + "," + g2, "-w", "5,0", "--quantification_window_center=-3,-8"],
        "window_qwc_ends_legacy": ["-r1", win_fq, "-a", F, "-g", g, "-qwc", "0-9_40-60_213-222", "--exclude_bp_from_left", "0",
                                   "--exclude_bp_from_right", "0", "--use_legacy_insertion_quantification"],
        "window_w0": ["-r1", win_fq, "-a", F, "-g", g, "-w", "0"],
        "window_cloned_hdr": ["-r1", win_fq, "-a", F, "-g", g, "-e", hdr_win, "-qwc", "110-125_128-132"],
    }


def window_fastq(path, fanc):
    """the first 120 FANC reads, and reads with edits planted on the run edges of the windows of the window_* cases"""
    import numpy as np
    import pe_case
    import test_window_space as WS
    lines = pe_case.fanc_fastq_text().split("\n")
    reads = [lines[k + 1] for k in range(0, len(lines) - 3, 4)][:120]
    rng = np.random.default_rng(223)
    for runs in ([(0, 9), (40, 60), (213, 222)], [(88, 97), (159, 168)], [(15, 207)], [(110, 125), (128, 132)]):
        reads += WS.edge_reads(rng, fanc, runs)
    with open(path, "w") as fh:
        fh.write("".join("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)) for k, s in enumerate(reads)))
    return path


def allele_panel(fanc):
    """five alleles of the FANC amplicon: itself and one SNP each at positions 30, 150, 60 and 100 (the last two inside the
    coding sequence 56-107 of the fanc_params case, outside the guide 75-95) -> (sequences, names)"""
    out = [fanc]
    for p in (30, 150, 60, 100):
        out.append(fanc[:p] + ("A" if fanc[p] != "A" else "C") + fanc[p + 1:])
    return out, ["FANC", "SNP30", "SNP150", "SNP60", "SNP100"]


SCORING_ARGS = ["--needleman_wunsch_aln_matrix_loc", os.path.join(HERE, "golden", "scoring_nuc.matrix"),
                "--needleman_wunsch_gap_open", "-6", "--needleman_wunsch_gap_extend", "-6", "--needleman_wunsch_gap_incentive", "3"]


@pytest.mark.parametrize("case", ["fanc_default", "fanc_params", "fanc_flags", "fanc_fastq_output", "fanc_legacy", "fanc_pe_scaffold",
                                  "fanc_pe_scaffold_discard", "fanc_paired_merge", "fanc_paired_merge_out", "fanc_scoring",
                                  "fanc_panel", "fanc_panel_fastq_output", "fanc_panel_coding", "window_two_guides",
                                  "window_qwc_ends_legacy", "window_w0", "window_cloned_hdr"])
def test_reference_cli_with_engine_process_fastq_is_byte_identical(case, tmp_path):
    import build_emu
    lib = build_emu.build()
    argv = _cases(tmp_path)[case]
    ref_dir, b200_dir = str(tmp_path / "ref"), str(tmp_path / "b200")
    _run("reference", "default", ref_dir, argv)
    rep = _run("b200", lib, b200_dir, argv)
    a, b = _snapshot(ref_dir), _snapshot(b200_dir)
    assert sorted(a) == sorted(b)
    diff = [k for k in a if a[k] != b[k]]
    assert not diff, diff
    assert len(a) >= 10
    assert _info_stats(ref_dir) == _info_stats(b200_dir)
    if "--crispresso_merge" in argv:                          # every global_align of the reference's loop came out of the GPU batch
        assert rep["memo"]["hits"] > 100 and rep["memo"]["misses"] == 0, rep["memo"]
    else:
        assert rep["checked"] > 20 and not rep["mismatch"], rep["mismatch"]

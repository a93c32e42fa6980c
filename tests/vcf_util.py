"""Shared by tests/test_vcf.py (warp emulator) and tests/test_gpu_vcf.py (sm_90a): the reference's own build_edit_counts
(writers/vcf.py of the package under oracle/_ref/install), the frames both are compared on, and the comparison: the same dict
in the same key order with int / str items, or the same exception type and message."""
import importlib
import os
import sys
import tempfile

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "install", "CRISPResso2", "writers", "vcf.py"))


def reference_vcf():
    from baseline import ref_shim
    ref_shim.load_core()
    return importlib.import_module("CRISPResso2.writers.vcf")


def _outcome(fn):
    try:
        return "ok", fn()
    except Exception as ex:                                     # noqa: BLE001 -- the exception is the result compared
        return type(ex), str(ex)


def check(df, amplicon_positions, engine, chunk=0):
    """the drop-in against the reference on one frame -> the reference's outcome"""
    from crispresso2_b200 import vcf
    want = _outcome(lambda: reference_vcf().build_edit_counts(df, amplicon_positions))
    got = _outcome(lambda: vcf.build_edit_counts(df, amplicon_positions, engine=engine, chunk=chunk))
    assert got[0] == want[0], (got, want)
    if want[0] == "ok":
        assert got[1] == want[1]
        assert list(got[1]) == list(want[1])
        assert all(type(v) is int for v in got[1].values())
        assert all(type(p) is int and type(r) is str and type(a) is str for _, p, r, a in got[1])
    else:
        assert got[1] == want[1], (got, want)
    return want


def ref_positions(aln_ref):
    """CRISPRessoCOREResources.pyx:105-133: the reference index of every column, -(index) in insertion columns"""
    out, idx = [], 0
    for c in aln_ref:
        if c != "-":
            out.append(idx)
            idx += 1
        else:
            out.append(-1 if idx == 0 else -idx)
    return out


def row(aln_ref, aln_seq, dels=(), ins=(), sizes=(), subs=(), reads=1, name="A", rp=None, n=(1, 1, 1)):
    return {"#Reads": reads, "Aligned_Sequence": aln_seq, "Reference_Sequence": aln_ref, "n_inserted": n[0], "n_deleted": n[1],
            "n_mutated": n[2], "Reference_Name": name, "ref_positions": ref_positions(aln_ref) if rp is None else rp,
            "insertion_coordinates": list(ins), "insertion_sizes": list(sizes), "deletion_coordinates": list(dels),
            "substitution_positions": list(subs)}


def frame(rows):
    return pd.DataFrame(rows)


def repeat_amplicon(rng, length=250, cut=117):
    """random amplicon with a homopolymer, a di- and a trinucleotide run around the cut and a homopolymer from position 0"""
    from crispresso2_b200 import synth
    a = list(synth.random_amplicon(rng, length))
    a[0:9] = "AAAAAAAAA"
    a[cut - 14:cut - 2] = "CACACACACACA"
    a[cut - 2:cut + 6] = "GGGGGGGG"
    a[cut + 6:cut + 18] = "ATTATTATTATT"
    return "".join(a)


def edited_reads(rng, amp, n, cut=117):
    """reads with deletions and insertions inside the runs (so that normalisation walks), some reaching position 0"""
    out = []
    for k in range(n):
        kind = k % 6
        if kind == 0:                                           # deletion inside a run, any length
            a = int(rng.integers(cut - 14, cut + 16)); d = int(rng.integers(1, 7))
            s = amp[:a] + amp[a + d:]
        elif kind == 1:                                         # insertion copying the run's unit
            a = int(rng.integers(cut - 12, cut + 16)); u = amp[a - 3:a]
            s = amp[:a] + u[int(rng.integers(0, 3)):] + amp[a:]
        elif kind == 2:                                         # deletion and insertion in one read
            a = int(rng.integers(cut - 10, cut)); d = int(rng.integers(1, 4))
            b = int(rng.integers(cut + 8, cut + 16))
            s = amp[:a] + amp[a + d:b] + "TTA"[:int(rng.integers(1, 4))] + amp[b:]
        elif kind == 3:                                         # deletion in the homopolymer at position 0
            d = int(rng.integers(1, 4)); a = int(rng.integers(2, 8))
            s = amp[:a] + amp[a + d:]
        elif kind == 4:                                         # substitutions only
            s = list(amp)
            for p in rng.integers(20, len(amp) - 20, size=int(rng.integers(1, 3))):
                s[p] = "ACGT"[(("ACGT".index(s[p])) + 1) % 4]
            s = "".join(s)
        else:                                                   # insertion in the homopolymer at the cut
            a = int(rng.integers(cut - 1, cut + 6))
            s = amp[:a] + "G" * int(rng.integers(1, 5)) + amp[a:]
        out.append(s)
    return out


def frame_from_cache(cache):
    """df_alleles with the columns build_edit_counts reads, one row per (read, aligned reference) as main() builds it
    (CRISPRessoCORE.py:3921-3945, 3964-4030; the AMBIGUOUS_ label of a read that aligned equally well to several)"""
    rows = []
    for v in cache.values():
        if not v["count"]:
            continue
        names = v["aln_ref_names"]
        pairs = [("AMBIGUOUS_" + names[0], names[0])] if v["class_name"] == "AMBIGUOUS" else [(r, r) for r in names]
        for label, r in pairs:
            p = v["variant_" + r]
            rows.append({"#Reads": v["count"], "Aligned_Sequence": p["aln_seq"], "Reference_Sequence": p["aln_ref"],
                         "n_inserted": p["insertion_n"], "n_deleted": p["deletion_n"], "n_mutated": p["substitution_n"],
                         "Reference_Name": label, "ref_positions": p["ref_positions"],
                         "insertion_coordinates": p["insertion_coordinates"], "insertion_sizes": p["insertion_sizes"],
                         "deletion_coordinates": p["deletion_coordinates"], "substitution_positions": p["substitution_positions"]})
    return pd.DataFrame(rows)


def engine_frame(engine, amps, reads, window_size=20):
    """the frame of one engine batch of `reads` against the amplicons `amps` (names A, B, ...)"""
    from crispresso2_b200 import core, synth
    from oracle import oracle as O
    from parity_util import args_from
    names = [chr(ord("A") + k) for k in range(len(amps))]
    refs = {}
    for nm, a in zip(names, amps):
        refs[nm] = synth.amplicon_setup(a, guide_start=97, window_size=window_size)
    params = O.Params()
    d = tempfile.mkdtemp()
    fq = os.path.join(d, "r.fastq")
    with open(fq, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    cache = {}
    core.process_fastq(fq, cache, names, refs, args_from({k: getattr(params, k) for k in vars(params)}), [], d, engine=engine,
                       aln_matrix=O.make_matrix())
    return frame_from_cache(cache), names


def hand_frames():
    """-> [(label, frame, amplicon_positions)] of hand-built rows at the edges of the reference's semantics"""
    R = "ACGTTGCAAGGCTTAC"                                      # no two equal neighbours except the runs below
    H = "AAAACGTCCCCGTAGG"
    out = []
    amp = {"A": ("chr1", 100)}
    out.append(("del_at_0", frame([row(H, "----" + H[4:], dels=[(0, 4)]), row(H, "-" + H[1:], dels=[(1, 2)])]), amp))
    out.append(("del_to_end", frame([row(R, R[:12] + "----", dels=[(12, 16)]), row(H, H[:14] + "--", dels=[(14, 16)])]), amp))
    out.append(("del_whole", frame([row(R, "-" * 16, dels=[(0, 16)]), row(H, "-" * 16, dels=[(0, 16)], reads=3)]), amp))
    ins_ref = H[:7] + "--" + H[7:]
    out.append(("ins_next_to_del", frame([row(ins_ref, H[:5] + "--GC" + H[7:], dels=[(5, 7)], ins=[(6, 7)], sizes=[2])]), amp))
    two = H[:4] + "-" + H[4:10] + "--" + H[10:]
    out.append(("two_ins", frame([row(two, H[:4] + "A" + H[4:10] + "CC" + H[10:], ins=[(3, 4), (9, 10)], sizes=[1, 2])]), amp))
    out.append(("ins_size_over_index", frame([row("--" + R, "GG" + R, ins=[(0, 0)], sizes=[5]),
                                              row(R[:4] + "---" + R[4:], R[:4] + "TTT" + R[4:], ins=[(3, 4)], sizes=[9])]), amp))
    out.append(("ins_left_anchor_is_len", frame([row(R + "--", R + "CC", ins=[(16, 15)], sizes=[2])]), amp))
    out.append(("ins_sizes_short", frame([row(two, H[:4] + "A" + H[4:10] + "CC" + H[10:], ins=[(3, 4), (9, 10)], sizes=[1])]), amp))
    out.append(("counted_but_empty", frame([row(R, R, n=(2, 1, 3)), row(R, R, dels=[(3, 4)], n=(0, 0, 0)),
                                            row(R, R[:3] + "-" + R[4:], dels=[(3, 4)], n=(0, 1, 0))]), amp))
    out.append(("reads_zero", frame([row(H, H[:6] + "A" + H[7:], subs=[6], reads=0), row(H, H[:6] + "A" + H[7:], subs=[6], reads=2)]),
                amp))
    sub = [row(R, R[:5] + "A" + R[6:], subs=[5], name="A", reads=2), row(R, R[:5] + "A" + R[6:], subs=[5], name="B", reads=5),
           row(R, R[:9] + "T" + R[10:], subs=[9], name="C", reads=7)]
    out.append(("two_amplicons_one_chrom", frame(sub), {"A": ("7", 10), "B": ("7", 10), "C": ("07", 10)}))
    out.append(("chrom_names", frame(sub), {"A": ("7", 0), "B": ("chrX", 1), "C": ("07", 1 << 40)}))
    out.append(("offsets", frame(sub), {"A": ("7", 0), "B": ("7", 1), "C": ("7", 2)}))
    neg = row(R, R, subs=[-3], rp=[-3] + list(range(1, 16)))
    out.append(("negative_positions", frame([neg]), amp))
    out.append(("missing_optional_columns", frame([row(R, R[:5] + "A" + R[6:], subs=[5])]).drop(columns=["insertion_sizes",
                                                                                                        "n_inserted"]), amp))
    return out


def error_frames():
    """-> [(label, frame, amplicon_positions)] whose reference call raises: the first failing row must win"""
    R = "ACGTTGCAAGGCTTAC"
    amp = {"A": ("chr1", 100)}
    good = row(R, R[:5] + "A" + R[6:], subs=[5])
    out = []
    out.append(("ambiguous_with_edits", frame([good, row(R, R[:5] + "A" + R[6:], subs=[5], name="AMBIGUOUS_A"),
                                               row(R, R, subs=[99])]), amp))
    out.append(("discarded_with_edits", frame([good, row(R, R[:5] + "A" + R[6:], subs=[5], name="DISCARDED_A")]), amp))
    out.append(("sub_not_in_list", frame([good, row(R, R, subs=[40]), row(R, R, name="ZZ")]), amp))
    out.append(("del_not_in_list", frame([row(R, R, dels=[(30, 33)]), row(R, R, name="ZZ")]), amp))
    out.append(("del_end_fallback_missing", frame([row(R, R, dels=[(3, 40)], rp=[0, 1, 2, 3, 4])]), amp))
    out.append(("ins_not_in_list", frame([good, row(R, R, ins=[(2, 77)], sizes=[1])]), amp))
    out.append(("no_nonnegative_position", frame([good, row("--", "AC", ins=[], rp=[-1, -1], n=(1, 0, 0)),
                                                  row(R, R, subs=[40])]), amp))
    out.append(("deletion_before_max", frame([row("--", "AC", dels=[(5, 6)], rp=[-1, -1])]), amp))
    out.append(("empty_ins_bases", frame([row(R, R, ins=[(5, 6)], sizes=[0])]), amp))
    out.append(("ins_size_over_index", frame([good, row(R[:2] + "---" + R[2:], R[:2] + "TTT" + R[2:], ins=[(1, 2)], sizes=[9])]),
                amp))
    out.append(("string_index", frame([row(R[:4], R[:4], subs=[9], rp=list(range(16)))]), amp))
    out.append(("empty_ref_seq_at_0", frame([row("", "", dels=[(0, 1)], rp=[0, 1])]), amp))
    return out


def big_frame(engine, rng, n_rows):
    """a frame of n_rows rows drawn from one engine batch on a repeat-rich amplicon, with per-row #Reads"""
    amp = repeat_amplicon(rng)
    df, names = engine_frame(engine, [amp], edited_reads(rng, amp, 240))
    take = rng.integers(0, len(df), size=n_rows)
    out = df.iloc[take].reset_index(drop=True)
    out["#Reads"] = rng.integers(0, 50, size=n_rows)
    return out, {names[0]: ("chr5", int(rng.integers(1, 1 << 30)))}

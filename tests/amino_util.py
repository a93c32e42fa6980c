"""Shared by tests/test_amino_acids.py (warp emulator) and tests/test_gpu_amino_acids.py (sm_90a): the reference's own
get_amino_acid_dataframe and global_align (the package under oracle/_ref/install), the frames and protein pairs both are
compared on, and the comparisons: the same frame under pandas' exact checks with the same cut-point warnings, or the same
exception type and message."""
import logging
import os
import sys

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "install", "CRISPResso2", "CRISPRessoShared.py"))
_REF = {}
AAS = "ACDEFGHIKLMNPQRSTVWY*"


def reference():
    """-> (get_amino_acid_dataframe, CRISPResso2Align module, path of the reference's BLOSUM62) as first imported"""
    if not _REF:
        from baseline import ref_shim
        ref_shim.load_core()
        from CRISPResso2 import CRISPResso2Align, CRISPRessoShared
        _REF["fn"] = CRISPRessoShared.get_amino_acid_dataframe
        _REF["align"] = CRISPResso2Align
        _REF["blosum"] = os.path.join(os.path.dirname(CRISPRessoShared.__file__), "BLOSUM62")
    return _REF["fn"], _REF["align"], _REF["blosum"]


class _Warnings(logging.Handler):
    def __init__(self):
        super().__init__()
        self.seen = []

    def emit(self, record):
        self.seen.append(record.getMessage())


def _outcome(fn):
    h = _Warnings()
    logging.getLogger().addHandler(h)
    try:
        return "ok", fn(), h.seen
    except Exception as ex:                                     # noqa: BLE001 -- the exception is the result compared
        return type(ex), str(ex), h.seen
    finally:
        logging.getLogger().removeHandler(h)


def check(df, left, seq_len, cut, engine, chunk=0):
    """the drop-in against the reference on one frame -> the reference's outcome"""
    from crispresso2_b200 import amino_acids
    fn, _, blosum = reference()
    want = _outcome(lambda: fn(df, left, seq_len, blosum, cut))
    got = _outcome(lambda: amino_acids.get_amino_acid_dataframe(df, left, seq_len, blosum, cut, engine=engine, chunk=chunk))
    assert got[2] == want[2], (got[2][:3], want[2][:3], len(got[2]), len(want[2]))
    assert got[0] == want[0], (got[:2], want[:2])
    if want[0] != "ok":
        assert got[1] == want[1], (got[:2], want[:2])
        return want
    if len(df) == 0:
        assert got[1] is df
    else:
        pd.testing.assert_frame_equal(got[1], want[1], check_exact=True, check_index_type=True, check_column_type=True,
                                      check_names=True)
    return want


def refuses_empty(df, left, seq_len, cut, engine, chunk=0):
    """a row whose read or reference translates to nothing: refused with the row named"""
    from crispresso2_b200 import amino_acids
    _, _, blosum = reference()
    try:
        amino_acids.get_amino_acid_dataframe(df, left, seq_len, blosum, cut, engine=engine, chunk=chunk)
    except ValueError as ex:
        return str(ex)
    raise AssertionError("not refused")


# ------------------------------------------------------------------------------------------------ hand-built rows
CDS = "ATGGCTAGCAAAGGAGAAGAACTTTTCACTGGAGTTGTCCCAATTCTTGTTGAATTAGATGGTGATGTTAATGGGCACAAATTTTCTGTCTAA"
AMP = "GGGTTT" + CDS + "TTTCCC"
LEFT = 6


def ref_positions(ref):
    """CRISPResso's ref_positions of an aligned reference: an insertion column holds the position before it (-1 at the start)"""
    out, k = [], -1
    for c in ref:
        if c != "-":
            k += 1
            out.append(k)
        else:
            out.append(k)
    return out


def row(aln, ref=AMP, reads=1, status=None, n=(0, 0, 0), pct=None, rp=None):
    return {"Aligned_Sequence": aln, "Reference_Sequence": ref, "ref_positions": ref_positions(ref) if rp is None else rp,
            "Read_Status": status or ("UNMODIFIED" if aln == ref else "MODIFIED"), "n_deleted": n[0], "n_inserted": n[1],
            "n_mutated": n[2], "#Reads": reads, "%Reads": float(reads) if pct is None else pct}


def frame(rows):
    return pd.DataFrame(rows)


def sub(s, i, c):
    return s[:i] + c + s[i + 1:]


def hand_cases():
    """-> [(label, frame, plot_left_idx, sequence_length, amino_acid_cut_point)]"""
    A, L = AMP, LEFT
    silent = sub(A, L + 5, "C")                                  # GCT -> GCC: A stays A
    missense = sub(A, L + 4, "T")                                # GCT -> GTT: A -> V
    ins = A[:L + 30] + "GGG" + A[L + 30:]
    ins_ref = A[:L + 30] + "---" + A[L + 30:]
    rows = [row(A, reads=20), row(silent, reads=7, n=(0, 0, 1)), row(missense, reads=7, n=(0, 0, 1)),
            row(A[:L + 9] + "---" + A[L + 12:], reads=5, n=(3, 0, 0)), row(A[:L + 10] + "-" + A[L + 11:], reads=4, n=(1, 0, 0)),
            row(ins, ins_ref, reads=3, n=(0, 3, 0)), row(sub(ins, L + 31, "A"), ins_ref, reads=2, n=(0, 3, 1)),
            row(sub(A[:L + 9] + "---" + A[L + 12:], L + 20, "T"), reads=1, n=(3, 0, 1))]
    out = [("mixed", frame(rows), L, 40, 4)]
    out.append(("sequence_length_below", frame(rows), L, 3, 4))
    out.append(("sequence_length_above", frame(rows), L, 500, 4))
    out.append(("sequence_length_negative", frame(rows), L, -2, 4))
    out.append(("cut_point_zero", frame(rows), L, 40, 0))
    out.append(("cut_point_last", frame(rows), L, 40, (len(A) - L) // 3))
    out.append(("cut_point_out_of_range", frame(rows), L, 40, 500))
    out.append(("cut_point_negative", frame(rows), L, 40, -1))
    out.append(("left_at_column_zero", frame(rows), 0, 40, 2))
    out.append(("left_next_to_insertion", frame([row(ins, ins_ref, 2), row(A, reads=3)]), L + 30, 40, 1))
    out.append(("left_after_insertion", frame([row(ins, ins_ref, 2), row(A, reads=3)]), L + 29, 40, 1))
    out.append(("left_at_last_columns", frame([row(A), row(sub(A, len(A) - 3, "T"))]), len(A) - 6, 10, 2))
    # groups that differ only in case: a silent and an identical read give 'A' and 'a' at one place, each its own group
    out.append(("case_only_groups", frame([row(A, reads=2), row(silent, reads=2), row(sub(A, L + 8, "C"), reads=2)]), L, 10, 1))
    # the reference's get_silent_edits unit tests, as rows: silent codon next to an inserted and a deleted codon
    s = A[:L + 3] + "ACT" + A[L + 3:]                            # inserted T after M, then GCT
    out.append(("silent_after_insertion", frame([row(sub(s, L + 8, "C"), A[:L + 3] + "---" + A[L + 3:], 3)]), L, 30, 1))
    d = A[:L + 3] + "---" + A[L + 6:]
    out.append(("silent_after_deletion", frame([row(sub(d, L + 8, "C"), A, 3), row(sub(d, L + 11, "G"), A, 1)]), L, 30, 2))
    out.append(("stop_codons", frame([row(sub(A, L + 4, "A") , reads=2), row(A[:L + 3] + "TAG" + A[L + 6:]),
                                      row(A[:L + 3] + "TGA" + A[L + 6:])]), L, 40, 3))
    out.append(("kahan_pct", frame([row(A, reads=1, pct=p) for p in (1e16, 1.0, 1.0, -1e16, 0.1)]), L, 40, 3))
    out.append(("empty_frame", frame([row(A)]).iloc[:0], L, 40, 3))
    for k in range(6):                                           # suffixes of k nt after left_idx (a read of 3..5 nt translates)
        a = A[:len(A) - 6] + "GCTGCA"[:k] + "-" * (6 - k)
        out.append(("suffix_%d" % k, frame([row(a), row(A)]), len(A) - 6, 10, 0))
    return out


def error_cases():
    """-> [(label, frame, plot_left_idx, sequence_length, cut)] whose reference call raises: the first failing row wins"""
    A, L = AMP, LEFT
    good = row(A, reads=3)
    nread = sub(A, L + 4, "N")
    return [
        ("left_missing", frame([good, row(A, rp=list(range(1000, len(A) + 1000)))]), L, 40, 2),
        ("left_missing_everywhere", frame([good]), 10 ** 6, 40, 2),
        ("n_in_read", frame([good, row(nread), row(sub(A, L + 7, "N"), sub(A, L + 7, "N"))]), L, 40, 500),
        ("lowercase_in_read", frame([good, row(sub(A, L + 4, "c"))]), L, 40, 2),
        ("n_in_reference", frame([good, row(A, sub(A, L + 10, "N"))]), L, 40, 2),
        ("n_in_both", frame([good, row(sub(A, L + 13, "R"), sub(A, L + 10, "N"))]), L, 40, 2),
        ("iupac_after_warnings", frame([good, good, row(sub(A, L + 1, "Y"))]), L, 40, -5),
    ]


def empty_cases():
    """-> [(label, frame, plot_left_idx, sequence_length, cut)] refused on their last row: a translation shorter than one codon,
    or a traceback outside the zone where global_align is defined (one residue each, the incentive at 0)"""
    A = AMP
    return [("undefined_traceback", frame([row(A), row(sub(A, len(A) - 3, "T"))]), len(A) - 3, 10, 0),("read_shorter_than_codon", frame([row(A), row(A[:len(A) - 4] + "----")]), len(A) - 4, 10, 0),
            ("both_shorter_than_codon", frame([row(A)]), len(A) - 2, 10, 0)]


def protein_pairs(rng, n, lo=1, hi=341):
    out = []
    for _ in range(n):
        a = "".join(rng.choice(list(AAS), int(rng.integers(lo, hi + 1))))
        b = "".join(rng.choice(list(AAS), int(rng.integers(lo, hi + 1))))
        out.append((a, b))
    return out


def protein_batch(engine, reads, ref, matrix, gi, go=-1, ge=-1):
    """c2b_protein_align of several reads against one reference -> [(aligned read, aligned ref, score)] as global_align returns
    them; alphabet: the reads' sorted symbols"""
    from crispresso2_b200 import align
    from crispresso2_b200.engine import EngineError
    alpha = "".join(sorted(set("".join(reads))))
    m = np.asarray(matrix)
    rows = np.ascontiguousarray(m[np.frombuffer(ref.encode(), dtype=np.uint8)][:, [ord(c) for c in alpha]].T, dtype=np.int64)
    off = np.zeros(len(reads) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in reads], out=off[1:])
    ops = np.zeros(32 * len(reads), dtype=np.uint64)
    n, k = np.zeros(len(reads), dtype=np.int32), np.zeros(len(reads), dtype=np.int32)
    gi = np.ascontiguousarray(gi, dtype=np.int64)
    rc = engine.L.c2b_protein_align(engine.h, ref.encode(), len(ref), "".join(reads).encode(), off.ctypes.data, len(reads),
                                    alpha.encode(), len(alpha), rows.ctypes.data, gi.ctypes.data, go, ge, ops.ctypes.data,
                                    n.ctypes.data, k.ctypes.data)
    if rc != 0:
        raise EngineError("c2b_protein_align failed (%d): %s" % (rc, engine.L.c2b_last_error(engine.h).decode()))
    out = []
    for r, s in enumerate(reads):
        a, b = align.spell(ops[32 * r:32 * r + 32], int(n[r]), s, ref)
        out.append((a, b, round(100 * int(k[r]) / float(n[r]), 3)))
    return out

"""--coding_seq amino-acid allele tables without a per-row Python pass: a drop-in for the reference's get_amino_acid_dataframe.

    get_amino_acid_dataframe(df_alleles, plot_left_idx, sequence_length, matrix_path, amino_acid_cut_point,
                             collapse_by_sequence=True, engine=None, chunk=0)
        -> the amino-acid allele frame of <ref>amino_acid_table_for_<label>.txt      CRISPRessoShared.py:1557-1653

The rows are packed column by column with numpy.  On the GPU (csrc/c2b_amino.cuh) one warp per row finds the column of
plot_left_idx in ref_positions and translates the gap-stripped read and reference from there; each distinct (read protein,
reference protein) pair is then aligned once by global_align on the engine's own DP (c2b_protein_align's kernel), the silent
edits are marked and the rows grouped and sorted on the host as pandas does (c2b_amino_table).  Only the per-group columns
(silent_edit_inds, the upper-cased index) are built here.  The matrix file is read once per call.  A row on which the reference
raises makes this raise the same exception type and message, for the first such row; a translation shorter than one codon,
where the reference's global_align reads past its strings, and a pair whose traceback leaves the zone where global_align is
defined (SURVEY 3.2) are refused with a ValueError naming the row.  Cells the packer
cannot take -- non-ASCII or non-string sequences, ref_positions that are not lists of ints, a #Reads or n_* value that is not
an int, a %Reads column that is not float -- raise vcf.UnsupportedCell naming the column.  chunk: rows per device pass (<= 0:
the library's default).  The time of the last call's parts, in seconds, is left in the function's last_timings.
"""
import ctypes as C
import logging
import time

import numpy as np

from . import _lib
from .align import read_matrix
from .base_edit import _get_engine, _ints, _p, _strings
from .engine import EngineError
from .vcf import LIMIT, UnsupportedCell, _lists

WHO = "get_amino_acid_dataframe"
_CODE = "KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF"     # c2b_amino.cuh's table: 16 a + 4 b + c over ACGT
CODON_TO_AMINO_ACID = {a + b + c: _CODE[16 * i + 4 * j + k] for i, a in enumerate("ACGT") for j, b in enumerate("ACGT")
                       for k, c in enumerate("ACGT")}
_WARNING = ('amino_acid_cut_point %d is out of range for gap_incentive (length %d); skipping gap incentive.')


def _protein_len(seq, left):
    """residues of get_amino_acids_and_codons(seq[left:].replace('-', '')), raising its KeyError"""
    s = seq[left:].replace("-", "")
    for k in range(0, len(s) - 2, 3):
        CODON_TO_AMINO_ACID[s[k:k + 3]]
    return len(s) // 3


def _warn_rows(ref_lens, cut):
    for n in ref_lens:
        if not 0 <= cut < n + 1:
            logging.warning(_WARNING, cut, n + 1)


def _raise_row(df, r, plot_left_idx, cut):
    """the reference's outcome on the first failing row r: its cut-point warnings for the rows before it, then its exception"""
    refs = df["Reference_Sequence"].to_numpy()
    rps = df["ref_positions"].to_numpy()
    _warn_rows([_protein_len(refs[k], rps[k].index(plot_left_idx)) for k in range(r)], cut)
    left = rps[r].index(plot_left_idx)
    n_read = _protein_len(df["Aligned_Sequence"].to_numpy()[r], left)
    n_ref = _protein_len(refs[r], left)
    if not 0 <= cut < n_ref + 1:
        logging.warning(_WARNING, cut, n_ref + 1)
    raise ValueError("%s: row %d translates to %d read and %d reference residues; global_align is undefined on an empty "
                     "sequence" % (WHO, r, n_read, n_ref))


def get_amino_acid_dataframe(df_alleles, plot_left_idx, sequence_length, matrix_path, amino_acid_cut_point,
                             collapse_by_sequence=True, engine=None, chunk=0):
    """Drop-in for CRISPRessoShared.get_amino_acid_dataframe (CRISPRessoShared.py:1557-1653)."""
    if df_alleles.shape[0] == 0:
        return df_alleles
    import pandas as pd
    t0 = time.perf_counter()
    for c in ("ref_positions", "Aligned_Sequence", "Reference_Sequence", "Read_Status", "n_deleted", "n_inserted", "n_mutated",
              "#Reads", "%Reads"):
        if c not in df_alleles.columns:
            raise KeyError(c)
    for name, v in (("plot_left_idx", plot_left_idx), ("sequence_length", sequence_length),
                    ("amino_acid_cut_point", amino_acid_cut_point)):
        if not isinstance(v, (int, np.integer)) or isinstance(v, bool) or not -LIMIT <= v < LIMIT:
            raise UnsupportedCell("%s: %s = %r is not an int below 2**62 in magnitude" % (WHO, name, v))
    ref, ref_off = _strings(df_alleles["Reference_Sequence"].to_numpy(), "Reference_Sequence", WHO)
    aln, aln_off = _strings(df_alleles["Aligned_Sequence"].to_numpy(), "Aligned_Sequence", WHO)
    try:
        rp, rp_off = _lists(df_alleles["ref_positions"].to_numpy(), "ref_positions")
    except UnsupportedCell as ex:
        raise UnsupportedCell(str(ex).replace("build_edit_counts", WHO)) from None
    unedited = np.asarray(df_alleles["Read_Status"].to_numpy() == "UNMODIFIED", dtype=np.uint8)
    nd, ni, nm, reads = (_ints(df_alleles[c].to_numpy(), c, WHO) for c in ("n_deleted", "n_inserted", "n_mutated", "#Reads"))
    pct = df_alleles["%Reads"].to_numpy()
    if pct.dtype.kind != "f":
        raise UnsupportedCell("%s: column '%%Reads' is not a float column" % WHO)
    pct = np.ascontiguousarray(pct, dtype=np.float64)
    matrix = np.ascontiguousarray(read_matrix(matrix_path), dtype=np.int64)
    t1 = time.perf_counter()
    eng = _get_engine(engine)
    L = eng.L
    err = np.zeros(2, dtype=np.int64)
    h = C.c_void_p()
    rc = L.c2b_amino_table(eng.h, len(df_alleles), int(plot_left_idx), _p(ref), _p(ref_off), _p(aln), _p(aln_off), _p(rp),
                           _p(rp_off), matrix.ctypes.data, matrix.shape[0], int(amino_acid_cut_point), int(sequence_length),
                           _p(unedited), _p(nd), _p(ni), _p(nm), _p(reads), _p(pct), int(chunk), err.ctypes.data, C.byref(h))
    if rc == _lib.E_ARG and err[0] >= 0 and err[1] == _lib.AA_E_UNDEFINED:
        raise ValueError("%s: row %d: global_align's traceback leaves the zone where the reference defines it (SURVEY 3.2)"
                         % (WHO, int(err[0])))
    if rc == _lib.E_ARG and err[0] >= 0:
        _raise_row(df_alleles, int(err[0]), plot_left_idx, amino_acid_cut_point)
    if rc != 0:
        raise EngineError("c2b_amino_table failed (%d): %s" % (rc, L.c2b_last_error(eng.h).decode()))
    try:
        row_ms, align_ms, group_ms, pairs = C.c_double(), C.c_double(), C.c_double(), C.c_int64()
        L.c2b_amino_timings(h, C.byref(row_ms), C.byref(align_ms), C.byref(group_ms), C.byref(pairs))
        t2 = time.perf_counter()
        n = len(df_alleles)
        ref_lens = np.ctypeslib.as_array(C.cast(L.c2b_amino_ref_lens(h), C.POINTER(C.c_int64)), shape=(n,))
        cut = int(amino_acid_cut_point)
        out_of_range = np.flatnonzero((cut < 0) | (cut >= ref_lens + 1))
        if len(out_of_range):
            _warn_rows(ref_lens[out_of_range].tolist(), cut)
        g, nb = L.c2b_amino_n(h), L.c2b_amino_bytes(h)
        seq, fseq, seq_off = np.zeros(max(nb, 1), dtype=np.uint8), np.zeros(max(nb, 1), dtype=np.uint8), np.zeros(g + 1, dtype=np.int64)
        un = np.zeros(g, dtype=np.uint8)
        gd, gi, gm, gr = (np.zeros(g, dtype=np.int64) for _ in range(4))
        gp = np.zeros(g, dtype=np.float64)
        rc = L.c2b_amino_fetch(h, seq.ctypes.data, fseq.ctypes.data, seq_off.ctypes.data, un.ctypes.data, gd.ctypes.data,
                               gi.ctypes.data, gm.ctypes.data, gr.ctypes.data, gp.ctypes.data)
        if rc != 0:
            raise EngineError("c2b_amino_fetch failed (%d)" % rc)
    finally:
        L.c2b_amino_free(h)
    a, b = seq_off[:-1].tolist(), seq_off[1:].tolist()
    raw, fraw = seq.tobytes().decode("ascii"), fseq.tobytes().decode("ascii")
    s1 = [raw[x:y] for x, y in zip(a, b)]
    df = pd.DataFrame({"Aligned_Sequence": s1, "Reference_Sequence": [fraw[x:y] for x, y in zip(a, b)],
                       "Unedited": un.astype(bool), "n_deleted": gd, "n_inserted": gi, "n_mutated": gm, "#Reads": gr,
                       "%Reads": gp}).set_index("Aligned_Sequence")
    df["silent_edit_inds"] = pd.Series([[i for i, c in enumerate(s) if c.islower()] for s in s1], index=df.index, dtype="object")
    df.index = df.index.str.upper()
    t3 = time.perf_counter()
    get_amino_acid_dataframe.last_timings = {"pack": t1 - t0, "rows": row_ms.value / 1e3, "align": align_ms.value / 1e3,
                                             "group": group_ms.value / 1e3, "frame": t3 - t2, "pairs": int(pairs.value)}
    return df


get_amino_acid_dataframe.last_timings = None

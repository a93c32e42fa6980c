"""--base_editor_output allele tables without a per-row Python pass: drop-ins for the reference's
get_upset_plot_counts and get_base_edit_dataframe_around_cut.

    get_upset_plot_counts(df_alleles, bp_substitutions_arr, wt_ref_name, engine=None, chunk=0)
        -> the 19-key dict of figure 10i                    plots/data_prep.py:1869-1988 (CRISPRessoCORE.py:209-327)
    get_base_edit_dataframe_around_cut(df_alleles, conversion_nuc_from, engine=None, chunk=0)
        -> the figure 10h quilt frame                       CRISPRessoShared.py:1472-1506

The rows are packed column by column with numpy and each row is handled by one warp on the GPU (csrc/c2b_base_edit.cuh):
the read bases of every target position with their category and the three keys of the upset counts, or the Aligned_Sequence
characters at the columns where Reference_Sequence holds conversion_nuc_from.  Equal upset keys sum their #Reads on the host
with the exact hash of the FASTQ front end, in first-seen order; quilt rows are grouped, Kahan-summed and sorted as pandas
does (c2b_group_around_cut, shared with the table around the cut).  A row on which the reference raises makes these raise the
same exception type and message, for the first such row.  Cells the packer cannot take -- non-ASCII or non-string sequences,
a #Reads or n_* value that is not an int, a %Reads column that is not float, a bp_substitutions_arr entry that is not
(int, str, str) -- raise vcf.UnsupportedCell naming the column.  chunk: rows per device pass (<= 0: the library's default).
The time of the last call's parts, in seconds, is left in the function's last_timings.
"""
import ctypes as C
import time
from collections import defaultdict

import numpy as np

from . import _lib
from .engine import EngineError
from .vcf import UnsupportedCell, _offsets

_engine = None
CATS = ("reference_base_counts", "target_base_counts", "deletion_base_counts", "insertion_base_counts", "other_base_counts")
_BIG = 1 << 63


def _get_engine(engine):
    global _engine
    if engine is not None:
        return engine
    if _engine is None:
        from .engine import Engine
        _engine = Engine()
    return _engine


def _p(a):
    return a.ctypes.data if a is not None and len(a) else None


def _strings(cells, name, who):
    try:
        data = "".join(cells).encode("ascii")
    except (TypeError, UnicodeEncodeError):
        raise UnsupportedCell("%s: column %r holds a cell that is not an ASCII string" % (who, name)) from None
    lens = np.fromiter(map(len, cells), dtype=np.int64, count=len(cells))
    return np.frombuffer(data, dtype=np.uint8), _offsets(lens)


def _ints(cells, name, who):
    a = np.asarray(cells)
    ok = a.dtype.kind in "iub" or (a.dtype.kind == "O" and all(issubclass(t, (int, np.integer)) for t in set(map(type, a))))
    if not ok:
        raise UnsupportedCell("%s: column %r holds a cell that is not an int" % (who, name))
    try:
        return np.asarray(a.tolist() if a.dtype.kind in "Ou" else a, dtype=np.int64)
    except OverflowError:
        raise UnsupportedCell("%s: column %r holds an int outside int64" % (who, name)) from None


def _on_ref(column, on):
    """the column's cells on wt_ref_name, '' elsewhere (rows on other references are never read)"""
    cells = np.array(column.to_numpy(), dtype=object)
    cells[~on] = ""
    return cells


def _targets(bp_substitutions_arr):
    """positions, string bytes and offsets (ref_base, mod_base per target) of bp_substitutions_arr"""
    pos, strs = [], []
    for item in bp_substitutions_arr:
        ok = isinstance(item, (tuple, list)) and len(item) == 3 and isinstance(item[0], (int, np.integer)) and \
            isinstance(item[1], str) and isinstance(item[2], str) and -_BIG <= item[0] < _BIG
        if ok:
            try:
                strs += [item[1].encode("ascii"), item[2].encode("ascii")]
            except UnicodeEncodeError:
                ok = False
        if not ok:
            raise UnsupportedCell("get_upset_plot_counts: bp_substitutions_arr holds %r, not an (int, str, str) of ASCII text" % (item,))
        pos.append(int(item[0]))
    toff = _offsets(np.asarray([len(s) for s in strs], dtype=np.int64))
    return np.asarray(pos, dtype=np.int64), np.frombuffer(b"".join(strs) or b"\0", dtype=np.uint8), toff


def _upset_dict(nt, keys=(), sums=(), totals=None):
    counts = [defaultdict(int), defaultdict(int), defaultdict(int)]
    for (tag, text), v in zip(keys, sums):
        counts[tag][text] = v
    T = [0] * _lib.BE_N_TOTALS if totals is None else totals[:_lib.BE_N_TOTALS]
    per = {name: ([0] * nt if totals is None else totals[_lib.BE_N_TOTALS + c * nt:_lib.BE_N_TOTALS + (c + 1) * nt])
           for c, name in enumerate(CATS)}
    return {
        "binary_allele_counts": counts[0],
        "category_allele_counts": counts[1],
        "precise_allele_counts": counts[2],
        "total_alleles": T[0],
        "total_alleles_reads": T[1],
        "total_alleles_on_ref": T[2],
        "total_alleles_reads_on_ref": T[3],
        "total_target_noindel_reads": T[6],
        "total_target_indel_reads": T[7],
        "total_reference_noindel_reads": T[4],
        "total_reference_indel_reads": T[5],
        "total_other_noindel_reads": T[8],
        "total_other_indel_reads": T[9],
        "target_base_counts": per["target_base_counts"],
        "reference_base_counts": per["reference_base_counts"],
        "deletion_base_counts": per["deletion_base_counts"],
        "insertion_base_counts": per["insertion_base_counts"],
        "other_base_counts": per["other_base_counts"],
        "total_counts": [T[1]] * nt,
    }


def get_upset_plot_counts(df_alleles, bp_substitutions_arr, wt_ref_name, engine=None, chunk=0):
    """Drop-in for get_upset_plot_counts (plots/data_prep.py:1869-1988 and CRISPRessoCORE.py:209-327)."""
    who = "get_upset_plot_counts"
    t0 = time.perf_counter()
    n = len(df_alleles)
    if n == 0:
        get_upset_plot_counts.last_timings = {"pack": time.perf_counter() - t0, "device": 0.0, "host": 0.0, "frame": 0.0}
        return _upset_dict(len(bp_substitutions_arr))
    tpos, tstr, toff = _targets(bp_substitutions_arr)
    nt = len(tpos)
    cols = df_alleles.columns
    if "#Reads" not in cols:                                    # allele['#Reads'] of the first row
        raise KeyError("#Reads")
    reads = _ints(df_alleles["#Reads"].to_numpy(), "#Reads", who)
    if "Reference_Name" not in cols:
        raise AttributeError("'Series' object has no attribute 'Reference_Name'")
    names = df_alleles["Reference_Name"].to_numpy()
    if isinstance(wt_ref_name, str):
        on = np.asarray(names == wt_ref_name, dtype=bool)
    else:
        on = np.fromiter((x == wt_ref_name for x in names), dtype=bool, count=n)
    flags = on.astype(np.uint8)
    if on.any():
        for c in ("n_deleted", "n_inserted", "Reference_Sequence", "Aligned_Sequence"):     # the first row on wt_ref_name
            if c not in cols:
                raise AttributeError("'Series' object has no attribute %r" % c)
        nd = _ints(df_alleles["n_deleted"].to_numpy()[on], "n_deleted", who)
        ni = _ints(df_alleles["n_inserted"].to_numpy()[on], "n_inserted", who)
        flags[on] |= (((nd > 0) | (ni > 0)).astype(np.uint8) << 1)
        ref, ref_off = _strings(_on_ref(df_alleles["Reference_Sequence"], on), "Reference_Sequence", who)
        aln, aln_off = _strings(_on_ref(df_alleles["Aligned_Sequence"], on), "Aligned_Sequence", who)
    else:
        ref = aln = None
        ref_off = aln_off = np.zeros(n + 1, dtype=np.int64)
    t1 = time.perf_counter()
    eng = _get_engine(engine)
    L = eng.L
    err = np.zeros(2, dtype=np.int64)
    h = C.c_void_p()
    rc = L.c2b_be_upset_counts(eng.h, n, _p(flags), _p(reads), _p(ref), _p(ref_off), _p(aln), _p(aln_off), nt, _p(tpos), _p(tstr),
                               _p(toff), int(chunk), err.ctypes.data, C.byref(h))
    if rc == _lib.E_ARG and err[0] >= 0:
        raise IndexError("string index out of range")
    if rc != 0:
        raise EngineError("c2b_be_upset_counts failed (%d): %s" % (rc, L.c2b_last_error(eng.h).decode()))
    try:
        dev_ms, sum_ms = C.c_double(), C.c_double()
        L.c2b_be_upset_timings(h, C.byref(dev_ms), C.byref(sum_ms))
        t2 = time.perf_counter()
        k = L.c2b_be_upset_n(h)
        ko = np.ctypeslib.as_array(C.cast(L.c2b_be_upset_key_offsets(h), C.POINTER(C.c_int64)), shape=(k + 1,)).copy()
        kb = (np.ctypeslib.as_array(C.cast(L.c2b_be_upset_keys(h), C.POINTER(C.c_uint8)), shape=(int(ko[-1]),)).tobytes()
              if ko[-1] else b"")
        sums = np.ctypeslib.as_array(C.cast(L.c2b_be_upset_reads(h), C.POINTER(C.c_int64)), shape=(k,)).tolist() if k else []
        totals = np.ctypeslib.as_array(C.cast(L.c2b_be_upset_totals(h), C.POINTER(C.c_int64)),
                                       shape=(_lib.BE_N_TOTALS + 5 * nt,)).tolist()
    finally:
        L.c2b_be_upset_free(h)
    text = kb.decode("latin-1")                                 # tag bytes 0 / 1 / 2 before ASCII key text
    keys = [(ord(text[a]), text[a + 1:b]) for a, b in zip(ko[:-1].tolist(), ko[1:].tolist())]
    out = _upset_dict(nt, keys, sums, totals)
    t3 = time.perf_counter()
    get_upset_plot_counts.last_timings = {"pack": t1 - t0, "device": dev_ms.value / 1e3, "host": sum_ms.value / 1e3,
                                          "frame": t3 - t2}
    return out


get_upset_plot_counts.last_timings = None


def get_base_edit_dataframe_around_cut(df_alleles, conversion_nuc_inds, engine=None, chunk=0):
    """Drop-in for CRISPRessoShared.get_base_edit_dataframe_around_cut (CRISPRessoShared.py:1472-1506); the second argument
    is conversion_nuc_from."""
    who = "get_base_edit_dataframe_around_cut"
    if df_alleles.shape[0] == 0:
        return df_alleles
    import pandas as pd
    t0 = time.perf_counter()
    nuc_from = conversion_nuc_inds
    nuc = ord(nuc_from) if isinstance(nuc_from, str) and len(nuc_from) == 1 and ord(nuc_from) < 128 else -1
    cols = df_alleles.columns
    # the columns get_base_edit_row_around_cut reads, in its order on the first row; Aligned_Sequence only where a column holds nuc
    if "Reference_Sequence" not in cols:
        raise KeyError("Reference_Sequence")
    refs = df_alleles["Reference_Sequence"].to_numpy()
    ref, ref_off = _strings(refs, "Reference_Sequence", who)
    uses = np.zeros(len(refs), dtype=bool) if nuc < 0 else \
        np.add.reduceat(np.append(ref == nuc, False), ref_off[:-1].clip(max=len(ref))) > 0
    uses &= np.diff(ref_off) > 0
    if "Aligned_Sequence" not in cols and uses[0]:
        raise KeyError("Aligned_Sequence")
    for c in ("Read_Status", "n_deleted", "n_inserted", "n_mutated", "#Reads", "%Reads"):
        if c not in cols:
            raise KeyError(c)
    if "Aligned_Sequence" not in cols:
        if uses.any():
            raise KeyError("Aligned_Sequence")
        aln, aln_off = None, np.zeros(len(refs) + 1, dtype=np.int64)
    else:
        aln, aln_off = _strings(df_alleles["Aligned_Sequence"].to_numpy(), "Aligned_Sequence", who)
    unedited = np.asarray(df_alleles["Read_Status"].to_numpy() == "UNMODIFIED", dtype=np.uint8)
    nd, ni, nm, reads = (_ints(df_alleles[c].to_numpy(), c, who) for c in ("n_deleted", "n_inserted", "n_mutated", "#Reads"))
    pct = df_alleles["%Reads"].to_numpy()
    if pct.dtype.kind != "f":
        raise UnsupportedCell("%s: column '%%Reads' is not a float column" % who)
    pct = np.ascontiguousarray(pct, dtype=np.float64)
    t1 = time.perf_counter()
    eng = _get_engine(engine)
    L = eng.L
    err = np.zeros(1, dtype=np.int64)
    h = C.c_void_p()
    rc = L.c2b_be_quilt_table(eng.h, len(refs), nuc, _p(ref), _p(ref_off), _p(aln), _p(aln_off), _p(unedited), _p(nd), _p(ni),
                              _p(nm), _p(reads), _p(pct), int(chunk), err.ctypes.data, C.byref(h))
    if rc == _lib.E_ARG and err[0] >= 0:
        raise IndexError("string index out of range")
    if rc != 0:
        raise EngineError("c2b_be_quilt_table failed (%d): %s" % (rc, L.c2b_last_error(eng.h).decode()))
    try:
        dev_ms, group_ms = C.c_double(), C.c_double()
        L.c2b_be_quilt_timings(h, C.byref(dev_ms), C.byref(group_ms))
        t2 = time.perf_counter()
        g, nb = L.c2b_be_quilt_n(h), L.c2b_be_quilt_bytes(h)
        seq, seq_off = np.zeros(max(nb, 1), dtype=np.uint8), np.zeros(g + 1, dtype=np.int64)
        un = np.zeros(g, dtype=np.uint8)
        gd, gi, gm, gr = (np.zeros(g, dtype=np.int64) for _ in range(4))
        gp = np.zeros(g, dtype=np.float64)
        rc = L.c2b_be_quilt_fetch(h, seq.ctypes.data, seq_off.ctypes.data, un.ctypes.data, gd.ctypes.data, gi.ctypes.data,
                                  gm.ctypes.data, gr.ctypes.data, gp.ctypes.data)
        if rc != 0:
            raise EngineError("c2b_be_quilt_fetch failed (%d)" % rc)
    finally:
        L.c2b_be_quilt_free(h)
    lens = np.diff(seq_off)
    from .alleles import _ext
    if _ext is not None:
        s1 = _ext.slices(seq, np.ascontiguousarray(seq_off[:-1]), np.ascontiguousarray(lens, dtype=np.int32))
    else:
        raw = seq.tobytes().decode("latin-1")
        s1 = [raw[a:b] for a, b in zip(seq_off[:-1].tolist(), seq_off[1:].tolist())]
    s2 = [nuc_from * k for k in lens.tolist()] if nuc >= 0 else [""] * g
    df = pd.DataFrame({"Aligned_Sequence": s1, "Reference_Sequence": s2, "Unedited": un.astype(bool), "n_deleted": gd,
                       "n_inserted": gi, "n_mutated": gm, "#Reads": gr, "%Reads": gp}).set_index("Aligned_Sequence")
    t3 = time.perf_counter()
    get_base_edit_dataframe_around_cut.last_timings = {"pack": t1 - t0, "device": dev_ms.value / 1e3, "host": group_ms.value / 1e3,
                                                       "frame": t3 - t2}
    return df


get_base_edit_dataframe_around_cut.last_timings = None

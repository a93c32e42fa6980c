"""--vcf_output edit counts without a per-row Python loop: a drop-in for CRISPResso2.writers.vcf.build_edit_counts.

    build_edit_counts(df_alleles, amplicon_positions, engine=None)
        -> {(chrom, pos, ref, alt): reads}                                    writers/vcf.py:172-212

The edited rows of the detailed allele table (any of n_inserted / n_deleted / n_mutated not 0; a missing column counts as 0)
are packed column by column with numpy, their deletions, insertions and substitutions are turned into left-normalised
(chrom, pos, REF, ALT) records on the GPU (csrc/c2b_vcf.cuh), and equal records sum their #Reads on the host
(c2b_vcf_sum_records).  The dict has Python int / str items in the reference's order.  A row on which the reference raises
makes this raise the same exception type and message, for the first such row.  Cells the packer cannot take -- non-ASCII or
non-string sequences, a non-integer #Reads, list cells that are not sequences of ints or (int, int) pairs, coordinates or
amplicon positions of 2**62 or more in magnitude -- raise UnsupportedCell naming the column.  The reference's
write_vcf_file / write_vcf_from_edits run unchanged on top of it.
"""
import ctypes as C
import itertools
import time

import numpy as np

from . import _lib
from .engine import EngineError

_engine = None
LIMIT = 1 << 62                                             # |coordinate| and |pos| below this: VCF positions stay in int64


class UnsupportedCell(ValueError):
    """a cell of df_alleles (or an amplicon position) outside what the packed form holds"""


def _column(df, name, rows, required=True):
    if name not in df.columns:
        if required:
            raise KeyError(name)
        return None
    return df[name].to_numpy()[rows]


def _strings(cells, name):
    try:
        data = "".join(cells).encode("ascii")
    except (TypeError, UnicodeEncodeError):
        raise UnsupportedCell("build_edit_counts: column %r holds a cell that is not an ASCII string" % name) from None
    lens = np.fromiter(map(len, cells), dtype=np.int64, count=len(cells))
    return np.frombuffer(data, dtype=np.uint8), _offsets(lens)


def _offsets(lens):
    off = np.zeros(len(lens) + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    return off


def _ints(it, count, name):
    """int64 array of the `count` integers of `it`; anything else -> UnsupportedCell"""
    items = list(it)
    try:
        total = sum(items)                                  # a float or a non-number anywhere makes this a non-integer
        if not isinstance(total, (int, np.integer)) or len(items) != count:
            raise TypeError
        vals = np.fromiter(items, dtype=np.int64, count=count)
    except (TypeError, ValueError, OverflowError):
        raise UnsupportedCell("build_edit_counts: column %r holds a cell that is not a sequence of ints" % name) from None
    if count and (vals.min() < -LIMIT or vals.max() >= LIMIT):
        raise UnsupportedCell("build_edit_counts: column %r holds a coordinate of 2**62 or more in magnitude" % name)
    return vals


def _lists(cells, name, pairs=False, or_empty=False):
    """flat int64 values and per-row offsets (in items: ints, or pairs) of list cells; with or_empty (`row.get(name, []) or []`)
    a missing column and None cells are empty"""
    if cells is None:
        return np.zeros(0, dtype=np.int64), None
    if or_empty:
        cells = cells.copy()
        for k in np.flatnonzero(np.asarray(cells == None, dtype=bool)):      # noqa: E711 -- elementwise
            cells[k] = ()
    try:
        lens = np.fromiter(map(len, cells), dtype=np.int64, count=len(cells))
        n = int(lens.sum())
        flat = itertools.chain.from_iterable(cells)
        if pairs:
            items = list(flat)
            if n and not (np.fromiter(map(len, items), dtype=np.int64, count=n) == 2).all():
                raise TypeError
            flat = itertools.chain.from_iterable(items)
    except TypeError:
        raise UnsupportedCell("build_edit_counts: column %r holds a cell that is not a sequence of %s"
                              % (name, "(int, int) pairs" if pairs else "ints")) from None
    return _ints(flat, 2 * n if pairs else n, name), _offsets(lens)


def _reads(cells):
    a = np.asarray(cells)
    if a.dtype.kind == "O":
        if not all(issubclass(t, (int, np.integer)) for t in set(map(type, a))):
            raise UnsupportedCell("build_edit_counts: column '#Reads' holds a cell that is not an int")
    elif a.dtype.kind not in "iub":
        raise UnsupportedCell("build_edit_counts: column '#Reads' holds a cell that is not an int")
    try:
        return np.asarray(a.tolist() if a.dtype.kind in "Ou" else a, dtype=np.int64)
    except OverflowError:
        raise UnsupportedCell("build_edit_counts: column '#Reads' holds a count outside int64") from None


def _edited_rows(df):
    n = len(df)
    unedited = np.ones(n, dtype=bool)
    for name in ("n_inserted", "n_deleted", "n_mutated"):   # row.get(name, 0) == 0
        if name in df.columns:
            unedited &= np.asarray(df[name].to_numpy() == 0, dtype=bool)
    return np.flatnonzero(~unedited)


def build_edit_counts(df_alleles, amplicon_positions, engine=None, chunk=0):
    """Drop-in for CRISPResso2.writers.vcf.build_edit_counts (writers/vcf.py:172-212).  chunk: rows per device pass (<= 0:
    the library's default).  The time of the last call's parts, in seconds, is left in build_edit_counts.last_timings."""
    global _engine
    t0 = time.perf_counter()
    rows = _edited_rows(df_alleles)
    if len(rows) == 0:
        build_edit_counts.last_timings = {"pack": time.perf_counter() - t0, "device": 0.0, "sum": 0.0, "dict": 0.0, "records": 0}
        return {}
    import pandas as pd
    names = _column(df_alleles, "Reference_Name", rows)
    amp_names = list(amplicon_positions)
    amp = pd.Index(amp_names, dtype=object).get_indexer(pd.Index(names, dtype=object)) if amp_names else np.full(len(rows), -1)
    first_missing = int(np.flatnonzero(amp < 0)[0]) if (amp < 0).any() else len(rows)
    chroms, chrom_id, amp_chrom, amp_pos = [], {}, [], []
    for nm in amp_names:
        chrom, pos = amplicon_positions[nm]
        if not isinstance(pos, (int, np.integer)) or isinstance(pos, bool) or not -LIMIT <= pos < LIMIT:
            raise UnsupportedCell("build_edit_counts: amplicon_positions[%r] has a position that is not an int below 2**62 in "
                                  "magnitude" % (nm,))
        if chrom not in chrom_id:
            chrom_id[chrom] = len(chroms)
            chroms.append(chrom)
        amp_chrom.append(chrom_id[chrom])
        amp_pos.append(int(pos))
    amp_chrom = np.asarray(amp_chrom + [-1], dtype=np.int32)
    amp_pos = np.asarray(amp_pos + [0], dtype=np.int64)
    chrom_r, pos_r = np.ascontiguousarray(amp_chrom[amp]), np.ascontiguousarray(amp_pos[amp])
    try:
        reads = _reads(_column(df_alleles, "#Reads", rows))
        ref, ref_off = _strings(_column(df_alleles, "Reference_Sequence", rows), "Reference_Sequence")
        aln, aln_off = _strings(_column(df_alleles, "Aligned_Sequence", rows), "Aligned_Sequence")
        rp, rp_off = _lists(_column(df_alleles, "ref_positions", rows), "ref_positions")
        dl, dl_off = _lists(_column(df_alleles, "deletion_coordinates", rows), "deletion_coordinates", pairs=True)
        ins, ins_off = _lists(_column(df_alleles, "insertion_coordinates", rows, required=False), "insertion_coordinates",
                              pairs=True, or_empty=True)
        isz, isz_off = _lists(_column(df_alleles, "insertion_sizes", rows, required=False), "insertion_sizes", or_empty=True)
        sub, sub_off = _lists(_column(df_alleles, "substitution_positions", rows), "substitution_positions")
    except KeyError:
        if first_missing == 0:                              # the first edited row already fails its amplicon_positions lookup
            raise KeyError(names[0]) from None
        raise
    empty = np.zeros(len(rows) + 1, dtype=np.int64)
    ins_off = empty if ins_off is None else ins_off
    isz_off = empty if isz_off is None else isz_off
    t1 = time.perf_counter()
    if engine is None:
        if _engine is None:
            from .engine import Engine
            _engine = Engine()
        engine = _engine
    L = engine.L
    err = np.zeros(3, dtype=np.int64)
    h = C.c_void_p()

    def p(a):
        return a.ctypes.data if a is not None and len(a) else None

    rc = L.c2b_vcf_edit_counts(engine.h, len(rows), p(chrom_r), p(pos_r), p(reads), p(ref), p(ref_off), p(aln), p(aln_off),
                               p(rp), p(rp_off), p(dl), p(dl_off), p(ins), p(ins_off), p(isz), p(isz_off), p(sub), p(sub_off),
                               int(chunk), err.ctypes.data, C.byref(h))
    if rc == _lib.E_ARG and err[0] >= 0:
        r, kind, value = int(err[0]), int(err[1]), int(err[2])
        if kind == _lib.VCF_E_KEY:
            raise KeyError(names[r])
        if kind == _lib.VCF_E_NOT_IN_LIST:
            raise ValueError("%d is not in list" % value)
        if kind == _lib.VCF_E_STRING_INDEX:
            raise IndexError("string index out of range")
        if kind == _lib.VCF_E_EMPTY_MAX:
            raise ValueError("max() iterable argument is empty")
    if rc != 0:
        raise EngineError("c2b_vcf_edit_counts failed (%d): %s" % (rc, L.c2b_last_error(engine.h).decode()))
    try:
        dev_ms, sum_ms = C.c_double(), C.c_double()
        L.c2b_vcf_timings(h, C.byref(dev_ms), C.byref(sum_ms))
        t2 = time.perf_counter()
        n = L.c2b_vcf_n(h)
        n_records = L.c2b_vcf_n_records(h)
        ko = np.ctypeslib.as_array(C.cast(L.c2b_vcf_key_offsets(h), C.POINTER(C.c_int64)), shape=(n + 1,)).copy()
        kb = np.ctypeslib.as_array(C.cast(L.c2b_vcf_keys(h), C.POINTER(C.c_uint8)), shape=(int(ko[-1]),)).copy() if ko[-1] \
            else np.zeros(0, dtype=np.uint8)
        sums = np.ctypeslib.as_array(C.cast(L.c2b_vcf_reads(h), C.POINTER(C.c_int64)), shape=(n,)).tolist() if n else []
    finally:
        L.c2b_vcf_free(h)
    # key i: chrom id (int32) | pos (int64) | len(REF) (int32) | REF | ALT
    hdr = kb[ko[:-1, None] + np.arange(16)] if n else np.zeros((0, 16), dtype=np.uint8)
    cid = hdr[:, 0:4].copy().view("<i4").ravel().tolist()
    vpos = hdr[:, 4:12].copy().view("<i8").ravel().tolist()
    a = (ko[:-1] + 16).tolist()
    b = (ko[:-1] + 16 + hdr[:, 12:16].copy().view("<i4").ravel()).tolist()
    e = ko[1:].tolist()
    text = kb.tobytes().decode("latin-1")                   # binary headers between the ASCII REF / ALT
    out = dict(zip([(chroms[c], v, text[x:y], text[y:z]) for c, v, x, y, z in zip(cid, vpos, a, b, e)], sums))
    t3 = time.perf_counter()
    build_edit_counts.last_timings = {"pack": t1 - t0, "device": dev_ms.value / 1e3, "sum": sum_ms.value / 1e3,
                                      "dict": t3 - t2, "records": int(n_records)}
    return out


build_edit_counts.last_timings = None

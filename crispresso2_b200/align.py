"""CRISPResso2Align-compatible surface (reference: CRISPResso2/CRISPResso2Align.pyx).

  read_matrix(path)            Align.pyx:33-61
  make_matrix(...)             Align.pyx:63-99
  global_align(seqj, seqi, matrix, gap_incentive, gap_open=-1, gap_extend=-1) -> (str, str, float)
                               Align.pyx:101-434 -- runs on the GPU through c2b_global_align, or through c2b_protein_align
                               when the read has 9 to 32 distinct symbols (protein strings).
"""
import ctypes as C

import numpy as np

_engine = None


def read_matrix(path):
    """NCBI-format matrix file -> int64 table with tab[ord(row_symbol), ord(col_symbol)] = score."""
    with open(path) as fh:
        lines = fh.read().split("\n")
    k = 0
    while k < len(lines) and (not lines[k].strip() or lines[k].strip().startswith("#")):
        k += 1
    symbols = [ord(t) for t in lines[k].split()]
    size = max(symbols) + 1
    tab = np.zeros((size, size), dtype=np.int64)
    row = 0
    for ln in lines[k + 1:]:
        toks = ln.split()
        if not toks:
            continue
        for col, tok in zip(symbols, toks[1:]):
            tab[symbols[row], col] = int(tok)
        row += 1
    return tab


def make_matrix(match_score=5, mismatch_score=-4, n_mismatch_score=-2, n_match_score=-1):
    size = ord("T") + 1
    tab = np.zeros((size, size), dtype=np.int64)
    bases = [ord(c) for c in "ATCG"]
    n = ord("N")
    for a in bases:
        tab[a, bases] = mismatch_score
        tab[a, a] = match_score
        tab[a, n] = tab[n, a] = n_mismatch_score
    tab[n, n] = n_match_score
    return tab


def global_align(pystr_seqj, pystr_seqi, matrix, gap_incentive, gap_open=-1, gap_extend=-1, engine=None):
    """Needleman-Wunsch of read `seqj` against reference `seqi` on the GPU; same return value as the
    reference: (aligned_read, aligned_ref, round(100*matches/columns, 3)).  A gap_incentive of the wrong
    length prints the reference's message and returns 0 (Align.pyx:124-126)."""
    from .engine import Engine, EngineError
    global _engine
    if engine is None:
        if _engine is None:
            _engine = Engine()
        engine = _engine
    J, I = len(pystr_seqj), len(pystr_seqi)
    gi = np.ascontiguousarray(gap_incentive, dtype=np.int64)
    if len(gi) != I + 1:
        print('\nERROR: Mismatch in gap_incentive length (gap_incentive: ' + str(len(gi)) + ' ref: ' + str(I + 1) + '\n')
        return 0
    if I < 1 or J < 1:
        raise ValueError("global_align needs non-empty sequences (the reference is undefined there)")
    matrix = np.asarray(matrix)
    alphabet = "".join(sorted(set(pystr_seqj)))
    codes = np.frombuffer(pystr_seqi.encode(), dtype=np.uint8).astype(np.int64)
    cols = [ord(c) for c in alphabet]
    if codes.max() >= matrix.shape[0] or max(cols) >= matrix.shape[1]:
        raise ValueError("sequence symbol outside the substitution matrix")
    rows = np.ascontiguousarray(matrix[codes][:, cols].T, dtype=np.int64)
    if len(alphabet) > 8:
        return _protein_align(engine, pystr_seqj, pystr_seqi, alphabet, rows, gi, gap_open, gap_extend)
    out_j = C.create_string_buffer(I + J + 1)
    out_i = C.create_string_buffer(I + J + 1)
    n, m = C.c_int32(0), C.c_int32(0)
    rc = engine.L.c2b_global_align(engine.h, pystr_seqj.encode(), J, pystr_seqi.encode(), I, alphabet.encode(),
                                   len(alphabet), rows.ctypes.data, gi.ctypes.data, int(gap_open), int(gap_extend),
                                   out_j, out_i, C.byref(n), C.byref(m))
    engine.n_refs = 0
    if rc != 0:
        raise EngineError("c2b_global_align failed (%d): %s" % (rc, engine.L.c2b_last_error(engine.h).decode()))
    s1, s2 = out_j.raw[:n.value].decode(), out_i.raw[:n.value].decode()
    return s1, s2, round(100 * m.value / float(n.value), 3)


def spell(ops, n, read, ref):
    """the aligned strings of an op stream of n columns (column k from the right: bits 2 (k & 31) of ops[k >> 5]; 0 both,
    1 gap in the read, 2 gap in the reference)"""
    a, b = [], []
    j, i = len(read), len(ref)
    for k in range(n):
        op = (int(ops[k >> 5]) >> (2 * (k & 31))) & 3
        if op != 1:
            j -= 1
        if op != 2:
            i -= 1
        a.append("-" if op == 1 else read[j])
        b.append("-" if op == 2 else ref[i])
    return "".join(reversed(a)), "".join(reversed(b))


def _protein_align(engine, seqj, seqi, alphabet, rows, gi, gap_open, gap_extend):
    """one read of 9-32 distinct symbols through c2b_protein_align; the engine's configuration is left as it is"""
    from .engine import EngineError
    ops = np.zeros(32, dtype=np.uint64)
    n, m = np.zeros(1, dtype=np.int32), np.zeros(1, dtype=np.int32)
    off = np.array([0, len(seqj)], dtype=np.int64)
    rc = engine.L.c2b_protein_align(engine.h, seqi.encode(), len(seqi), seqj.encode(), off.ctypes.data, 1, alphabet.encode(),
                                    len(alphabet), rows.ctypes.data, gi.ctypes.data, int(gap_open), int(gap_extend),
                                    ops.ctypes.data, n.ctypes.data, m.ctypes.data)
    if rc != 0:
        raise EngineError("c2b_protein_align failed (%d): %s" % (rc, engine.L.c2b_last_error(engine.h).decode()))
    s1, s2 = spell(ops, int(n[0]), seqj, seqi)
    return s1, s2, round(100 * int(m[0]) / float(n[0]), 3)

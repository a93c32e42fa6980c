"""Host-side mirror of the reference's per-read driver for the GPU path.

Same call signatures as the reference functions they stand in for:
  process_fastq(fastq_filename, variantCache, ref_names, refs, args, files_to_remove, output_directory)
      -> (aln_stats, not_aligned_variants)                        CRISPRessoCORE.py:1735-2000
  get_new_variant_object(args, fastq_seq, refs, ref_names, aln_matrix, pe_scaffold_dna_info)
      -> variant dict                                             CRISPRessoCORE.py:627-798
and, for the count arrays the quantification loop builds from variantCache (CRISPRessoCORE.py:3964-4115),
  quantify(variantCache) -> CountBlock        (the device block accumulated by the process_fastq call)

Everything decided per read (strand, alignment, best reference, classification, counts) is decided by the CUDA
kernel; this module parses the FASTQ, de-duplicates reads exactly like the reference (:1825-1849), derives the
reverse-complement merge weights of :3971-3975, launches one batch and re-labels the outputs as the reference's
dict / ResultsSlotsDict shapes.  process_fastq bypasses CRISPRessoMultiProcessing (n_processes is ignored) and
follows the SERIAL branch's statistics (:1956-1981).
"""
import os

import numpy as np

from . import _lib
from .align import read_matrix
from . import fastq
from .engine import Engine, EngineError, pack_reads
from .resources import payload_from_lists

_COMP = str.maketrans("ACGTN_-", "TGCAN_-")
_engines = {}
_blocks = {}
_sources = {}                     # id(variantCache) -> lazy.BatchSource of the process_fastq call that filled it (alleles.py)
last_timings = {}                 # seconds of the last process_fastq call by stage (bench.py's api leg reports them)


def reverse_complement(seq):
    """CRISPRessoShared.py:399-403 (KeyError on symbols outside ACGTN_- like the reference)."""
    up = seq.upper()
    bad = set(up) - set("ACGTN_-")
    if bad:
        raise KeyError(sorted(bad)[0])
    return up.translate(_COMP)[::-1]


def _flags(args):
    f = 0
    if getattr(args, "ignore_substitutions", False):
        f |= _lib.F_IGNORE_SUBSTITUTIONS
    if getattr(args, "ignore_insertions", False):
        f |= _lib.F_IGNORE_INSERTIONS
    if getattr(args, "ignore_deletions", False):
        f |= _lib.F_IGNORE_DELETIONS
    if getattr(args, "expand_ambiguous_alignments", False):
        f |= _lib.F_EXPAND_AMBIGUOUS
    if getattr(args, "assign_ambiguous_alignments_to_first_reference", False):
        f |= _lib.F_ASSIGN_FIRST
    if getattr(args, "discard_indel_reads", False):
        f |= _lib.F_DISCARD_INDEL_READS
    if getattr(args, "expected_hdr_amplicon_seq", "") or getattr(args, "prime_editing_pegRNA_extension_seq", ""):
        f |= _lib.F_HDR_REF1
    if getattr(args, "use_legacy_insertion_quantification", False):
        f |= _lib.F_LEGACY_INS
    return f


def _unsupported(args, refs=None):
    if getattr(args, "use_legacy_insertion_quantification", False) and refs and any(r.get("contains_coding_seq") for r in refs.values()):
        raise NotImplementedError("use_legacy_insertion_quantification together with a coding sequence is not built on the GPU path")


SCAFFOLD_REF, PE_REF = "Scaffold-incorporated", "Prime-edited"


def scaffold_search(args, refs):
    """pe_scaffold_dna_info of process_fastq (CRISPRessoCORE.py:1814-1816; plots/data_prep.py:3827-3860): (position in the
    prime-edited amplicon right after the pegRNA extension, the shortest scaffold prefix whose presence there cannot come from
    the amplicon itself), or None when no scaffold sequence was given."""
    scaf = getattr(args, "prime_editing_pegRNA_scaffold_seq", "") or ""
    if not scaf:
        return None
    ext = getattr(args, "prime_editing_pegRNA_extension_seq", "") or ""
    if not ext:
        raise ValueError("prime_editing_pegRNA_scaffold_seq needs prime_editing_pegRNA_extension_seq")
    amplicon = refs[PE_REF]["sequence"]
    scaffold_dna = reverse_complement(scaf.upper().replace("U", "T"))
    ext_dna = reverse_complement(ext.upper().replace("U", "T"))
    loc = amplicon.index(ext_dna) + len(ext_dna)
    k = int(getattr(args, "prime_editing_pegRNA_scaffold_min_match_length", 1))
    while ext_dna + scaffold_dna[:k] in amplicon:
        if k > len(scaffold_dna):
            raise ValueError("The DNA scaffold provided is found in the unedited reference sequence. "
                             "Please provide a longer scaffold sequence.")
        k += 1
    return loc, scaffold_dna[:k]


def scaffold_hits(res, pe_idx, loc, seq, block=32768):
    """Reads of a batch that the scaffold step of get_new_variant_object re-labels (CRISPRessoCORE.py:789-796): 'Prime-edited'
    among the best references, and the read's aligned string carrying `seq` right after the column of prime-edited position
    loc - 1.  Vectorised over the aligned strings (rebuilt from the op streams block by block).  -> bool [n]"""
    n = len(res.recs)
    out = np.zeros(n, dtype=bool)
    cand = ((res.recs["winner_mask"].astype(np.int64) >> pe_idx) & 1).astype(bool) & (res.recs["best_score_milli"] > 0)
    if not cand.any():
        return out
    W, k = res.W, len(seq)
    want = np.frombuffer(seq.encode(), dtype=np.uint8)
    cols = np.arange(W, dtype=np.int32)
    for lo in range(0, n, block):
        hi = min(n, lo + block)
        idx = np.nonzero(cand[lo:hi])[0]
        if not len(idx):
            continue
        S = res.strings_block(lo, hi)[idx, pe_idx]                       # [m, 2, W], right-aligned
        alen = res.alns["aln_len"][lo:hi][idx, pe_idx].astype(np.int32)
        base = (S[:, 1, :] != ord("-")) & (cols[None, :] >= (W - alen)[:, None])
        here = base & (np.cumsum(base, axis=1, dtype=np.int32) == loc)
        at = np.argmax(here, axis=1) + 1                                  # ref_positions.index(loc - 1) + 1
        ok = here.any(axis=1) & (at + k <= W)
        take = np.minimum(at[:, None] + np.arange(k, dtype=np.int64)[None, :], W - 1)
        got = np.take_along_axis(S[:, 0, :], take, axis=1)
        out[lo + idx] = ok & (got == want[None, :]).all(axis=1)
    return out


def get_engine(device=0, lib_path=None):
    key = (device, lib_path)
    if key not in _engines:
        _engines[key] = Engine(device, lib_path)
    return _engines[key]


def configure_engine(engine, args, refs, ref_names, aln_matrix, edit_cap=12):
    engine.configure(refs, ref_names, aln_matrix, args.needleman_wunsch_gap_open, args.needleman_wunsch_gap_extend,
                     args.aln_seed_count, args.aln_seed_min, _flags(args), "ACGTN", edit_cap)
    return engine


def merge_weights(uniques, counts):
    """Weights the quantification loop ends up using after its reverse-complement merge (CRISPRessoCORE.py:3971-3975):
    walking the cache in first-seen order, a read absorbs the count of its reverse complement (which drops to 0);
    a palindromic read absorbs itself.  Valid because a read and its reverse complement always share their aligned
    status (same score set), so both are in the cache or neither is."""
    pos = {s: k for k, s in enumerate(uniques)}
    w = list(counts)
    for k, s in enumerate(uniques):
        if w[k] == 0:
            continue
        try:
            rc = reverse_complement(s)
        except KeyError:
            continue
        j = pos.get(rc)
        if j is not None and w[j] > 0:
            tot = w[k] + w[j]
            w[j] = 0
            w[k] = tot
    return w


class _BatchLists:
    """Plain-Python views of a batch's output arrays, converted with one .tolist() per block of reads: the per-read
    work then touches tuples instead of numpy scalars (about 5x less host time per unique read)."""
    BLOCK = 4096

    def __init__(self, res):
        self.res = res
        self.W, self.nref = res.W, res.alns.shape[1]
        self.lo = self.hi = 0
        self.text = None

    def block(self, i):
        if not (self.lo <= i < self.hi):
            self.lo = (i // self.BLOCK) * self.BLOCK
            self.hi = min(self.lo + self.BLOCK, len(self.res.recs))
            r = self.res
            self.recs = r.recs[self.lo:self.hi].tolist()     # (winner_mask, best_score_milli, best_ref, n_winners, ambiguous, status)
            self.alns = r.alns[self.lo:self.hi].tolist()     # [read][ref] -> ALN_DTYPE field order
            self.edits = r.edits[self.lo:self.hi].tolist() if r.edits is not None else None
            # one decode per block; bytes left of an alignment are undefined, hence latin-1 (never fails, 1 char per byte)
            self.text = (r.strings_block(self.lo, self.hi).tobytes().decode("latin-1")
                         if (r.strings is not None or r.ops is not None) else None)
        return i - self.lo

    def pair(self, i, r, n):
        base = (((i - self.lo) * self.nref + r) * 2) * self.W
        return self.text[base + self.W - n: base + self.W], self.text[base + 2 * self.W - n: base + 2 * self.W]


# ALN_DTYPE field positions (crispresso2_b200/_lib.py)
(_A_NMATCH, _A_ALNLEN, _A_SCORE, _A_STRAND, _A_STATUS, _A_NEDITS, _A_INS_N, _A_DEL_N, _A_SUB_N, _A_NINS_ALL, _A_NINS_WIN,
 _A_NDEL_ALL, _A_NDEL_WIN, _A_NDELPOS_ALL, _A_NSUB_ALL, _A_IRR, _A_MOD) = range(17)


def _variant_from(res, i, seq, ref_names, refs):
    """dict of get_new_variant_object (CRISPRessoCORE.py:709-798) for read i of a batch result."""
    L = getattr(res, "_lists", None)
    if L is None:
        L = res._lists = _BatchLists(res)
    k = L.block(i)
    winner_mask, best_milli, _, _, ambiguous, _ = L.recs[k]
    nref = len(ref_names)
    alns = L.alns[k]
    scores = [alns[r][_A_SCORE] / 1000.0 for r in range(nref)]
    details = []
    for r in range(nref):
        s1, s2 = L.pair(i, r, alns[r][_A_ALNLEN])
        details.append((ref_names[r], s1, s2, scores[r]))
    if best_milli <= 0:
        return {"count": 1, "aln_scores": scores, "ref_aln_details": details, "best_match_score": -1}
    winners = [r for r in range(nref) if (winner_mask >> r) & 1]
    # key order of CRISPRessoCORE.py:711-715
    v = {"count": 1, "aln_ref_names": [ref_names[r] for r in winners], "aln_scores": scores, "ref_aln_details": details,
         "best_match_score": best_milli / 1000.0}
    labels = []
    for r in winners:
        a = alns[r]
        name = ref_names[r]
        s1, s2 = details[r][1], details[r][2]
        n = a[_A_NEDITS]
        if a[_A_STATUS] & _lib.ST_EDIT_OVERFLOW or L.edits is None or n > len(L.edits[k][r]):
            raise OverflowError("edit list overflow")
        p = payload_from_lists(a[_A_INS_N], a[_A_DEL_N], a[_A_SUB_N], L.edits[k][r][:n], s2, legacy=bool(res_flags(res) & _lib.F_LEGACY_INS))
        p.ref_name = name
        p.aln_scores = scores
        p.irregular_ends = bool(a[_A_IRR])
        n_ins_all, n_ins_win = a[_A_NINS_ALL], a[_A_NINS_WIN]
        p.insertions_outside_window = n_ins_all - n_ins_win
        p.deletions_outside_window = a[_A_NDEL_ALL] - a[_A_NDEL_WIN]
        p.substitutions_outside_window = a[_A_NSUB_ALL] - a[_A_SUB_N]
        p.total_mods = n_ins_all + a[_A_NDELPOS_ALL] + a[_A_NSUB_ALL]
        p.mods_in_window = a[_A_SUB_N] + a[_A_DEL_N] + a[_A_INS_N]
        p.mods_outside_window = p.total_mods - p.mods_in_window
        p.classification = "MODIFIED" if a[_A_MOD] else "UNMODIFIED"
        labels.append(name + "_" + p.classification)
        p.aln_seq, p.aln_ref = s1, s2
        p.aln_strand = "-" if a[_A_STRAND] else "+"
        v["variant_" + name] = p
        v["best_match_name"] = name
    v["class_name"] = "&".join(labels)
    if len(winners) > 1:                                     # CRISPRessoCORE.py:780-785: assign-first is tested first
        if res_flags(res) & _lib.F_ASSIGN_FIRST:
            v["class_name"] = labels[0]
            v["aln_ref_names"] = [ref_names[winners[0]]]
        elif not (res_flags(res) & _lib.F_EXPAND_AMBIGUOUS):
            v["class_name"] = "AMBIGUOUS"
    sc = getattr(res, "scaffold", None)
    if sc is not None and any(ref_names[r] == PE_REF for r in winners):     # CRISPRessoCORE.py:789-796
        from copy import deepcopy
        loc, seq = sc
        pe = v["variant_" + PE_REF]
        at = pe.ref_positions.index(loc - 1) + 1
        if pe.aln_seq[at:at + len(seq)] == seq:
            v["aln_ref_names"] = [SCAFFOLD_REF]
            v["class_name"] = SCAFFOLD_REF
            old = deepcopy(pe)
            old.ref_name = SCAFFOLD_REF
            v["variant_" + SCAFFOLD_REF] = old
    return v


def res_flags(res):
    return getattr(res, "flags", 0)


def merge_weights_packed(buf, off, counts, member=None, lib_path=None):
    """merge_weights for packed unique reads, natively (c2b_rc_merge_weights: host threads, exact)."""
    L = _lib.load(lib_path)
    n = len(off) - 1
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    w = np.zeros(n, dtype=np.int32)
    mem = None if member is None else np.ascontiguousarray(member, dtype=np.uint8)
    rc = L.c2b_rc_merge_weights(buf.ctypes.data if len(buf) else None, off.ctypes.data, n, counts.ctypes.data,
                                mem.ctypes.data if mem is not None else None, w.ctypes.data, 0)
    if rc != 0:
        raise EngineError("c2b_rc_merge_weights failed (%d)" % rc)
    return w


def screen_reads(buf, off, lib_path=None):
    """-> bool mask of unique reads outside the engine's contract: empty, longer than MAX_READ_LEN, or holding a symbol
    other than A C G T N (lower case and IUPAC codes included: the reference indexes its score table with them -- lower case
    out of bounds, Align.pyx:212 -- and its quantification loop raises KeyError on them at CRISPRessoCORE.py:4081).
    Native (c2b_screen_reads, host threads)."""
    L = _lib.load(lib_path)
    n = len(off) - 1
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    out = np.zeros(n, dtype=np.uint8)
    rc = L.c2b_screen_reads(buf.ctypes.data if len(buf) else None, off.ctypes.data, n, _lib.MAX_READ_LEN, out.ctypes.data, 0)
    if rc < 0:
        raise EngineError("c2b_screen_reads failed (%d)" % rc)
    return out.astype(bool)


def align_uniques(engine, uniques, counts, ref_names, refs, flags, weights=None, packed=None, compact=False, on_launch=None):
    """One GPU batch over unique reads -> (BatchResult, merge weights).  `packed` = (bytes, offsets) of `uniques`
    when the caller already holds them in the engine's layout."""
    buf, off = packed if packed is not None else pack_reads(uniques)
    if weights is None:
        weights = merge_weights_packed(buf, off, counts, lib_path=engine.lib_path)
    res = engine.align_packed(buf, off, count=np.asarray(counts, dtype=np.int32), qweight=np.asarray(weights, dtype=np.int32),
                              compact=compact, on_launch=on_launch)
    res.flags = flags
    st = res.recs["status"]
    hard = st & ~np.uint32(_lib.ST_EDIT_OVERFLOW)
    if hard.any():
        k = int(np.nonzero(hard)[0][0])
        raise EngineError("read %d outside the engine's contract: status %d" % (k, int(st[k])))
    return res, weights


def _subset(buf, off, idx):
    lens = (off[idx + 1] - off[idx]).astype(np.int64)
    o2 = np.zeros(len(idx) + 1, dtype=np.int64)
    np.cumsum(lens, out=o2[1:])
    b2 = np.concatenate([buf[off[k]:off[k + 1]] for k in idx.tolist()]) if len(idx) else np.zeros(0, np.uint8)
    return np.ascontiguousarray(b2), o2


def _batch(engine, buf, off, counts, weights, ref_names, refs, flags, args, aln_matrix, scaffold, on_launch=None):
    """The batch over (a slice of) the unique reads.  -> (BatchResult, scaffold extra or None).
    Prime editing with a scaffold sequence (CRISPRessoCORE.py:789-796): reads the scaffold step re-labels count under the
    extra reference 'Scaffold-incorporated' with their alignment to the prime-edited amplicon, whatever else they tied with.
    All of it stays on the device, as further passes of the same kernels:
      1. the batch as usual; scaffold_hits() picks the re-labelled reads H out of the aligned strings;
      A. H alone, every read bound to the prime-edited amplicon (the per-read reference id of Pooled batches): that
         amplicon's segment of the count block is the new reference's segment;
      B. H alone, bound to reference 0 with no score threshold and no --discard_indel_reads: reference 0's all_* rows are what
         the HDR / prime-editing re-projection (:4226-4272) adds for the new reference;
      2. the batch again with H's weights at zero: the block of the ordinary references."""
    res, _ = align_uniques(engine, None, counts, ref_names, refs, flags, weights=weights, packed=(buf, off), compact=True,
                           on_launch=on_launch)
    if scaffold is None:
        return res, None
    loc, seq = scaffold
    pe_idx = list(ref_names).index(PE_REF)
    res.scaffold = scaffold
    hits = res._scaffold_hits = scaffold_hits(res, pe_idx, loc, seq)
    extra = {"rawA": None, "rawB": None, "weight": 0, "pe_idx": pe_idx}
    if not hits.any():
        return res, extra
    idx = np.nonzero(hits)[0]
    bS, oS = _subset(buf, off, idx)
    wS = np.ascontiguousarray(np.asarray(weights, dtype=np.int32)[idx])
    zero = np.zeros(len(idx), dtype=np.int32)
    engine.counts_reset()
    engine.align_packed(bS, oS, count=zero, qweight=wS, ref_id=np.full(len(idx), pe_idx, dtype=np.int32), compact=True)
    extra["rawA"] = engine.counts_raw()
    refs_b = dict(refs)
    refs_b[ref_names[0]] = dict(refs[ref_names[0]], min_aln_score=-1.0)
    engine.configure(refs_b, ref_names, aln_matrix, args.needleman_wunsch_gap_open, args.needleman_wunsch_gap_extend,
                     args.aln_seed_count, args.aln_seed_min, flags & ~_lib.F_DISCARD_INDEL_READS, "ACGTN", engine.edit_cap)
    engine.counts_reset()
    engine.align_packed(bS, oS, count=zero, qweight=wS, ref_id=np.zeros(len(idx), dtype=np.int32), compact=True)
    extra["rawB"] = engine.counts_raw()
    extra["weight"] = int(wS.astype(np.int64).sum())
    configure_engine(engine, args, refs, ref_names, aln_matrix)
    engine.counts_reset()
    w2 = np.array(weights, dtype=np.int32)
    w2[hits] = 0
    res, _ = align_uniques(engine, None, counts, ref_names, refs, flags, weights=w2, packed=(buf, off), compact=True)
    res.scaffold, res._scaffold_hits = scaffold, hits
    return res, extra


def _complete_edit_lists(engine, res, buf, off, flags, ref_id=None):
    """Reads whose edit list overflowed the batch's cap: their counts are already in the block (only the LIST was
    truncated), so they are re-run with zero weights and a cap sized from the largest list, in slices of bounded memory.
    -> {read index: (BatchResult, index)}"""
    over = np.nonzero(res.recs["status"] & _lib.ST_EDIT_OVERFLOW)[0]
    if not len(over):
        return {}
    cap0 = engine.edit_cap
    need = int(res.alns["n_edits"][over].max())
    engine.set_edit_cap(need)
    fix = {}
    nr = res.alns.shape[1]
    step = max(1, (256 << 20) // max(1, nr * need * 8))
    try:
        for a in range(0, len(over), step):
            idx = over[a:a + step]
            lens = (off[idx + 1] - off[idx]).astype(np.int64)
            o2 = np.zeros(len(idx) + 1, dtype=np.int64)
            np.cumsum(lens, out=o2[1:])
            b2 = np.concatenate([buf[off[k]:off[k + 1]] for k in idx]) if len(idx) else np.zeros(0, np.uint8)
            zero = np.zeros(len(idx), dtype=np.int32)
            r2 = engine.align_packed(b2, o2, count=zero, qweight=zero, ref_id=None if ref_id is None else ref_id[idx], compact=True)
            r2.flags = flags
            for j, k in enumerate(idx.tolist()):
                fix[k] = (r2, j)
    finally:
        engine.set_edit_cap(cap0)
    return fix


_STAT_KEYS = ["N_TOT_READS", "N_CACHED_ALN", "N_CACHED_NOTALN", "N_COMPUTED_ALN", "N_COMPUTED_NOTALN", "N_GLOBAL_SUBS",
              "N_SUBS_OUTSIDE_WINDOW", "N_MODS_IN_WINDOW", "N_MODS_OUTSIDE_WINDOW", "N_READS_IRREGULAR_ENDS", "READ_LENGTH"]


def _serial_stats(res, counts, n_extra_notaln=0, extra_count=0, lib_path=None):
    """aln_stats of the serial branch (CRISPRessoCORE.py:1956-1999) from the per-read records, natively (c2b_serial_stats: one
    threaded pass): the statistics of an aligned unique read are those of its best_match_name (the LAST winner)."""
    L = _lib.load(lib_path)
    n, nr = res.alns.shape
    recs = np.ascontiguousarray(res.recs)
    alns = np.ascontiguousarray(res.alns)
    c = np.ascontiguousarray(counts, dtype=np.int32)
    out = np.zeros(11, dtype=np.int64)
    aligned = np.zeros(n, dtype=np.uint8)
    rc = L.c2b_serial_stats(recs.ctypes.data, alns.ctypes.data, c.ctypes.data, n, nr, out.ctypes.data, aligned.ctypes.data, 0)
    if rc != 0:
        raise EngineError("c2b_serial_stats failed (%d)" % rc)
    st = dict(zip(_STAT_KEYS, (int(x) for x in out)))
    st["N_TOT_READS"] += int(extra_count)
    st["N_COMPUTED_NOTALN"] += int(n_extra_notaln)
    st["N_CACHED_NOTALN"] += int(extra_count) - int(n_extra_notaln)
    return st, aligned.view(bool)


def _joined_classes(res, weights, ref_names, flags):
    """class_counts entries of reads with several best references under --expand_ambiguous_alignments: their label is the
    '&'-joined list of '<ref>_<classification>' (CRISPRessoCORE.py:762-785), grouped here by (winner set, classifications)."""
    if not (flags & _lib.F_EXPAND_AMBIGUOUS) or (flags & _lib.F_ASSIGN_FIRST) or res.alns.shape[1] < 2:
        return {}
    w = np.asarray(weights, dtype=np.int64)
    pick = np.nonzero((res.recs["n_winners"] > 1) & (res.recs["best_score_milli"] > 0) & (w > 0))[0]
    out = {}
    if not len(pick):
        return out
    mask = res.recs["winner_mask"][pick].astype(np.int64)
    mod = np.zeros(len(pick), dtype=np.int64)
    for r in range(res.alns.shape[1]):
        mod |= (res.alns[pick, r]["modified"].astype(np.int64) != 0).astype(np.int64) << r
    key = mask | ((mod & mask) << 32)
    for kv in np.unique(key):
        m, md = int(kv) & 0xffffffff, int(kv) >> 32
        label = "&".join(ref_names[r] + ("_MODIFIED" if (md >> r) & 1 else "_UNMODIFIED") for r in range(len(ref_names)) if (m >> r) & 1)
        out[label] = int(w[pick][key == kv].sum())
    return out


def process_fastq(fastq_filename, variantCache, ref_names, refs, args, files_to_remove, output_directory,
                  engine=None, aln_matrix=None, on_out_of_contract="not_aligned"):
    """Drop-in for CRISPRessoCORE.process_fastq (:1735-2000).  The per-unique-read dicts are LazyVariant objects (lazy.py):
    nothing per read is built in Python until somebody reads it.
    on_out_of_contract: what to do with unique reads the engine cannot take (empty, > 512 bp, symbols outside ACGTN):
    "not_aligned" (default) files them under not_aligned_variants with best_match_score -1 and logs their number; "error"
    raises EngineError before anything is launched."""
    from . import lazy
    _unsupported(args, refs)
    if aln_matrix is None:
        loc = args.needleman_wunsch_aln_matrix_loc
        if not os.path.isabs(loc) and not os.path.exists(loc):
            raise FileNotFoundError("needleman_wunsch_aln_matrix_loc %r not found (pass an absolute path)" % loc)
        aln_matrix = read_matrix(loc)
    engine = engine or get_engine()
    # FASTQ read + dedup of CRISPRessoCORE.py:1820-1849, done natively (c2b_fastq_dedup: threads, exact); the packed
    # unique sequences feed the batch call directly
    import time
    t0 = time.perf_counter()
    dd = fastq.dedup_for_process_fastq(fastq_filename, engine.device, engine.lib_path)
    last_timings.clear()
    last_timings["ingest_dedup"] = time.perf_counter() - t0
    last_timings["n_reads"], last_timings["n_unique"] = int(dd.n_reads), int(len(dd.counts))
    t0 = time.perf_counter()
    if not variantCache:
        buf, off, counts = dd.buf, dd.off, dd.counts
        keys = None                                         # made while the GPU batch runs (_process_uniques)
    else:                                                   # caller pre-seeded the cache: same += semantics, same key order
        for seq, c in zip(dd.uniques, dd.counts.tolist()):
            variantCache[seq] = variantCache.get(seq, 0) + c
        keys = list(variantCache.keys())
        counts = np.asarray([variantCache[s] for s in keys], dtype=np.int32)
        buf, off = pack_reads([s.encode("utf-8", errors="surrogateescape") for s in keys])
    return _process_uniques(engine, buf, off, counts, keys, variantCache, ref_names, refs, args, aln_matrix, on_out_of_contract)


def _result_arrays(res):
    return {"recs": res.recs, "alns": res.alns, "ops": res.ops, "meta": res.meta, "edits": res.edits, "W": res.W,
            "buf": res._buf, "off": res._off}


def _result_from(engine, d, flags):
    from .engine import BatchResult
    r = BatchResult(d["recs"], d["alns"], None, d["edits"], d["W"], ops=d["ops"], meta=d["meta"], engine=engine, buf=d["buf"], off=d["off"])
    r.flags = flags
    return r


def _process_uniques(engine, buf, off, counts, keys, variantCache, ref_names, refs, args, aln_matrix, on_out_of_contract,
                     group=None):
    """The batch over the unique reads and everything after it.  With a torch.distributed `group` (one process per GPU) every
    rank aligns its contiguous slice of the unique reads (the reference's own sharding rule, CRISPRessoCORE.py:1172-1195), the
    count blocks meet in ONE all-reduce, the compact per-read results are gathered, and every rank ends with what the
    single-process call produces."""
    from . import lazy
    import logging
    import time
    t_start = time.perf_counter()
    n = len(off) - 1
    flags = _flags(args)
    scaffold = scaffold_search(args, refs)
    configure_engine(engine, args, refs, ref_names, aln_matrix)
    engine.counts_reset()
    bad = screen_reads(buf, off, lib_path=engine.lib_path) if n else np.zeros(0, dtype=bool)
    n_bad = int(bad.sum())
    if n_bad:
        k = int(np.nonzero(bad)[0][0])
        first = bytes(buf[off[k]:off[k + 1]][:40]).decode("utf-8", errors="replace")
        msg = ("%d unique read(s) (%d reads) are outside the engine's contract (empty, longer than %d bp, or symbols other than "
               "ACGTN), first: %r" % (n_bad, int(counts[bad].sum()), _lib.MAX_READ_LEN, first))
        if on_out_of_contract == "error":
            raise EngineError(msg)
        logging.getLogger("CRISPResso2").warning("crispresso2_b200: %s -- filed under not-aligned reads", msg)
        good = np.nonzero(~bad)[0]
        lens = (off[good + 1] - off[good]).astype(np.int64)
        o2 = np.zeros(len(good) + 1, dtype=np.int64)
        np.cumsum(lens, out=o2[1:])
        keep = np.repeat(~bad, np.diff(off))
        buf_g, off_g, counts_g = buf[keep], o2, np.ascontiguousarray(counts[good])
    else:
        buf_g, off_g, counts_g = buf, off, counts
    ng = len(off_g) - 1

    def key_lists():
        """the unique reads as Python strings (variantCache keys): all of them, and the ones the engine takes"""
        t0 = time.perf_counter()
        ks = keys if keys is not None else lazy.make_keys(buf, off)
        last_timings["keys"] = time.perf_counter() - t0
        return ks, ([ks[k] for k in good.tolist()] if n_bad else ks)

    weights = merge_weights_packed(buf_g, off_g, counts_g, lib_path=engine.lib_path)     # needs the global unique table: before sharding
    last_timings["screen_rc_merge"] = time.perf_counter() - t_start
    t_gpu = time.perf_counter()
    if group is None:
        # the batch call spends its time inside the library (GIL released): the key strings are made meanwhile
        import threading
        box = {}
        launched = threading.Event()                        # set when the batch thread is about to enter the library: key creation
                                                            # holds the GIL in one long native call and would otherwise run FIRST

        def batch():
            try:
                box["res"], box["extra"] = _batch(engine, buf_g, off_g, counts_g, weights, ref_names, refs, flags, args, aln_matrix,
                                                  scaffold, on_launch=launched.set)
            except BaseException as ex:                     # noqa: BLE001 -- re-raised on the calling thread
                box["err"] = ex
            finally:
                launched.set()

        th = threading.Thread(target=batch)
        th.start()
        launched.wait()
        keys, keys_g = key_lists()
        th.join()
        if "err" in box:
            raise box["err"]
        res, sc_extra = box["res"], box["extra"]
        parts = [(0, res, _complete_edit_lists(engine, res, buf_g, off_g, flags))]
        raw = None
    else:
        keys, keys_g = key_lists()
        import torch.distributed as dist
        from . import dist as cdist
        rank, world = dist.get_rank(group), dist.get_world_size(group)
        lo, hi = cdist.shard_bounds(ng, rank, world)
        mine = None
        sc_extra = None
        if hi > lo:
            b0, b1 = int(off_g[lo]), int(off_g[hi])
            sb, so = np.ascontiguousarray(buf_g[b0:b1]), np.ascontiguousarray(off_g[lo:hi + 1] - b0)
            res, sc_extra = _batch(engine, sb, so, counts_g[lo:hi], weights[lo:hi], ref_names, refs, flags, args, aln_matrix, scaffold)
            fix = _complete_edit_lists(engine, res, sb, so, flags)
            mine = {"lo": lo, "res": _result_arrays(res), "fix": {k: (_result_arrays(r2), j) for k, (r2, j) in fix.items()}}
        raw = cdist.allreduce_counts(engine, group)          # the path's one collective on device data
        if scaffold is not None:                             # the scaffold reference's segments: summed over ranks like the block
            size = len(raw)
            sc_extra = sc_extra or {"rawA": None, "rawB": None, "weight": 0, "pe_idx": list(ref_names).index(PE_REF)}
            both = np.zeros(2 * size + 1, dtype=np.int64)
            if sc_extra["rawA"] is not None:
                both[:size], both[size:2 * size], both[-1] = sc_extra["rawA"], sc_extra["rawB"], sc_extra["weight"]
            both = cdist.allreduce_array(both, engine, group)
            sc_extra = dict(sc_extra, rawA=both[:size], rawB=both[size:2 * size], weight=int(both[-1]))
        gathered = [None] * world
        dist.all_gather_object(gathered, mine, group=group)
        parts = []
        for g in gathered:
            if g is None:
                continue
            cache_r2 = {}
            fx = {}
            for k, (d, j) in g["fix"].items():
                if id(d) not in cache_r2:
                    cache_r2[id(d)] = _result_from(engine, d, flags)
                fx[k] = (cache_r2[id(d)], j)
            parts.append((g["lo"], _result_from(engine, g["res"], flags), fx))
    last_timings["gpu_batch"] = time.perf_counter() - t_gpu
    t_tab = time.perf_counter()
    # serial-branch statistics, part by part (rank order = unique order)
    st = dict.fromkeys(_STAT_KEYS, 0)
    aligned = np.zeros(ng, dtype=bool)
    extra = {}
    for lo, res, _fx in parts:
        hi = lo + len(res.recs)
        w_part = weights[lo:hi]
        if scaffold is not None:                            # re-labelled reads carry the scaffold class, nothing else
            res.scaffold = scaffold
            for r2, _j in _fx.values():
                r2.scaffold = scaffold
            h = getattr(res, "_scaffold_hits", None)
            if h is None:
                h = scaffold_hits(res, list(ref_names).index(PE_REF), scaffold[0], scaffold[1])
            w_part = np.where(h, 0, w_part)
        s1, al = _serial_stats(res, counts_g[lo:hi], lib_path=engine.lib_path)
        aligned[lo:hi] = al
        for key, val in s1.items():
            if key == "READ_LENGTH":
                st[key] = st[key] or val
            else:
                st[key] += val
        for lab, val in _joined_classes(res, w_part, ref_names, flags).items():
            extra[lab] = extra.get(lab, 0) + val
    if n_bad:
        cb = int(counts[bad].sum())
        st["N_TOT_READS"] += cb
        st["N_COMPUTED_NOTALN"] += n_bad
        st["N_CACHED_NOTALN"] += cb - n_bad
    src = lazy.BatchSource(None, keys_g, ref_names, refs, counts_g, parts=parts)
    src.weights, src.flags, src.lib_path, src.scaffold = weights, flags, engine.lib_path, scaffold
    src.engine, src.packed_all, src.good = engine, (buf, off), (good if n_bad else None)     # annotate.py
    _sources[id(variantCache)] = src
    cls = src.lazy_class()
    not_aligned = {}
    sel = aligned.astype(np.uint8)
    lazy.fill_cache(variantCache, keys_g, sel, counts_g, cls, 1)          # pre-seeded cache: counts replaced in place, order kept
    lazy.fill_cache(not_aligned, keys_g, sel, counts_g, cls, 0)
    for seq in not_aligned:
        variantCache.pop(seq, None)
    if n_bad:
        for k in np.nonzero(bad)[0].tolist():
            not_aligned[keys[k]] = {"count": int(counts[k]), "aln_scores": [], "ref_aln_details": [], "best_match_score": -1}
            variantCache.pop(keys[k], None)
    block = engine.counts(raw=raw)
    if scaffold is not None:
        block.add_scaffold_reference(SCAFFOLD_REF, refs[PE_REF]["sequence"], sc_extra["pe_idx"], sc_extra["rawA"], sc_extra["rawB"],
                                     sc_extra["weight"])
    dev = block.aln_stats_partial()                         # the kernel's own sums must agree with the records
    for key, val in dev.items():
        if val != st[key]:
            raise EngineError("device aln_stats disagree with per-read records for %s: %d != %d" % (key, val, st[key]))
    for lab, val in extra.items():
        block.class_extra[lab] = block.class_extra.get(lab, 0) + val
    _blocks[id(variantCache)] = block
    last_timings["stats_cache"] = time.perf_counter() - t_tab
    return st, not_aligned


def process_fastq_sharded(fastq_filename, variantCache, ref_names, refs, args, files_to_remove, output_directory,
                          engine=None, aln_matrix=None, group=None, on_out_of_contract="not_aligned"):
    """process_fastq for one process per GPU (torch.distributed initialised): same arguments, same results on every rank.
    Without an explicit engine the rank uses the GPU named by LOCAL_RANK (torchrun) -- never all ranks on device 0."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size(group) == 1:
        return process_fastq(fastq_filename, variantCache, ref_names, refs, args, files_to_remove, output_directory,
                             engine=engine, aln_matrix=aln_matrix, on_out_of_contract=on_out_of_contract)
    from . import lazy
    _unsupported(args, refs)
    if aln_matrix is None:
        aln_matrix = read_matrix(args.needleman_wunsch_aln_matrix_loc)
    if engine is None:
        dev = int(os.environ.get("LOCAL_RANK", "0"))
        if dist.get_backend(group) == "nccl":
            import torch
            torch.cuda.set_device(dev)
        engine = get_engine(dev)
    dd = fastq.dedup_for_process_fastq(fastq_filename, engine.device, engine.lib_path)
    if not variantCache:
        buf, off, counts = dd.buf, dd.off, dd.counts
        keys = None
    else:
        for seq, c in zip(dd.uniques, dd.counts.tolist()):
            variantCache[seq] = variantCache.get(seq, 0) + c
        keys = list(variantCache.keys())
        counts = np.asarray([variantCache[s] for s in keys], dtype=np.int32)
        buf, off = pack_reads([s.encode("utf-8", errors="surrogateescape") for s in keys])
    world_group = group if group is not None else dist.group.WORLD
    return _process_uniques(engine, buf, off, counts, keys, variantCache, ref_names, refs, args, aln_matrix, on_out_of_contract,
                            group=world_group)


def source_of(variantCache):
    """Compact results (lazy.BatchSource) of the process_fastq call that filled this variantCache."""
    try:
        return _sources[id(variantCache)]
    except KeyError:
        raise KeyError("this variantCache was not filled by crispresso2_b200.core.process_fastq") from None


def quantify(variantCache):
    """Count block accumulated on the device by the process_fastq call that filled this variantCache."""
    return _blocks[id(variantCache)]


def get_new_variant_object(args, fastq_seq, refs, ref_names, aln_matrix, pe_scaffold_dna_info=None, engine=None):
    _unsupported(args, refs)
    engine = engine or get_engine()
    configure_engine(engine, args, refs, ref_names, aln_matrix, edit_cap=max(len(refs[r]["sequence"]) for r in ref_names)
                     + len(fastq_seq) + 1)
    res, _ = align_uniques(engine, [fastq_seq], [1], ref_names, refs, _flags(args), weights=[0])
    if getattr(args, "prime_editing_pegRNA_scaffold_seq", ""):
        res.scaffold = tuple(pe_scaffold_dna_info)
    return _variant_from(res, 0, fastq_seq, ref_names, refs)

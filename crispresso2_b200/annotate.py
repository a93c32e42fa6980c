"""Annotated read outputs: CRISPResso's --fastq_output and --bam_output without a per-read Python loop.

Same call signatures and return values as the reference functions they stand in for:
  process_fastq_write_out(fastq_input, fastq_output, variantCache, ref_names, refs, args, files_to_remove, output_directory)
      -> (aln_stats, not_aligned_variants)                        CRISPRessoCORE.py:2283-2348
  process_single_fastq_write_bam_out(fastq_input, bam_output, bam_header, variantCache, ref_names, refs, args, files_to_remove,
                                     output_directory)
      -> (aln_stats, not_aligned_variants)                        CRISPRessoCORE.py:2351-2514
Both first call `process_fastq` (keyword argument; the engine's core.process_fastq by default), whose variantCache must be the
engine's lazy cache.  The annotation text of every unique read -- and the CIGAR / flag / MAPQ of its first aligned reference --
is built on the GPU from the batch's compact results (c2b_annotate_build, csrc/c2b_annotate.cuh); the host derives only the
labels it already knows (class_name, the names after the prime-editing scaffold re-labelling) as small ids.  The records are
then written by host threads (c2b_annotate_write_fastq / _sam): the FASTQ as a multi-member gzip file whose decompressed bytes
are the reference's, the SAM as text, sorted and indexed by `samtools` as in the reference.

The cache entries receive 'crispresso2_annotation' / 'sam_entry' as the reference sets them (last in key order, same values),
when they materialise: nothing per read is built in Python during the write.
"""
import ctypes as C
import logging
import os
import subprocess

import numpy as np

from . import _lib, core
from .core import PE_REF, SCAFFOLD_REF

_log = logging.getLogger("CRISPResso2")


def _bad_parameter(msg):
    try:
        from CRISPResso2 import CRISPRessoShared
        return CRISPRessoShared.BadParameterException(msg)
    except ImportError:                                         # the reference's exception when it is installed
        return RuntimeError(msg)


def _comp256():
    """the engine's complement of the alphabet ACGTN (reads aligned as their reverse complement), identity elsewhere"""
    t = np.arange(256, dtype=np.uint8)
    for a, b in ("AT", "TA", "CG", "GC"):
        t[ord(a)] = ord(b)
    return t


def _label(ref_names, wm, md, flags):
    """class_name of an aligned read from its winners and their classifications (CRISPRessoCORE.py:762-785)"""
    win = [r for r in range(len(ref_names)) if (wm >> r) & 1]
    labels = [ref_names[r] + ("_MODIFIED" if (md >> r) & 1 else "_UNMODIFIED") for r in win]
    if len(win) > 1:
        if flags & _lib.F_ASSIGN_FIRST:
            return labels[0]
        if not flags & _lib.F_EXPAND_AMBIGUOUS:
            return "AMBIGUOUS"
    return "&".join(labels)


def _cstrings(items):
    arr = (C.c_char_p * max(1, len(items)))(*[s.encode() for s in items])
    return arr


class Annotation:
    """Per-unique-read annotations of the process_fastq call that filled `variantCache` (one GPU pass, host arena)."""

    def __init__(self, variantCache, refs, sam_strands=False, chunk=0, sam_optional=False):
        """sam_optional: the text of process_bam (C2B_ANN_SAM_OPTIONAL): "c2:Z:" first, no scores / details for aligned reads"""
        src = core.source_of(variantCache)
        if len(src.parts) != 1:
            raise NotImplementedError("annotated outputs of a run sharded over several processes are not built")
        self.src = src
        _, res, fix = src.parts[0]
        if res.ops is None or res.edits is None:
            raise ValueError("the batch holds no compact results")
        ref_names = list(src.ref_names)
        R = res.alns.shape[1]
        recs, alns, edits = res.recs, res.alns, res.edits
        if fix:                                                 # reads re-run with complete edit lists (core._complete_edit_lists)
            cap = max([edits.shape[2]] + [r2.edits.shape[2] for r2, _ in fix.values()])
            e2 = np.zeros((len(recs), R, cap), dtype=_lib.EDIT_DTYPE)
            e2[:, :, :edits.shape[2]] = edits
            alns = alns.copy()
            for k, (r2, j) in fix.items():
                e2[k, :, :r2.edits.shape[2]] = r2.edits[j]
                alns[k] = r2.alns[j]
            edits = e2
        flags = int(src.flags)
        # aln_ref_names: the winners, the first one only under --assign_ambiguous_alignments_to_first_reference
        wm = np.where(recs["best_score_milli"] > 0, recs["winner_mask"], 0).astype(np.uint32)
        amask = (wm & (~wm + np.uint32(1))) if flags & _lib.F_ASSIGN_FIRST else wm.copy()
        mod = np.zeros(len(recs), dtype=np.uint64)
        for r in range(R):
            mod |= (alns[:, r]["modified"] != 0).astype(np.uint64) << np.uint64(r)
        key = wm.astype(np.uint64) | ((mod & wm.astype(np.uint64)) << np.uint64(32))
        ukeys, inv = np.unique(key, return_inverse=True)
        labels = [_label(ref_names, int(kv) & 0xffffffff, int(kv) >> 32, flags) for kv in ukeys.tolist()]
        label = inv.astype(np.int32).reshape(-1)
        names = ref_names + [SCAFFOLD_REF]
        aname = np.full(len(recs), -1, dtype=np.int16)
        hits = getattr(res, "_scaffold_hits", None) if src.scaffold is not None else None
        if hits is not None and hits.any():                     # CRISPRessoCORE.py:789-796: re-labelled to the scaffold reference
            pe = ref_names.index(PE_REF)
            amask[hits] = np.uint32(1 << pe)
            aname[hits] = len(ref_names)
            label[hits] = len(labels)
            labels.append(SCAFFOLD_REF)
        self.names = names
        rev = np.zeros(len(names), dtype=np.uint8)
        if sam_strands:
            for i, nm in enumerate(names):
                if nm in refs and refs[nm].get("aln_strand") == "-":
                    rev[i] = 1
        self.rev = rev
        buf, off = src.packed_all
        n = len(off) - 1
        kidx = np.arange(n, dtype=np.int64) if src.good is None else np.asarray(src.good, dtype=np.int64)
        bidx = np.full(n, -1, dtype=np.int32)
        bidx[kidx] = np.arange(len(kidx), dtype=np.int32)
        self.kidx, self.buf, self.off, self.n = kidx, np.ascontiguousarray(buf, dtype=np.uint8), np.ascontiguousarray(off, dtype=np.int64), n
        self.aligned = amask != 0
        seqs = [refs[nm]["sequence"] for nm in ref_names]
        lens = np.asarray([len(s) for s in seqs], dtype=np.int32)
        recs, alns, ops = np.ascontiguousarray(recs), np.ascontiguousarray(alns), np.ascontiguousarray(res.ops)
        meta, edits = np.ascontiguousarray(res.meta), np.ascontiguousarray(edits)
        amask, label = np.ascontiguousarray(amask), np.ascontiguousarray(label)
        comp = _comp256()
        eng = src.engine
        if not eng.h:                                           # the pass runs on the engine's device; its configuration is not read
            raise core.EngineError("c2b_annotate_build: the engine that ran this batch was closed")
        L = self.L = eng.L
        h = C.c_void_p()
        NW = ops.shape[2]
        rc = L.c2b_annotate_build(eng.h, self.buf.ctypes.data if len(self.buf) else None, self.off.ctypes.data, n, bidx.ctypes.data,
                                  R, NW, edits.shape[2], recs.ctypes.data, alns.ctypes.data, ops.ctypes.data, meta.ctypes.data,
                                  edits.ctypes.data, amask.ctypes.data, aname.ctypes.data, label.ctypes.data,
                                  len(names), _cstrings(names), rev.ctypes.data, len(labels), _cstrings(labels),
                                  _cstrings(seqs), lens.ctypes.data, comp.ctypes.data,
                                  (flags & _lib.F_LEGACY_INS) | (_lib.ANN_SAM_OPTIONAL if sam_optional else 0), int(chunk), C.byref(h))
        if rc != 0:
            raise core.EngineError("c2b_annotate_build failed (%d): %s" % (rc, L.c2b_last_error(eng.h).decode()))
        self.h = h
        self.ann_off = self._view("c2b_annotate_offsets", C.c_int64, n + 1)
        self.arena = self._view("c2b_annotate_arena", C.c_uint8, int(self.ann_off[-1]))
        self.last_rec = None

    def _view(self, fn, ct, count):
        """numpy view of an array the handle owns (lives as long as this object)"""
        p = getattr(self.L, fn)(self.h)
        if not count or not p:
            return np.zeros(count, dtype=np.dtype(ct))
        return np.ctypeslib.as_array(C.cast(p, C.POINTER(ct)), shape=(count,))

    def __del__(self):
        h, self.h = getattr(self, "h", None), None
        if h:
            self.L.c2b_annotate_free(h)

    def text(self, u):
        """annotation of unique read u (the FASTQ form: leading space; the process_bam form: "c2:Z:" first)"""
        return self.arena[self.ann_off[u]:self.ann_off[u + 1]].tobytes().decode("ascii")

    # ---------------------------------------------------------------------------------------------------- writers
    def write_fastq(self, fastq_input, fastq_output):
        rc = self.L.c2b_annotate_write_fastq(self.h, self.buf.ctypes.data if len(self.buf) else None, self.off.ctypes.data, self.n,
                                             os.fsencode(fastq_input), os.fsencode(fastq_output), 0)
        if rc != 0:
            raise core.EngineError("c2b_annotate_write_fastq failed (%d): %s" % (rc, self.L.c2b_fastq_last_error().decode()))

    def write_sam(self, fastq_input, sam_out, bam_header, refs):
        first = self._view("c2b_annotate_first", C.c_int16, self.n)
        used = set(np.unique(first[first >= 0]).tolist()) if self.n else set()
        chr_, pos = [], []
        for i, nm in enumerate(self.names):
            if i in used:
                chr_.append(str(refs[nm]["aln_chr"]))             # KeyError like the reference's refs[first_ref_name] lookups
                pos.append(str(refs[nm]["aln_start"]))
            else:
                chr_.append("")
                pos.append("")
        rc = self.L.c2b_annotate_write_sam(self.h, self.buf.ctypes.data if len(self.buf) else None, self.off.ctypes.data, self.n,
                                           os.fsencode(fastq_input), os.fsencode(sam_out), bam_header.encode(), len(self.names),
                                           _cstrings(chr_), _cstrings(pos), self.rev.ctypes.data, 0)
        if rc != 0:
            raise core.EngineError("c2b_annotate_write_sam failed (%d): %s" % (rc, self.L.c2b_fastq_last_error().decode()))
        self.chr, self.pos = chr_, pos
        self.last_rec = self._view("c2b_annotate_last_record", C.c_int64, self.n)
        self.rec_off = self._view("c2b_annotate_record_offsets", C.c_int64, 2 * self.n + 1)
        self.rec = self._view("c2b_annotate_record_arena", C.c_uint8, int(self.rec_off[-1]))
        cig_off = self._view("c2b_annotate_cigar_offsets", C.c_int64, self.n + 1)
        self.cig_off, self.cig = cig_off, self._view("c2b_annotate_cigar_arena", C.c_uint8, int(cig_off[-1]))
        self.flag = self._view("c2b_annotate_flags", C.c_uint8, self.n)
        self.mapq = self._view("c2b_annotate_mapq", C.c_int32, self.n)
        self.first = first

    def write_sam_passthrough(self, text, sam_out):
        """pass 2 of process_bam: the lines of `text` (SAM, bytes) whose read is a unique read here, with their annotation,
        appended to sam_out"""
        arr = np.frombuffer(text, dtype=np.uint8)
        rc = self.L.c2b_annotate_write_sam_passthrough(self.h, self.buf.ctypes.data if len(self.buf) else None, self.off.ctypes.data,
                                                       self.n, arr.ctypes.data if len(arr) else None, len(arr), os.fsencode(sam_out), 0)
        if rc == _lib.E_LIMIT:
            raise IndexError("list index out of range: %s" % self.L.c2b_fastq_last_error().decode())
        if rc != 0:
            raise core.EngineError("c2b_annotate_write_sam_passthrough failed (%d): %s" % (rc, self.L.c2b_fastq_last_error().decode()))

    # ---------------------------------------------------------------------------------------------------- cache entries
    def annotation_of(self, k):
        """'crispresso2_annotation' of batch read k (aligned reads only, CRISPRessoCORE.py:2343)"""
        return self.text(int(self.kidx[k])) if self.aligned[k] else None

    def sam_entry_of(self, k):
        """'sam_entry' of batch read k: the field list of its last SAM line (CRISPRessoCORE.py:2471-2497)"""
        if not self.aligned[k]:
            return None
        u = int(self.kidx[k])
        if self.last_rec[u] < 0:
            return None
        ro = self.rec_off
        rid = self.rec[ro[2 * u]:ro[2 * u + 1]].tobytes().decode("ascii")
        qual = self.rec[ro[2 * u + 1]:ro[2 * u + 2]].tobytes().decode("ascii")
        seq = self.src.keys[k]
        f = int(self.first[u])
        if self.rev[f]:
            seq, qual = core.reverse_complement(seq), qual[::-1]
        return [rid, str(int(self.flag[u])), self.chr[f], self.pos[f], str(int(self.mapq[u])),
                self.cig[self.cig_off[u]:self.cig_off[u + 1]].tobytes().decode("ascii"), "*", "0", "0", seq, qual,
                "c2:Z:" + self.text(u)[1:]]

    def attach(self, variantCache, key, value_of, also=()):
        """variantCache entries (and those of the dicts in `also`, filled by the same call: not_aligned_variants) get `key` when
        they materialise; entries already materialised get it now"""
        src = self.src
        src.extra_keys.append((key, value_of))
        if src.n_filled:
            for v in (v for d in (variantCache,) + tuple(also) for v in d.values()):
                k = getattr(v, "_k", -1)
                if k < -1:
                    val = value_of(-2 - k)
                    if val is not None:
                        dict.__setitem__(v, key, val)


def process_fastq_write_out(fastq_input, fastq_output, variantCache, ref_names, refs, args, files_to_remove, output_directory,
                            process_fastq=None):
    """Drop-in for CRISPRessoCORE.process_fastq_write_out (:2283-2348)."""
    process_fastq = process_fastq or core.process_fastq
    aln_stats, not_aln = process_fastq(fastq_input, variantCache, ref_names, refs, args, files_to_remove, output_directory)
    _log.info("Reads processed, now annotating fastq_output file: %s" % (fastq_output))
    A = Annotation(variantCache, refs)
    A.write_fastq(fastq_input, fastq_output)
    A.attach(variantCache, "crispresso2_annotation", A.annotation_of)
    return aln_stats, not_aln


def process_single_fastq_write_bam_out(fastq_input, bam_output, bam_header, variantCache, ref_names, refs, args, files_to_remove,
                                       output_directory, process_fastq=None):
    """Drop-in for CRISPRessoCORE.process_single_fastq_write_bam_out (:2351-2514): the SAM text natively, then the reference's
    `samtools sort` / `samtools index` command."""
    process_fastq = process_fastq or core.process_fastq
    aln_stats, not_aln = process_fastq(fastq_input, variantCache, ref_names, refs, args, files_to_remove, output_directory)
    _log.info("Reads processed, now annotating fastq_output file: %s" % (bam_output))
    A = Annotation(variantCache, refs, sam_strands=True)
    sam_out = bam_output + ".sam"
    A.write_sam(fastq_input, sam_out, bam_header, refs)
    A.attach(variantCache, "sam_entry", A.sam_entry_of)
    sort_and_index_cmd = 'samtools sort ' + sam_out + ' -o ' + bam_output + ' && samtools index ' + bam_output
    if subprocess.call(sort_and_index_cmd, shell=True):
        raise _bad_parameter('Bam sort failed. Command used: {0}'.format(sort_and_index_cmd))
    if not args.debug:
        os.remove(sam_out)
    _log.info("Finished writing out to bam file: %s" % (bam_output))
    return aln_stats, not_aln

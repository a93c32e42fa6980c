"""--bam_input: CRISPResso's process_bam without a per-read Python loop.

Same call signature and return value as the reference function it stands in for:
  process_bam(bam_filename, bam_chr_loc, output_bam, variantCache, ref_names, refs, args, files_to_remove, output_directory)
      -> (aln_stats, not_aln)                                         CRISPRessoCORE.py:2003-2280
plus engine= / aln_matrix= / on_out_of_contract= as core.process_fastq has them.

The SAM text comes from the user's `samtools`, with the reference's argv lists: `view -H` for the header, `view -F <flags>` for
pass 1 and `view` without -F for pass 2 (region appended when given).  The three processes start at once; a host thread drains
pass 2 into memory while pass 1 goes through the SAM front end (field 10 of every line, exact dedup in first-seen order, on the
GPU by the same rule as process_fastq's front end: fastq.dedup_for_process_bam) and the engine batch (core._process_uniques, as
process_fastq runs it: the reference's single-process branch).  The annotation of every unique read is built on the GPU in the
form of process_bam (annotate.Annotation, sam_optional=True) and the pass-2 lines are written natively by host threads
(c2b_annotate_write_sam_passthrough).  Both passes read the same file, so the output is what the sequential order gives.

As in the reference, `output_bam` itself is not written: the result is `output_bam + ".sam"`, unsorted and unindexed.
"""
import logging
import os
import subprocess
import sys
import threading
import time

import numpy as np

from . import annotate, core, fastq

_log = logging.getLogger("CRISPResso2")

SAM_NA = "c2:Z:ALN=NA ALN_SCORES= ALN_DETAILS="                 # reads outside the engine's contract (filed as not aligned)
last_timings = {}


def _universal_newlines(data):
    """bytes of a text-mode pipe as the reference reads them (encoding='utf-8', universal newlines)"""
    return data.decode("utf-8").replace("\r\n", "\n").replace("\r", "\n")


def _version():
    from CRISPResso2 import CRISPRessoShared                     # the reference's own version string goes into @PG
    return CRISPRessoShared.__version__


def _global_subs_quirk(st, src):
    """N_GLOBAL_SUBS of process_bam's serial branch (CRISPRessoCORE.py:2241): substitution_n + substitutions_outside_window *
    count per aligned unique read, where process_fastq weights both terms -- corrected from the per-read records"""
    _, res, _ = src.parts[0]
    recs, alns = res.recs, res.alns
    n, nr = alns.shape
    if not n:
        return
    col = recs["best_ref"].astype(np.int64) if nr > 1 else np.zeros(n, dtype=np.int64)
    col = np.where((col < 0) | (col >= nr), 0, col)             # the column c2b_serial_stats reads
    sub = alns["substitution_n"][np.arange(n), col].astype(np.int64)
    extra = (np.asarray(src.counts, dtype=np.int64) - 1) * sub
    st["N_GLOBAL_SUBS"] -= int(extra[recs["best_score_milli"] > 0].sum())


def process_bam(bam_filename, bam_chr_loc, output_bam, variantCache, ref_names, refs, args, files_to_remove, output_directory,
                engine=None, aln_matrix=None, on_out_of_contract="not_aligned"):
    """Drop-in for CRISPRessoCORE.process_bam (:2003-2280), single-process branch."""
    core._unsupported(args, refs, ref_names)
    if aln_matrix is None:
        loc = args.needleman_wunsch_aln_matrix_loc
        if not os.path.isabs(loc) and not os.path.exists(loc):
            raise FileNotFoundError("needleman_wunsch_aln_matrix_loc %r not found (pass an absolute path)" % loc)
        aln_matrix = core.read_matrix(loc)
    engine = engine or core.get_engine()
    last_timings.clear()
    t0 = time.perf_counter()
    region = [bam_chr_loc] if bam_chr_loc != "" else []
    head = subprocess.Popen(["samtools", "view", "-H", bam_filename], stdout=subprocess.PIPE, stderr=subprocess.PIPE)
    pass1 = subprocess.Popen(["samtools", "view", "-F", args.samtools_exclude_flags, bam_filename] + region, stdout=subprocess.PIPE)
    pass2 = subprocess.Popen(["samtools", "view", bam_filename] + region, stdout=subprocess.PIPE)
    box = {}

    def drain():
        try:
            box["text"] = pass2.stdout.read()
        finally:
            pass2.wait()

    th = threading.Thread(target=drain, daemon=True)
    th.start()
    try:
        header, _ = head.communicate()
        text1 = pass1.stdout.read()
        pass1.wait()
        output_sam = output_bam + ".sam"
        with open(output_sam, "w") as sam_out:
            sam_out.write(_universal_newlines(header))
            sam_out.write("@PG\tID:crispresso2\tPN:crispresso2\tVN:" + _version() + '\tCL:"' + " ".join(sys.argv) + '"\n')
        last_timings["pass1_text"] = time.perf_counter() - t0

        t0 = time.perf_counter()
        dd = fastq.dedup_for_process_bam(text1, engine.device, engine.lib_path)
        del text1
        last_timings["front_end"] = time.perf_counter() - t0
        last_timings["n_reads"], last_timings["n_unique"] = int(dd.n_reads), int(len(dd.counts))
        _log.info("Finished reading bam file; %d unique reads found of %d total reads found " % (len(dd.counts), dd.n_reads))
        if not variantCache:
            buf, off, counts = dd.buf, dd.off, dd.counts
            keys = None
        else:                                                   # caller pre-seeded the cache: += onto it, key order kept
            for seq, c in zip(dd.uniques, dd.counts.tolist()):
                variantCache[seq] = variantCache.get(seq, 0) + c
            keys = list(variantCache.keys())
            counts = np.asarray([variantCache[s] for s in keys], dtype=np.int32)
            buf, off = core.pack_reads([s.encode("utf-8", errors="surrogateescape") for s in keys])
        if len(off) == 1:
            # the reference's serial loop leaves its index unbound when there is no read, and reads it after the loop
            raise UnboundLocalError("cannot access local variable 'idx' where it is not associated with a value")

        t0 = time.perf_counter()
        st, not_aln = core._process_uniques(engine, buf, off, counts, keys, variantCache, ref_names, refs, args, aln_matrix,
                                            on_out_of_contract)
        src = core.source_of(variantCache)
        _global_subs_quirk(st, src)
        last_timings["batch"] = time.perf_counter() - t0

        t0 = time.perf_counter()
        A = annotate.Annotation(variantCache, refs, sam_optional=True)
        last_timings["annotate"] = time.perf_counter() - t0

        t0 = time.perf_counter()
        th.join()
        last_timings["pass2_wait"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        A.write_sam_passthrough(box["text"], output_sam)
        last_timings["writer"] = time.perf_counter() - t0
    finally:
        for p in (head, pass1, pass2):
            if p.poll() is None:
                p.kill()
                p.wait()
        th.join()
    A.attach(variantCache, "crispresso2_annotation", A.annotation_of, also=(not_aln,))
    A.attach(variantCache, "crispresso_sam_optional_fields",
             lambda k: None if A.aligned[k] else A.text(int(A.kidx[k])), also=(not_aln,))
    for v in not_aln.values():                                  # outside the engine's contract: plain dicts
        if type(v) is dict:
            v["crispresso_sam_optional_fields"] = SAM_NA
    _log.info("Finished reads; N_TOT_READS: %d N_COMPUTED_ALN: %d N_CACHED_ALN: %d N_COMPUTED_NOTALN: %d N_CACHED_NOTALN: %d" % (
        st["N_TOT_READS"], st["N_COMPUTED_ALN"], st["N_CACHED_ALN"], st["N_COMPUTED_NOTALN"], st["N_CACHED_NOTALN"]))
    return st, not_aln

"""Python face of the CUDA engine: packs the reference's `refs` / `args` into the C structs of
include/c2b200.h, calls the batch entry points and exposes results as numpy arrays.

No alignment or classification decision is taken here; this module only formats inputs (tabulating
aln_matrix look-ups per reference position, Align.pyx:212) and views outputs.
"""
import ctypes as C

import numpy as np

from . import _lib

_DNA_COMP = {"A": "T", "C": "G", "G": "C", "T": "A"}


class EngineError(RuntimeError):
    pass


class BatchResult:
    """Views over one batch's outputs.

    recs    : REC_DTYPE  [n]
    alns    : ALN_DTYPE  [n, R]            R = n_refs, or 1 when the batch carried a per-read ref_id (Pooled)
    strings : uint8      [n, R, 2, W]      (right-aligned; [.., 0, :] read, [.., 1, :] reference) or None
    edits   : EDIT_DTYPE [n, R, cap] or None
    ops/meta: compact form (c2b_align_batch_compact): uint64 [n, R, W/32] op streams, uint32 [n, R] meta words; the strings
              of any block of reads are rebuilt on demand by the library's host-side expansion (strings_block)
    A compact result owns what its expansion needs -- the configured reference sequences, the string width and the complement
    table the batch ran with (`tables`, Engine.tables) -- so it spells the same strings whatever its engine does afterwards:
    reconfigured for another run, used for a batch of another size, or closed.
    """

    def __init__(self, recs, alns, strings, edits, W, ops=None, meta=None, lib=None, buf=None, off=None, ref_id=None, tables=None):
        self.recs, self.alns, self.strings, self.edits, self.W = recs, alns, strings, edits, W
        self.ops, self.meta, self._lib, self._buf, self._off, self._ref_id = ops, meta, lib, buf, off, ref_id
        self.tables = tables
        if ops is not None:
            seqs, comp = tables
            self._c_seqs = (C.c_char_p * len(seqs))(*seqs)
            self._c_lens = np.asarray([len(x) for x in seqs], dtype=np.int32)
            self._c_comp = np.ascontiguousarray(comp, dtype=np.uint8)

    def strings_block(self, lo, hi):
        """uint8 [hi-lo, R, 2, W] aligned strings of reads lo..hi-1"""
        if self.strings is not None:
            return self.strings[lo:hi]
        off = np.ascontiguousarray(self._off[lo:hi + 1])
        rid = None if self._ref_id is None else np.ascontiguousarray(self._ref_id[lo:hi], dtype=np.int32)
        ops = np.ascontiguousarray(self.ops[lo:hi])
        meta = np.ascontiguousarray(self.meta[lo:hi])
        R = self.alns.shape[1]
        out = np.zeros((hi - lo, R, 2, self.W), dtype=np.uint8)
        rc = self._lib.c2b_expand_batch_tables(self._buf.ctypes.data, off.ctypes.data, hi - lo,
                                               rid.ctypes.data if rid is not None else None, ops.ctypes.data, meta.ctypes.data,
                                               R, self.W, len(self._c_lens), self._c_seqs, self._c_lens.ctypes.data,
                                               self._c_comp.ctypes.data, out.ctypes.data, 0)
        if rc != 0:
            raise EngineError("c2b_expand_batch_tables failed (%d): an op stream does not fit its read and reference" % rc)
        return out

    def pair(self, i, r=0):
        """(aligned_read, aligned_ref) of read i against reference r, as str."""
        n = int(self.alns[i, r]["aln_len"])
        s = self.strings_block(i, i + 1)[0, r]
        return s[0, self.W - n:].tobytes().decode(), s[1, self.W - n:].tobytes().decode()

    def score(self, i, r=0):
        """global_align's third return value (Align.pyx:433-434), exactly."""
        return int(self.alns[i, r]["score_milli"]) / 1000.0


def pack_reads(reads):
    """list of str/bytes -> (uint8 array, int64 offsets)"""
    bs = [r.encode() if isinstance(r, str) else bytes(r) for r in reads]
    off = np.zeros(len(bs) + 1, dtype=np.int64)
    if bs:
        np.cumsum([len(b) for b in bs], out=off[1:])
    buf = np.frombuffer(b"".join(bs), dtype=np.uint8) if bs else np.zeros(0, dtype=np.uint8)
    return buf, off


class Engine:
    def __init__(self, device=0, lib_path=None):
        self.L = _lib.load(lib_path)
        self.lib_path = lib_path
        h = C.c_void_p()
        rc = self.L.c2b_create(int(device), C.byref(h))
        if rc != 0:
            raise EngineError("c2b_create failed (%d): %s" % (rc, self.L.c2b_last_error(None).decode()))
        self.h = h
        self.device = device
        self.n_refs = 0
        self.alphabet = "ACGTN"
        self.edit_cap = 0
        self._keep = None
        self.tables = None

    def close(self):
        if getattr(self, "h", None):
            self.L.c2b_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc, what):
        if rc != 0:
            raise EngineError("%s failed (%d): %s" % (what, rc, self.L.c2b_last_error(self.h).decode()))

    # ------------------------------------------------------------------ configuration
    def configure(self, refs, ref_names, matrix, gap_open, gap_extend, seed_count=5, seed_min=2, flags=0,
                  alphabet="ACGTN", edit_cap=24):
        """refs[name] needs: sequence, gap_incentive, include_idxs, min_aln_score, fw_seeds, rc_seeds
        (the keys get_new_variant_object reads, CRISPRessoCORE.py:627-798)."""
        matrix = np.asarray(matrix)
        nq = len(alphabet)
        if nq > _lib.MAX_Q:
            raise EngineError("alphabet larger than %d symbols" % _lib.MAX_Q)
        p = _lib.Params()
        p.gap_open, p.gap_extend, p.seed_count, p.seed_min = int(gap_open), int(gap_extend), int(seed_count), int(seed_min)
        p.flags, p.nq, p.edit_cap = int(flags), nq, int(edit_cap)
        p.alphabet = alphabet.encode().ljust(_lib.MAX_Q, b"\0")
        for q, ch in enumerate(alphabet):
            p.complement[q] = alphabet.index(_DNA_COMP.get(ch, ch)) if _DNA_COMP.get(ch, ch) in alphabet else q
        arr = (_lib.Ref * len(ref_names))()
        keep = []
        for k, name in enumerate(ref_names):
            ref = refs[name]
            seq = ref["sequence"]
            sb = seq.encode()
            gi = np.ascontiguousarray(ref["gap_incentive"], dtype=np.int64)
            if len(gi) != len(sb) + 1:
                raise EngineError("gap_incentive length mismatch for %s (Align.pyx:124-126)" % name)
            inc = np.ascontiguousarray(ref.get("include_idxs", []), dtype=np.int64)
            codes = np.frombuffer(sb, dtype=np.uint8).astype(np.int64)
            if codes.max() >= matrix.shape[0] or max(ord(c) for c in alphabet) >= matrix.shape[1]:
                raise EngineError("sequence symbol outside the substitution matrix")
            rows = np.ascontiguousarray(matrix[codes][:, [ord(c) for c in alphabet]].T, dtype=np.int64)   # [nq][len]
            ns = min(int(seed_count), len(ref.get("fw_seeds", [])), len(ref.get("rc_seeds", [])))
            fw = (C.c_char_p * max(ns, 1))(*[s.encode() for s in ref.get("fw_seeds", [])[:ns]])
            rc = (C.c_char_p * max(ns, 1))(*[s.encode() for s in ref.get("rc_seeds", [])[:ns]])
            arr[k].seq, arr[k].len = sb, len(sb)
            arr[k].gap_incentive, arr[k].include_idx, arr[k].n_include = gi.ctypes.data, inc.ctypes.data, len(inc)
            arr[k].min_aln_score = float(ref.get("min_aln_score", 0))
            arr[k].score_rows = rows.ctypes.data
            arr[k].fw_seeds, arr[k].rc_seeds, arr[k].n_seeds = fw, rc, ns
            # --coding_seq inputs of the quantification loop (CRISPRessoCORE.py:4083-4087); absent keys = no coding sequence
            arr[k].tot_exon_len_mod = int(sum(ref.get("exon_len_mods", []) or []))
            cmask = None
            if ref.get("contains_coding_seq", False):
                cmask = np.zeros(len(sb), dtype=np.uint8)
                ex = np.asarray(sorted(set(ref.get("exon_positions", []))), dtype=np.int64)
                sp = np.asarray(sorted(set(ref.get("splicing_positions", []))), dtype=np.int64)
                cmask[ex[(ex >= 0) & (ex < len(sb))]] |= 1
                cmask[sp[(sp >= 0) & (sp < len(sb))]] |= 2
                arr[k].coding_mask = cmask.ctypes.data
            keep.append((sb, gi, inc, rows, fw, rc, cmask))
        self._check(self.L.c2b_configure(self.h, C.byref(p), len(ref_names), arr), "c2b_configure")
        self.n_refs, self.alphabet, self.edit_cap = len(ref_names), alphabet, int(edit_cap)
        self.ref_names = list(ref_names)
        self.ref_lens = [len(refs[n]["sequence"]) for n in ref_names]
        self.ref_seqs = [refs[n]["sequence"] for n in ref_names]
        self.flags = int(flags)
        comp = np.arange(256, dtype=np.uint8)              # p.complement over every byte, identity outside the alphabet
        for q, ch in enumerate(alphabet):
            comp[ord(ch)] = ord(alphabet[p.complement[q]])
        self.tables = (tuple(k[0] for k in keep), comp)    # what a compact BatchResult needs to spell its strings
        return self

    def set_edit_cap(self, cap):
        self._check(self.L.c2b_set_edit_cap(self.h, int(cap)), "c2b_set_edit_cap")
        self.edit_cap = int(cap)

    # ------------------------------------------------------------------ batches
    def string_width(self, max_read_len):
        w = self.L.c2b_string_width(self.h, int(max_read_len))
        if w < 0:
            raise EngineError("engine not configured")
        return w

    def align_packed(self, buf, off, count=None, qweight=None, ref_id=None, strings=True, edits=True, compact=False, on_launch=None):
        """One batch through the host-buffer entry.  compact=True: op streams + meta words come back instead of the aligned
        strings (c2b_align_batch_compact); BatchResult rebuilds strings for the reads somebody looks at."""
        n = len(off) - 1
        maxj = int(np.max(np.diff(off))) if n else 1
        W = self.string_width(max(maxj, 1))
        nr = 1 if ref_id is not None else self.n_refs      # Pooled (per-read ref_id): compact outputs, [read][0]
        recs = np.zeros(n, dtype=_lib.REC_DTYPE)
        alns = np.zeros((n, nr), dtype=_lib.ALN_DTYPE)
        earr = np.zeros((n, nr, self.edit_cap), dtype=_lib.EDIT_DTYPE) if (edits and self.edit_cap) else None

        def ptr(a):
            return None if a is None else a.ctypes.data

        buf = np.ascontiguousarray(buf, dtype=np.uint8)
        off = np.ascontiguousarray(off, dtype=np.int64)
        cnt = None if count is None else np.ascontiguousarray(count, dtype=np.int32)
        qw = None if qweight is None else np.ascontiguousarray(qweight, dtype=np.int32)
        rid = None if ref_id is None else np.ascontiguousarray(ref_id, dtype=np.int32)
        if compact:
            ops = np.zeros((n, nr, W // 32), dtype=np.uint64)
            meta = np.zeros((n, nr), dtype=np.uint32)
            if on_launch is not None:                       # the call below releases the GIL: a waiting thread may take it now
                on_launch()
            self._check(self.L.c2b_align_batch_compact(self.h, ptr(buf) if len(buf) else None, ptr(off), n, ptr(cnt), ptr(qw),
                                                       ptr(rid), ptr(recs), ptr(alns), ptr(ops), ptr(meta), ptr(earr)),
                        "c2b_align_batch_compact")
            return BatchResult(recs, alns, None, earr, W, ops=ops, meta=meta, lib=self.L, buf=buf, off=off, ref_id=rid,
                               tables=self.tables)
        sarr = np.zeros((n, nr, 2, W), dtype=np.uint8) if strings else None
        self._check(self.L.c2b_align_batch(self.h, ptr(buf) if len(buf) else None, ptr(off), n, ptr(cnt), ptr(qw),
                                           ptr(rid), ptr(recs), ptr(alns), ptr(sarr), ptr(earr)), "c2b_align_batch")
        return BatchResult(recs, alns, sarr, earr, W)

    def align(self, reads, **kw):
        buf, off = pack_reads(reads)
        return self.align_packed(buf, off, **kw)

    def classify_pair(self, read_al, ref_al, include_idx, alphabet=None, legacy=False):
        """find_indels_substitutions (legacy=True: find_indels_substitutions_legacy) on one aligned pair (GPU row-classification
        kernel).  Reconfigures."""
        n = len(ref_al)
        if alphabet is None:
            extra = sorted(set(read_al) - set("ACGTN-"))
            alphabet = "ACGTN" + "".join(extra)
        inc = np.ascontiguousarray(include_idx, dtype=np.int64)
        aln = np.zeros(1, dtype=_lib.ALN_DTYPE)
        edits = np.zeros(n + 1, dtype=_lib.EDIT_DTYPE)
        rc = self.L.c2b_classify_aligned_flags(self.h, read_al.encode(), ref_al.encode(), n, alphabet.encode(), len(alphabet),
                                               inc.ctypes.data, len(inc), _lib.F_LEGACY_INS if legacy else 0, aln.ctypes.data,
                                               edits.ctypes.data)
        self.n_refs = 0
        if rc == -2:
            raise NotImplementedError("aligned pair outside the aligner's invariants: %s"
                                      % self.L.c2b_last_error(self.h).decode())
        self._check(rc, "c2b_classify_aligned")
        if aln[0]["status"]:
            raise EngineError("c2b_classify_aligned: status %d" % aln[0]["status"])
        return aln[0], edits

    # ------------------------------------------------------------------ count block
    def counts_layout(self):
        a, b, c, d = C.c_int32(), C.c_int32(), C.c_int32(), C.c_int32()
        self._check(self.L.c2b_counts_layout(self.h, C.byref(a), C.byref(b), C.byref(c), C.byref(d)), "c2b_counts_layout")
        return a.value, b.value, c.value, d.value

    def counts_reset(self):
        self._check(self.L.c2b_counts_reset(self.h), "c2b_counts_reset")

    def hist_layout(self):
        a, b, c = C.c_int32(), C.c_int32(), C.c_int32()
        self._check(self.L.c2b_counts_hist_layout(self.h, C.byref(a), C.byref(b), C.byref(c)), "c2b_counts_hist_layout")
        return a.value, b.value, c.value

    def counts_raw(self):
        nr, nv, st, ns = self.counts_layout()
        nh, hs, _ = self.hist_layout()
        out = np.zeros(nr * (nv * st + nh * hs + ns), dtype=np.int64)
        self._check(self.L.c2b_counts_read(self.h, out.ctypes.data, out.size), "c2b_counts_read")
        return out

    def counts_device(self):
        p, n = C.c_void_p(), C.c_size_t()
        self._check(self.L.c2b_counts_device(self.h, C.byref(p), C.byref(n)), "c2b_counts_device")
        return p.value, n.value

    def counts(self, raw=None):
        """-> CountBlock built from the device block (or from an already reduced `raw` array)."""
        from .counts import CountBlock
        nr, nv, st, ns = self.counts_layout()
        raw = self.counts_raw() if raw is None else np.asarray(raw, dtype=np.int64)
        nh, hs, hz = self.hist_layout()
        return CountBlock(raw, self.ref_names, self.ref_seqs, self.alphabet, nv, st, ns, nh, hs, hz, self.flags)

    def sync(self):
        self._check(self.L.c2b_sync(self.h), "c2b_sync")

    def last_kernel_ms(self):
        return float(self.L.c2b_last_kernel_ms(self.h))

    def path_counts(self):
        """(pair_items, single_items) of the last launch: how many work items took the packed 16-bit path."""
        a, b = C.c_int64(), C.c_int64()
        self._check(self.L.c2b_path_counts(self.h, C.byref(a), C.byref(b)), "c2b_path_counts")
        return a.value, b.value

    def band_reruns(self):
        """pairs re-run with the full traceback slab since the last counts_reset (call path_counts() first)"""
        return int(self.L.c2b_band_reruns(self.h))

    def ring_counts(self):
        """(pairs aligned by the ring-banded DP, pairs of ring-eligible groups that took the full matrix) since the last
        counts_reset (call path_counts() first)"""
        a, b = C.c_int64(0), C.c_int64(0)
        self.L.c2b_ring_counts(self.h, C.byref(a), C.byref(b))
        return a.value, b.value

    def diag_counts(self):
        """(reads proved on the main diagonal, reads the diagonal tier did not prove, reads that went on to the wide ring --
        routed there by the diagonal tier or sent by the narrow tier) since the last counts_reset"""
        a, b, c = C.c_int64(0), C.c_int64(0), C.c_int64(0)
        self._check(self.L.c2b_diag_counts(self.h, C.byref(a), C.byref(b), C.byref(c)), "c2b_diag_counts")
        return a.value, b.value, c.value

    def route_counts(self):
        """(reads the diagonal tier sent straight to the wide ring, unproved reads it kept for the narrow tier) since the
        last counts_reset"""
        a, b = C.c_int64(0), C.c_int64(0)
        self._check(self.L.c2b_route_counts(self.h, C.byref(a), C.byref(b)), "c2b_route_counts")
        return a.value, b.value

    def diag_popcount_reads(self):
        """reads the diagonal tier scored by popcounts (a two-valued matrix over the amplicon, a read of A/C/G/T only)
        since the last counts_reset"""
        a = C.c_int64(0)
        self._check(self.L.c2b_diag_popcount_reads(self.h, C.byref(a)), "c2b_diag_popcount_reads")
        return a.value

    def launch_count(self):
        return int(self.L.c2b_launch_count(self.h))

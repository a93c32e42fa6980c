"""ctypes binding of libc2b200.so (the C ABI of include/c2b200.h).

The library is the product: if it is missing this module raises -- there is no CPU fallback.
Build it with `python -c "import __graft_entry__ as g; g.build()"` (nvcc, sm_90a).
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, "libc2b200.so")

MAX_Q = 8
MAX_SEEDS = 8
MAX_READ_LEN = 512
MAX_REF_LEN = 1024
MAX_REFS = 32                                           # C2B_MAX_REFS: amplicons tried per read without a per-read ref_id

F_IGNORE_SUBSTITUTIONS = 1
F_IGNORE_INSERTIONS = 2
F_IGNORE_DELETIONS = 4
F_EXPAND_AMBIGUOUS = 8
F_ASSIGN_FIRST = 16
F_DISCARD_INDEL_READS = 32
F_NO_STRAND_SEARCH = 64
F_NO_PAIRING = 128
F_HDR_REF1 = 256
F_NO_RING = 512
F_LEGACY_INS = 1024
ANN_SAM_OPTIONAL = 1 << 16                              # C2B_ANN_SAM_OPTIONAL: c2b_annotate_build's process_bam form

ST_BAD_CHAR = 1
ST_UNDEFINED = 2
ST_EDIT_OVERFLOW = 4
E_ARG, E_LIMIT, E_STATE = -2, -3, -4                    # C2B_E_* of include/c2b200.h
ST_TOO_LONG = 8
VCF_E_KEY, VCF_E_NOT_IN_LIST, VCF_E_STRING_INDEX, VCF_E_EMPTY_MAX = 1, 2, 3, 4     # C2B_VCF_E_*: c2b_vcf_edit_counts' err[1]

# count-block layout (enum order of c2b200.h)
V_ALL_INS, V_ALL_INS_LEFT, V_ALL_DEL, V_ALL_SUB, V_INS, V_DEL, V_SUB, V_SUBBASE0 = range(8)
V_BASEDEV0 = V_SUBBASE0 + MAX_Q
V_INS_LEN = V_BASEDEV0 + MAX_Q + 1
V_DEL_LEN = V_INS_LEN + 1
V_R1_ALL_INS, V_R1_ALL_INS_LEFT, V_R1_ALL_DEL, V_R1_ALL_SUB = V_DEL_LEN + 1, V_DEL_LEN + 2, V_DEL_LEN + 3, V_DEL_LEN + 4
V_R1_BASEDEV0 = V_DEL_LEN + 5
V_INS_NONCODING = V_R1_BASEDEV0 + MAX_Q + 1
V_DEL_NONCODING, V_SUB_NONCODING = V_INS_NONCODING + 1, V_INS_NONCODING + 2
NVEC = V_INS_NONCODING + 3
H_INS_N, H_DEL_N, H_SUB_N, H_EFF_LEN, H_INFRAME, H_FRAMESHIFT, NHIST = range(7)
SCALARS = ["TOTAL", "MODIFIED", "UNMODIFIED", "DISCARDED", "INS", "DEL", "SUB", "ONLY_INS", "ONLY_DEL", "ONLY_SUB",
           "INS_DEL", "INS_SUB", "DEL_SUB", "INS_DEL_SUB", "AMBIGUOUS_W", "N_GLOBAL_SUBS", "N_SUBS_OUTSIDE_WINDOW",
           "N_MODS_IN_WINDOW", "N_MODS_OUTSIDE_WINDOW", "N_READS_IRREGULAR_ENDS", "N_ALIGNED_UNIQUE",
           "N_ALIGNED_COUNT", "REF1_W", "CLASS_MODIFIED", "CLASS_UNMODIFIED", "MOD_FRAMESHIFT", "MOD_NON_FRAMESHIFT",
           "NON_MOD_NON_FRAMESHIFT", "SPLICING_MODIFIED"]
NSCAL = len(SCALARS)
S = {n: k for k, n in enumerate(SCALARS)}


class Params(C.Structure):
    _fields_ = [("gap_open", C.c_int32), ("gap_extend", C.c_int32), ("seed_count", C.c_int32),
                ("seed_min", C.c_int32), ("flags", C.c_uint32), ("nq", C.c_int32),
                ("alphabet", C.c_char * MAX_Q), ("complement", C.c_uint8 * MAX_Q), ("edit_cap", C.c_int32)]


class Ref(C.Structure):
    _fields_ = [("seq", C.c_char_p), ("len", C.c_int32), ("gap_incentive", C.c_void_p),
                ("include_idx", C.c_void_p), ("n_include", C.c_int32), ("min_aln_score", C.c_double),
                ("score_rows", C.c_void_p), ("fw_seeds", C.POINTER(C.c_char_p)), ("rc_seeds", C.POINTER(C.c_char_p)),
                ("n_seeds", C.c_int32), ("tot_exon_len_mod", C.c_int32), ("coding_mask", C.c_void_p)]


ALN_DTYPE = np.dtype([("n_match", "<u2"), ("aln_len", "<u2"), ("score_milli", "<i4"), ("strand", "u1"),
                      ("status", "u1"), ("n_edits", "<u2"), ("insertion_n", "<u2"), ("deletion_n", "<u2"),
                      ("substitution_n", "<u2"), ("n_ins_all", "<u2"), ("n_ins_win", "<u2"), ("n_del_all", "<u2"),
                      ("n_del_win", "<u2"), ("n_del_pos_all", "<u2"), ("n_sub_all", "<u2"),
                      ("irregular_ends", "u1"), ("modified", "u1")])
REC_DTYPE = np.dtype([("winner_mask", "<u4"), ("best_score_milli", "<i4"), ("best_ref", "<i2"), ("n_winners", "u1"),
                      ("ambiguous", "u1"), ("status", "<u4")])
EDIT_DTYPE = np.dtype([("a", "<u2"), ("b", "<u2"), ("type", "u1"), ("in_window", "u1"), ("base", "u1"), ("pad", "u1")])
assert ALN_DTYPE.itemsize == 32 and REC_DTYPE.itemsize == 16 and EDIT_DTYPE.itemsize == 8

EXPORTS = ["c2b_create", "c2b_destroy", "c2b_last_error", "c2b_configure", "c2b_set_edit_cap", "c2b_string_width", "c2b_align_batch",
           "c2b_align_batch_compact", "c2b_ops_words", "c2b_expand_alignment", "c2b_expand_batch", "c2b_expand_batch_tables",
           "c2b_ops_device",
           "c2b_align_batch_device", "c2b_set_pair_order", "c2b_sync", "c2b_stream", "c2b_last_kernel_ms", "c2b_launch_count", "c2b_path_counts", "c2b_band_reruns", "c2b_ring_counts", "c2b_diag_counts", "c2b_route_counts", "c2b_diag_popcount_reads",
           "c2b_counts_layout", "c2b_counts_hist_layout", "c2b_counts_reset", "c2b_counts_read", "c2b_counts_device", "c2b_global_align",
           "c2b_classify_aligned", "c2b_classify_aligned_flags", "c2b_host_alloc", "c2b_host_free",
           "c2b_fastq_dedup", "c2b_fastq_dedup_buffer", "c2b_fastq_gpu_available", "c2b_fastq_dedup_gpu", "c2b_fastq_dedup_gpu_buffer", "c2b_sam_dedup_gpu_buffer", "c2b_sam_dedup_buffer", "c2b_fastq_n_reads", "c2b_fastq_n_unique", "c2b_fastq_max_len",
           "c2b_fastq_seqs", "c2b_fastq_offsets", "c2b_fastq_counts", "c2b_fastq_first_index", "c2b_fastq_free",
           "c2b_fastq_last_error", "c2b_fastq_filter", "c2b_fastq_filter_pair", "c2b_rc_merge_weights", "c2b_screen_reads", "c2b_serial_stats",
           "c2b_consensus_from_pairs", "c2b_alleles_build", "c2b_alleles_free", "c2b_alleles_n", "c2b_alleles_order", "c2b_alleles_arena", "c2b_alleles_offsets",
           "c2b_alleles_lengths", "c2b_alleles_write_tsv", "c2b_alleles_around_cut", "c2b_alleles_cut_width", "c2b_alleles_cut_fetch",
           "c2b_annotate_build", "c2b_annotate_free", "c2b_annotate_n", "c2b_annotate_arena", "c2b_annotate_offsets",
           "c2b_annotate_cigar_arena", "c2b_annotate_cigar_offsets", "c2b_annotate_flags", "c2b_annotate_mapq", "c2b_annotate_first",
           "c2b_annotate_last_record", "c2b_annotate_record_arena", "c2b_annotate_record_offsets", "c2b_annotate_write_fastq",
           "c2b_annotate_write_sam", "c2b_annotate_write_sam_passthrough", "c2b_vcf_edit_counts", "c2b_vcf_free", "c2b_vcf_n",
           "c2b_vcf_keys", "c2b_vcf_key_offsets", "c2b_vcf_reads", "c2b_vcf_n_records", "c2b_vcf_timings"]

_cache = {}


class LibraryMissing(ImportError):
    pass


def load(path=None):
    """Loads the engine library.  `path` is a test hook (the CPU warp-emulator build under tests/emu/);
    the product default is the nvcc-built libc2b200.so next to this file."""
    path = path or os.environ.get("C2B200_LIB") or DEFAULT_LIB     # C2B200_LIB: another nvcc build variant (A/B runs)
    if path in _cache:
        return _cache[path]
    if not os.path.exists(path):
        raise LibraryMissing("%s not found: build the CUDA extension first (python -c 'import __graft_entry__ as g; "
                             "g.build()'); crispresso2_b200 has no CPU fallback" % path)
    L = C.CDLL(path)
    vp, i32, i64 = C.c_void_p, C.c_int32, C.c_int64
    L.c2b_create.restype = C.c_int
    L.c2b_create.argtypes = [C.c_int, C.POINTER(vp)]
    L.c2b_destroy.restype = None
    L.c2b_destroy.argtypes = [vp]
    L.c2b_last_error.restype = C.c_char_p
    L.c2b_last_error.argtypes = [vp]
    L.c2b_configure.restype = C.c_int
    L.c2b_configure.argtypes = [vp, C.POINTER(Params), i32, C.POINTER(Ref)]
    L.c2b_set_edit_cap.restype = C.c_int
    L.c2b_set_edit_cap.argtypes = [vp, i32]
    L.c2b_string_width.restype = C.c_int
    L.c2b_string_width.argtypes = [vp, i32]
    L.c2b_align_batch.restype = C.c_int
    L.c2b_align_batch.argtypes = [vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp]
    L.c2b_align_batch_compact.restype = C.c_int
    L.c2b_align_batch_compact.argtypes = [vp, vp, vp, i64, vp, vp, vp, vp, vp, vp, vp, vp]
    L.c2b_ops_words.restype = C.c_int
    L.c2b_ops_words.argtypes = [vp, i32]
    L.c2b_expand_alignment.restype = C.c_int
    L.c2b_expand_alignment.argtypes = [vp, vp, C.c_uint32, C.c_char_p, i32, C.c_char_p, i32, vp, vp]
    L.c2b_expand_batch.restype = C.c_int
    L.c2b_expand_batch.argtypes = [vp, vp, vp, i64, vp, vp, vp, i32, vp, i32]
    L.c2b_expand_batch_tables.restype = C.c_int
    L.c2b_expand_batch_tables.argtypes = [vp, vp, i64, vp, vp, vp, i32, i32, i32, C.POINTER(C.c_char_p), vp, vp, vp, i32]
    L.c2b_ops_device.restype = C.c_int
    L.c2b_ops_device.argtypes = [vp, C.POINTER(vp), C.POINTER(vp)]
    L.c2b_align_batch_device.restype = C.c_int
    L.c2b_align_batch_device.argtypes = [vp, vp, vp, i64, i32, vp, vp, vp, vp, vp, vp, vp]
    L.c2b_set_pair_order.restype = C.c_int
    L.c2b_set_pair_order.argtypes = [vp, vp]
    L.c2b_sync.restype = C.c_int
    L.c2b_sync.argtypes = [vp]
    L.c2b_stream.restype = vp
    L.c2b_stream.argtypes = [vp]
    L.c2b_last_kernel_ms.restype = C.c_double
    L.c2b_last_kernel_ms.argtypes = [vp]
    L.c2b_launch_count.restype = i64
    L.c2b_launch_count.argtypes = [vp]
    L.c2b_path_counts.restype = C.c_int
    L.c2b_path_counts.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    L.c2b_band_reruns.restype = i64
    L.c2b_band_reruns.argtypes = [vp]
    L.c2b_ring_counts.restype = C.c_int
    L.c2b_ring_counts.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    L.c2b_diag_counts.restype = C.c_int
    L.c2b_diag_counts.argtypes = [vp, C.POINTER(i64), C.POINTER(i64), C.POINTER(i64)]
    L.c2b_route_counts.restype = C.c_int
    L.c2b_route_counts.argtypes = [vp, C.POINTER(i64), C.POINTER(i64)]
    L.c2b_diag_popcount_reads.restype = C.c_int
    L.c2b_diag_popcount_reads.argtypes = [vp, C.POINTER(i64)]
    L.c2b_counts_layout.restype = C.c_int
    L.c2b_counts_layout.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.c2b_counts_hist_layout.restype = C.c_int
    L.c2b_counts_hist_layout.argtypes = [vp, C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.c2b_counts_reset.restype = C.c_int
    L.c2b_counts_reset.argtypes = [vp]
    L.c2b_counts_read.restype = C.c_int
    L.c2b_counts_read.argtypes = [vp, vp, C.c_size_t]
    L.c2b_counts_device.restype = C.c_int
    L.c2b_counts_device.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_size_t)]
    L.c2b_global_align.restype = C.c_int
    L.c2b_global_align.argtypes = [vp, C.c_char_p, i32, C.c_char_p, i32, C.c_char_p, i32, vp, vp, i32, i32,
                                   C.c_char_p, C.c_char_p, C.POINTER(i32), C.POINTER(i32)]
    L.c2b_classify_aligned.restype = C.c_int
    L.c2b_classify_aligned.argtypes = [vp, C.c_char_p, C.c_char_p, i32, C.c_char_p, i32, vp, i32, vp, vp]
    L.c2b_classify_aligned_flags.restype = C.c_int
    L.c2b_classify_aligned_flags.argtypes = [vp, C.c_char_p, C.c_char_p, i32, C.c_char_p, i32, vp, i32, C.c_uint32, vp, vp]
    L.c2b_host_alloc.restype = vp
    L.c2b_host_alloc.argtypes = [C.c_size_t]
    L.c2b_host_free.restype = None
    L.c2b_host_free.argtypes = [vp]
    L.c2b_fastq_dedup.restype = C.c_int
    L.c2b_fastq_dedup.argtypes = [C.c_char_p, i32, C.POINTER(vp)]
    L.c2b_fastq_dedup_buffer.restype = C.c_int
    L.c2b_fastq_dedup_buffer.argtypes = [vp, C.c_size_t, i32, C.POINTER(vp)]
    for name, rt in (("c2b_fastq_n_reads", i64), ("c2b_fastq_n_unique", i64), ("c2b_fastq_max_len", i32),
                     ("c2b_fastq_seqs", vp), ("c2b_fastq_offsets", vp), ("c2b_fastq_counts", vp),
                     ("c2b_fastq_first_index", vp)):
        getattr(L, name).restype = rt
        getattr(L, name).argtypes = [vp]
    L.c2b_fastq_free.restype = None
    L.c2b_fastq_free.argtypes = [vp]
    L.c2b_consensus_from_pairs.restype = C.c_int
    L.c2b_consensus_from_pairs.argtypes = [C.c_char_p, i32, C.c_char_p, i32, C.c_double, C.c_char_p, i32,
                                           C.c_char_p, i32, C.c_char_p, i32, C.c_double, C.c_char_p, i32,
                                           C.c_char_p, C.c_char_p, C.c_char_p, i32,
                                           C.POINTER(i32), C.POINTER(i32), C.POINTER(i32), C.POINTER(i32)]
    L.c2b_fastq_gpu_available.restype = C.c_int
    L.c2b_fastq_gpu_available.argtypes = []
    L.c2b_fastq_dedup_gpu.restype = C.c_int
    L.c2b_fastq_dedup_gpu.argtypes = [C.c_char_p, i32, C.POINTER(vp)]
    L.c2b_fastq_dedup_gpu_buffer.restype = C.c_int
    L.c2b_fastq_dedup_gpu_buffer.argtypes = [vp, C.c_size_t, i32, C.POINTER(vp)]
    L.c2b_sam_dedup_gpu_buffer.restype = C.c_int
    L.c2b_sam_dedup_gpu_buffer.argtypes = [vp, C.c_size_t, i32, C.POINTER(vp)]
    L.c2b_sam_dedup_buffer.restype = C.c_int
    L.c2b_sam_dedup_buffer.argtypes = [vp, C.c_size_t, i32, C.POINTER(vp)]
    L.c2b_fastq_filter.restype = C.c_int
    L.c2b_fastq_filter.argtypes = [C.c_char_p, C.c_char_p, i32, i32, i32, i32, C.POINTER(i64), C.POINTER(i64)]
    L.c2b_fastq_filter_pair.restype = C.c_int
    L.c2b_fastq_filter_pair.argtypes = [C.c_char_p, C.c_char_p, C.c_char_p, C.c_char_p, i32, i32, i32, i32, C.POINTER(i64), C.POINTER(i64)]
    L.c2b_rc_merge_weights.restype = C.c_int
    L.c2b_rc_merge_weights.argtypes = [vp, vp, i64, vp, vp, vp, i32]
    L.c2b_screen_reads.restype = i64
    L.c2b_screen_reads.argtypes = [vp, vp, i64, i32, vp, i32]
    L.c2b_fastq_last_error.restype = C.c_char_p
    L.c2b_fastq_last_error.argtypes = []
    L.c2b_serial_stats.restype = C.c_int
    L.c2b_serial_stats.argtypes = [vp, vp, vp, i64, i32, vp, vp, i32]
    L.c2b_alleles_build.restype = C.c_int
    L.c2b_alleles_build.argtypes = [vp, vp, vp, vp, i32, i64, vp, vp, vp, vp, i32, C.POINTER(C.c_char_p), vp, vp, i32, C.POINTER(vp)]
    L.c2b_alleles_free.restype = None
    L.c2b_alleles_free.argtypes = [vp]
    L.c2b_alleles_n.restype = i64
    L.c2b_alleles_n.argtypes = [vp]
    for name in ("c2b_alleles_order", "c2b_alleles_arena", "c2b_alleles_offsets", "c2b_alleles_lengths"):
        getattr(L, name).restype = vp
        getattr(L, name).argtypes = [vp]
    L.c2b_alleles_write_tsv.restype = C.c_int
    L.c2b_alleles_write_tsv.argtypes = [vp, C.c_char_p, i64, vp, vp, C.POINTER(C.c_char_p), vp, C.POINTER(C.c_char_p), vp, vp, vp, vp,
                                        C.POINTER(C.c_char_p), i32]
    L.c2b_alleles_around_cut.restype = i64
    L.c2b_alleles_around_cut.argtypes = [vp, i64, vp, i32, i32, i32, vp, vp, vp, vp, vp]
    L.c2b_alleles_cut_width.restype = i32
    L.c2b_alleles_cut_width.argtypes = [vp]
    L.c2b_alleles_cut_fetch.restype = C.c_int
    L.c2b_alleles_cut_fetch.argtypes = [vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    cpp = C.POINTER(C.c_char_p)
    L.c2b_annotate_build.restype = C.c_int
    L.c2b_annotate_build.argtypes = [vp, vp, vp, i64, vp, i32, i32, i32, vp, vp, vp, vp, vp, vp, vp, vp, i32, cpp, vp, i32, cpp, cpp, vp,
                                     vp, C.c_uint32, i64, C.POINTER(vp)]
    L.c2b_annotate_free.restype = None
    L.c2b_annotate_free.argtypes = [vp]
    L.c2b_annotate_n.restype = i64
    L.c2b_annotate_n.argtypes = [vp]
    for name in ("c2b_annotate_arena", "c2b_annotate_offsets", "c2b_annotate_cigar_arena", "c2b_annotate_cigar_offsets",
                 "c2b_annotate_flags", "c2b_annotate_mapq", "c2b_annotate_first", "c2b_annotate_last_record",
                 "c2b_annotate_record_arena", "c2b_annotate_record_offsets"):
        getattr(L, name).restype = vp
        getattr(L, name).argtypes = [vp]
    L.c2b_annotate_write_fastq.restype = C.c_int
    L.c2b_annotate_write_fastq.argtypes = [vp, vp, vp, i64, C.c_char_p, C.c_char_p, i32]
    L.c2b_annotate_write_sam.restype = C.c_int
    L.c2b_annotate_write_sam.argtypes = [vp, vp, vp, i64, C.c_char_p, C.c_char_p, C.c_char_p, i32, cpp, cpp, vp, i32]
    L.c2b_annotate_write_sam_passthrough.restype = C.c_int
    L.c2b_annotate_write_sam_passthrough.argtypes = [vp, vp, vp, i64, vp, C.c_size_t, C.c_char_p, i32]
    L.c2b_vcf_edit_counts.restype = C.c_int
    L.c2b_vcf_edit_counts.argtypes = [vp, i64] + [vp] * 17 + [i64, vp, C.POINTER(vp)]
    L.c2b_vcf_free.restype = None
    L.c2b_vcf_free.argtypes = [vp]
    for name, rt in (("c2b_vcf_n", i64), ("c2b_vcf_keys", vp), ("c2b_vcf_key_offsets", vp), ("c2b_vcf_reads", vp),
                     ("c2b_vcf_n_records", i64)):
        getattr(L, name).restype = rt
        getattr(L, name).argtypes = [vp]
    L.c2b_vcf_timings.restype = C.c_int
    L.c2b_vcf_timings.argtypes = [vp, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    _cache[path] = L
    return L

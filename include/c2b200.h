/*
 * c2b200.h -- C ABI of the H100 align-and-classify engine (libc2b200.so).
 *
 * This is the drop-in boundary for CRISPResso2's per-read hot path.  The reference has no FFI of its own
 * (its two native modules are Cython, called from Python); each entry point below names the reference
 * interface it replaces (paths relative to the reference repository root).  Plain pointers and sizes only;
 * no torch / Python types.  INTEGRATION.md shows the ctypes binding a reference maintainer would add.
 *
 * Threading: an engine is owned by one host thread at a time.  All calls are synchronous unless suffixed
 * _async.  Never create an engine in a process that will later fork() CUDA work (reference workers are
 * forked by CRISPRessoCORE.py:1878-1896; the GPU path bypasses them).
 */
#ifndef C2B200_H
#define C2B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define C2B_MAX_Q        8      /* read alphabet size (codes 0..nq-1); DNA uses "ACGTN" */
#define C2B_MAX_SEEDS    8      /* seeds tested per strand (args.aln_seed_count, default 5) */
#define C2B_MAX_SEED_LEN 20
#define C2B_MAX_REF_LEN  1024   /* amplicon length limit of this build */
#define C2B_MAX_READ_LEN 512
#define C2B_MAX_ALN_LEN  1024   /* I + J */
#define C2B_MAX_REFS     32     /* references tried per read (ref_id == NULL) */
#define C2B_MAX_POOLED_REFS 1024 /* references per configuration when every read names its own (ref_id, Pooled) */

/* status codes */
#define C2B_OK            0
#define C2B_E_CUDA       -1
#define C2B_E_ARG        -2
#define C2B_E_LIMIT      -3     /* a length / range limit of this build is exceeded */
#define C2B_E_STATE      -4

/* c2b_params.flags  (CRISPRessoCORE.py:746-760, 780-785, 3998-4002) */
#define C2B_F_IGNORE_SUBSTITUTIONS  1u
#define C2B_F_IGNORE_INSERTIONS     2u
#define C2B_F_IGNORE_DELETIONS      4u
#define C2B_F_EXPAND_AMBIGUOUS      8u
#define C2B_F_ASSIGN_FIRST         16u
#define C2B_F_DISCARD_INDEL_READS  32u
#define C2B_F_NO_STRAND_SEARCH     64u   /* global_align-only mode: forward strand, no seed test */
#define C2B_F_NO_PAIRING          128u   /* debugging / A-B runs: never use the packed two-reads-per-warp path */
#define C2B_F_LEGACY_INS         1024u   /* args.use_legacy_insertion_quantification: find_indels_substitutions_legacy (COREResources.pyx:190-315) */
#define C2B_F_NO_RING             512u   /* debugging / A-B runs: never use the ring-banded four-pairs-per-warp path */
#define C2B_F_HDR_REF1            256u   /* args.expected_hdr_amplicon_seq / prime-editing extension set: also build the
                                            "ref1" re-projection vectors of CRISPRessoCORE.py:4195-4272 */

typedef struct {
    int32_t  gap_open;        /* args.needleman_wunsch_gap_open   (Align.pyx:104) */
    int32_t  gap_extend;      /* args.needleman_wunsch_gap_extend */
    int32_t  seed_count;      /* args.aln_seed_count */
    int32_t  seed_min;        /* args.aln_seed_min   */
    uint32_t flags;
    int32_t  nq;              /* alphabet size */
    char     alphabet[C2B_MAX_Q];   /* code -> ASCII, e.g. "ACGTN" */
    uint8_t  complement[C2B_MAX_Q]; /* code -> code of the complementary base (CRISPRessoShared.py:399-403) */
    int32_t  edit_cap;        /* edit-list slots per (read, winning reference); see c2b_edit */
} c2b_params;

/* One amplicon: the refs[ref_name] keys the hot path reads (SURVEY.md Appendix A). */
typedef struct {
    const char    *seq;            /* refs[name]['sequence'] */
    int32_t        len;
    const int64_t *gap_incentive;  /* refs[name]['gap_incentive'], len+1 entries (CRISPRessoCORE.py:3205-3207) */
    const int64_t *include_idx;    /* refs[name]['include_idxs'] */
    int32_t        n_include;
    double         min_aln_score;  /* refs[name]['min_aln_score'] */
    const int64_t *score_rows;     /* [nq][len]: matrix[ord(seq[i]), ord(alphabet[q])] -- the aln_matrix
                                      lookups of Align.pyx:212, tabulated per reference position by the host */
    const char *const *fw_seeds;   /* refs[name]['fw_seeds'][:seed_count] */
    const char *const *rc_seeds;   /* refs[name]['rc_seeds'][:seed_count] */
    int32_t        n_seeds;
    /* --coding_seq quantification (CRISPRessoCORE.py:4083-4180); all optional */
    int32_t        tot_exon_len_mod;   /* sum(refs[name]['exon_len_mods']) */
    const uint8_t *coding_mask;    /* NULL when refs[name]['contains_coding_seq'] is false; else [len] bytes:
                                      bit 0 = position in refs[name]['exon_positions'], bit 1 = in ['splicing_positions'] */
} c2b_ref;

/* Per (read, reference) alignment result: what global_align returns (Align.pyx:422-434) plus, when the
 * reference is a best match, the scalar fields of find_indels_substitutions / get_new_variant_object
 * (COREResources.pyx:161-186, CRISPRessoCORE.py:726-760). 32 bytes. */
typedef struct {
    uint16_t n_match;          /* matchCount */
    uint16_t aln_len;          /* alignment columns */
    int32_t  score_milli;      /* round(100*n_match/aln_len, 3) * 1000, exact (half-even) */
    uint8_t  strand;           /* 0 '+', 1 '-' */
    uint8_t  status;           /* 0 ok; C2B_ST_* bits otherwise */
    uint16_t n_edits;          /* edit-list entries produced (may exceed edit_cap: then C2B_ST_EDIT_OVERFLOW) */
    uint16_t insertion_n, deletion_n, substitution_n;          /* inside the quantification window */
    uint16_t n_ins_all, n_ins_win;        /* insertion runs: all / in window  */
    uint16_t n_del_all, n_del_win;        /* deletion runs */
    uint16_t n_del_pos_all;               /* len(all_deletion_positions) */
    uint16_t n_sub_all;                   /* len(all_substitution_positions) */
    uint8_t  irregular_ends;
    uint8_t  modified;                    /* classification == 'MODIFIED' */
} c2b_aln_rec;

#define C2B_ST_BAD_CHAR       1u   /* read holds a symbol outside the alphabet */
#define C2B_ST_UNDEFINED      2u   /* traceback left the zone where the reference is defined (SURVEY 3.2) */
#define C2B_ST_EDIT_OVERFLOW  4u   /* more edits than edit_cap: the LIST is truncated (scalars and counts are complete) */
#define C2B_ST_TOO_LONG       8u

/* Per read: best-reference selection of get_new_variant_object (CRISPRessoCORE.py:690-716, 780-785). 16 bytes */
typedef struct {
    uint32_t winner_mask;      /* bit r set: reference r is in best_match_names (before assign-first trimming); under a
                                  per-read ref_id (Pooled) the one candidate sets bit ref_id mod 32 */
    int32_t  best_score_milli; /* best_match_score*1000 ; <= 0: not aligned */
    int16_t  best_ref;         /* index of new_variant['best_match_name'] (last winner), -1 if none */
    uint8_t  n_winners;
    uint8_t  ambiguous;        /* class_name == 'AMBIGUOUS' */
    uint32_t status;           /* OR of the per-alignment status bits */
} c2b_read_rec;

/* Edit list entry (8 bytes); expands on the host into the list fields of ResultsSlotsDict
 * (COREResources.pyx:18-65).  Entries of one type appear in increasing reference position. */
typedef struct {
    uint16_t a;        /* SUB: position           INS: left flank (start)        DEL: start            */
    uint16_t b;        /* SUB: unused             INS: size of the insertion     DEL: end (exclusive)  */
    uint8_t  type;     /* 1 SUB, 2 INS, 3 DEL */
    uint8_t  in_window;
    uint8_t  base;     /* SUB: read base (ASCII) */
    uint8_t  pad;
} c2b_edit;

/* Count block: per reference r one chunk of int64: [C2B_NVEC][stride] vectors, [C2B_NHIST][hstride] histograms,
 * [C2B_NSCAL] scalars; chunks follow each other.  Vectors follow CRISPRessoCORE.py:3865-3896 / the table in
 * SURVEY.md 3.4. */
enum {
    C2B_V_ALL_INS = 0, C2B_V_ALL_INS_LEFT, C2B_V_ALL_DEL, C2B_V_ALL_SUB,
    C2B_V_INS, C2B_V_DEL, C2B_V_SUB,
    C2B_V_SUBBASE0,                    /* + alphabet code : all_substitution_base_vectors */
    C2B_V_BASEDEV0 = C2B_V_SUBBASE0 + C2B_MAX_Q,   /* + code (nq = '-') : all_base_count deviation from "read == ref" */
    C2B_V_INS_LEN = C2B_V_BASEDEV0 + C2B_MAX_Q + 1,
    C2B_V_DEL_LEN,
    /* HDR mode: reads assigned to THIS reference, re-classified on their alignment to reference 0; positions are
     * reference-0 positions (ref1_all_*_count_vectors[this ref], CRISPRessoCORE.py:4255-4272) */
    C2B_V_R1_ALL_INS, C2B_V_R1_ALL_INS_LEFT, C2B_V_R1_ALL_DEL, C2B_V_R1_ALL_SUB,
    C2B_V_R1_BASEDEV0,                 /* + code (nq = '-'): deviation from "read == reference-0 base" */
    /* --coding_seq: window edits of modified reads that touch no exon (CRISPRessoCORE.py:4166-4171) */
    C2B_V_INS_NONCODING = C2B_V_R1_BASEDEV0 + C2B_MAX_Q + 1, C2B_V_DEL_NONCODING, C2B_V_SUB_NONCODING,
    C2B_NVEC
};
/* Histograms keyed by a small integer (the reference's Counters, CRISPRessoCORE.py:3898-3906).  Bucket index =
 * key for the first four rows, key + hist_zero for the two frame rows.  The most common bucket of the first four rows
 * is NOT stored (it would be one hot address for every unedited read): key 0 of INS_N / DEL_N / SUB_N and key
 * len(ref) of EFF_LEN equal counts_total minus the sum of the stored buckets (crispresso2_b200/counts.py). */
enum {
    C2B_H_INS_N = 0,       /* inserted_n_dicts[ref][insertion_n]        (:4020, unless ignore_insertions)    */
    C2B_H_DEL_N,           /* deleted_n_dicts[ref][deletion_n]          (:4031, unless ignore_deletions)     */
    C2B_H_SUB_N,           /* substituted_n_dicts[ref][substitution_n]  (:4043, unless ignore_substitutions) */
    C2B_H_EFF_LEN,         /* effective_len_dicts[ref][len - deletion_n + insertion_n]   (:4037)             */
    C2B_H_INFRAME,         /* hists_inframe[ref][effective_length]      (:4144-4177)                         */
    C2B_H_FRAMESHIFT,      /* hists_frameshift[ref][effective_length]                                        */
    C2B_NHIST
};
enum {
    C2B_S_TOTAL = 0, C2B_S_MODIFIED, C2B_S_UNMODIFIED, C2B_S_DISCARDED,
    C2B_S_INS, C2B_S_DEL, C2B_S_SUB,
    C2B_S_ONLY_INS, C2B_S_ONLY_DEL, C2B_S_ONLY_SUB, C2B_S_INS_DEL, C2B_S_INS_SUB, C2B_S_DEL_SUB, C2B_S_INS_DEL_SUB,
    C2B_S_AMBIGUOUS_W,     /* weight of reads classed AMBIGUOUS with this reference as first winner */
    /* aln_stats of process_fastq (CRISPRessoCORE.py:1988-1999), accumulated with the dedup count */
    C2B_S_N_GLOBAL_SUBS, C2B_S_N_SUBS_OUTSIDE_WINDOW, C2B_S_N_MODS_IN_WINDOW, C2B_S_N_MODS_OUTSIDE_WINDOW,
    C2B_S_N_READS_IRREGULAR_ENDS, C2B_S_N_ALIGNED_UNIQUE, C2B_S_N_ALIGNED_COUNT,
    C2B_S_REF1_W,          /* weight re-projected onto reference 0 for this reference (C2B_F_HDR_REF1) */
    /* class_counts (CRISPRessoCORE.py:3984-3986): class_counts["<ref>_MODIFIED"] = counts_modified + C2B_S_CLASS_MODIFIED
     * (signed deviation: + reads discarded by --discard_indel_reads, which keep their class; - winners of
     * --expand_ambiguous_alignments reads with several best references, whose joined label is derived from the read
     * records on the host); likewise _UNMODIFIED; "AMBIGUOUS" = sum of C2B_S_AMBIGUOUS_W */
    C2B_S_CLASS_MODIFIED, C2B_S_CLASS_UNMODIFIED,
    /* --coding_seq counters (:4134-4171) */
    C2B_S_MOD_FRAMESHIFT, C2B_S_MOD_NON_FRAMESHIFT, C2B_S_NON_MOD_NON_FRAMESHIFT, C2B_S_SPLICING_MODIFIED,
    C2B_NSCAL
};

typedef struct c2b_engine c2b_engine;

/* lifecycle -------------------------------------------------------------------------------------------- */
int  c2b_create(int device, c2b_engine **out);
void c2b_destroy(c2b_engine *e);
const char *c2b_last_error(const c2b_engine *e);   /* e may be NULL: error of the last failed c2b_create */

/* replaces: the args/refs plumbing of process_fastq (CRISPRessoCORE.py:1735, :1811-1813) */
int  c2b_configure(c2b_engine *e, const c2b_params *p, int32_t n_refs, const c2b_ref *refs);

/* Changes c2b_params.edit_cap for the following batches without touching tables or counts (used to re-run
 * the few reads whose edit list overflowed with a cap that cannot overflow). */
int  c2b_set_edit_cap(c2b_engine *e, int32_t edit_cap);

/* Output geometry for a batch whose longest read is max_read_len:
 *   string width W (multiple of 16): every aligned string is right-aligned in a W-byte slot;
 *   alns    : n_reads * R records, [read][ref]
 *   strings : n_reads * R * 2 * W bytes, [read][ref][0 = read, 1 = reference][W]
 *   edits   : n_reads * R * edit_cap entries
 * R = n_refs when every reference is tried (ref_id == NULL); R = 1 when ref_id is given (Pooled: each read is aligned
 * to its own amplicon only, so the outputs are compact [read][0]).                                   */
int  c2b_string_width(const c2b_engine *e, int32_t max_read_len);

/* replaces: the serial loop of process_fastq over unique reads (CRISPRessoCORE.py:1956-1981), i.e. one
 * get_new_variant_object (:627-798) per read = seed test, global_align per strand and reference,
 * best-reference choice, find_indels_substitutions per winner, and the per-read part of the
 * quantification loop (:3964-4115).  Host buffers in, host buffers out (copies inside).
 *   reads/offsets : packed ASCII reads, offsets[n_reads+1]
 *   count         : dedup multiplicity per read (variant_count of :1957)          (NULL = 1)
 *   qweight       : count after the reverse-complement merge of :3971-3975        (NULL = count)
 *   ref_id        : NULL = try every reference (at most C2B_MAX_REFS configured); else the single reference index of
 *                   each read (Pooled; up to C2B_MAX_POOLED_REFS configured; outputs are [read][0])
 *   strings/edits may be NULL (not produced).                                                         */
int  c2b_align_batch(c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads,
                     const int32_t *count, const int32_t *qweight, const int32_t *ref_id,
                     c2b_read_rec *recs, c2b_aln_rec *alns, uint8_t *strings, c2b_edit *edits);

/* Compact form of c2b_align_batch: instead of the two W-byte aligned strings per (read, reference) slot the alignment itself
 * comes back -- what Align.pyx:338-421's traceback decides, before :422-432 spell it out as strings:
 *   ops  : n_reads * R * NW words (NW = c2b_ops_words()); column q counted from the RIGHT end of the alignment is op
 *          (ops[slot * NW + (q >> 5)] >> 2 * (q & 31)) & 3 : 0 read base over reference base, 1 gap in the read (deletion),
 *          2 gap in the reference (insertion), 3 past the alignment's left end
 *   meta : n_reads * R words: bits 0-15 alignment columns, bit 16 strand ('-' = the read was aligned as its reverse
 *          complement), bits 24-31 non-zero when the slot holds an alignment
 * c2b_expand_alignment / c2b_expand_batch rebuild the strings on the host (bit-identical to c2b_align_batch's); 5 to 8 times
 * fewer bytes cross PCIe (DESIGN.md section 6b).                                                           */
int  c2b_align_batch_compact(c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads,
                             const int32_t *count, const int32_t *qweight, const int32_t *ref_id,
                             c2b_read_rec *recs, c2b_aln_rec *alns, uint64_t *ops, uint32_t *meta, c2b_edit *edits);
int  c2b_ops_words(const c2b_engine *e, int32_t max_read_len);
/* out_read / out_ref receive (meta & 0xffff) characters each, left to right as global_align returns them (Align.pyx:422-434) */
int  c2b_expand_alignment(const c2b_engine *e, const uint64_t *ops, uint32_t meta, const char *read, int32_t read_len,
                          const char *ref, int32_t ref_len, char *out_read, char *out_ref);
/* strings: n_reads * R * 2 * W bytes, right-aligned slots as c2b_align_batch writes them; host threads (n_threads <= 0: all).
 * Reads the engine's CURRENT references, max_I and complement table: valid only while the engine keeps the configuration the
 * batch ran under. */
int  c2b_expand_batch(const c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_reads, const int32_t *ref_id,
                      const uint64_t *ops, const uint32_t *meta, int32_t max_read_len, uint8_t *strings, int32_t n_threads);
/* Same, with no engine: the caller passes what the batch ran with -- R slots per read (1 with ref_id), the string width W
 * (a multiple of 32; NW = W / 32 op words per slot), the n_refs configured reference sequences and their lengths, and the
 * complement of every byte (identity outside the alphabet).  A batch's results expand the same way whatever its engine does
 * afterwards, closed included.  C2B_E_ARG on an op stream that does not fit its read and reference, or a ref_id outside
 * 0..n_refs-1. */
int  c2b_expand_batch_tables(const uint8_t *reads, const int64_t *offsets, int64_t n_reads, const int32_t *ref_id,
                             const uint64_t *ops, const uint32_t *meta, int32_t R, int32_t W, int32_t n_refs,
                             const char *const *ref_seqs, const int32_t *ref_lens, const uint8_t *comp256,
                             uint8_t *strings, int32_t n_threads);

/* Same, with every pointer a DEVICE pointer on the engine's device and no copies; the launch is queued on
 * the engine's stream.  max_read_len must bound the reads.  Use c2b_sync() before reading results.     */
int  c2b_align_batch_device(c2b_engine *e, const uint8_t *d_reads, const int64_t *d_offsets, int64_t n_reads,
                            int32_t max_read_len, const int32_t *d_count, const int32_t *d_qweight,
                            const int32_t *d_ref_id, c2b_read_rec *d_recs, c2b_aln_rec *d_alns,
                            uint8_t *d_strings, c2b_edit *d_edits);
/* Optional pairing order for the next c2b_align_batch_device call(s): a permutation of 0..n_reads-1 (device pointer,
 * or NULL to clear) in which reads of equal length (and equal ref_id) are adjacent, so that mixed-length batches still
 * use the packed two-reads-per-warp path.  Results are always written at the reads' own indices.  c2b_align_batch
 * builds this order itself. */
int  c2b_set_pair_order(c2b_engine *e, const int32_t *d_order);
/* op streams / meta words (layout of c2b_align_batch_compact) of the last c2b_align_batch_device call, device pointers */
int  c2b_ops_device(c2b_engine *e, void **d_ops, void **d_meta);
int  c2b_sync(c2b_engine *e);
void *c2b_stream(c2b_engine *e);                    /* cudaStream_t of the engine */
double c2b_last_kernel_ms(c2b_engine *e);           /* CUDA-event time of the last align kernel launch */
int64_t c2b_launch_count(const c2b_engine *e);      /* kernels launched by this engine so far */
/* work items (pairs of reads) since the last c2b_counts_reset that took the packed two-reads-per-warp path /
 * the 32-bit one-read-per-warp path */
int  c2b_path_counts(c2b_engine *e, int64_t *pair_items, int64_t *single_items);
/* packed pairs whose traceback left the banded slab and were re-run with the full slab (as of the last c2b_path_counts) */
int64_t c2b_band_reruns(c2b_engine *e);
/* pairs aligned by the ring-banded DP (four pairs per warp, band proven sufficient by a score bound) / pairs of
 * ring-eligible groups that fell back to the full matrix (as of the last c2b_path_counts) */
int  c2b_ring_counts(c2b_engine *e, int64_t *ring_pairs, int64_t *ring_fallbacks);
/* reads since the last c2b_counts_reset that the diagonal tier proved aligned on the main diagonal / that it did not prove
 * (0 while the tier does not run: C2B_NO_DIAG, no eligible reference) / that went on to the wide-ring second tier, routed
 * there by the diagonal tier or sent by the narrow first tier */
int  c2b_diag_counts(c2b_engine *e, int64_t *proved, int64_t *tier1, int64_t *tier2);
/* of the reads the diagonal tier did not prove since the last c2b_counts_reset: those it sent straight to the wide-ring
 * second tier (its routing test: C2B_NO_ROUTE switches it off) / those it kept for the narrow first tier */
int  c2b_route_counts(c2b_engine *e, int64_t *routed, int64_t *kept);
/* reads since the last c2b_counts_reset that the diagonal tier scored by popcounts of bit planes: reads of codes 0..3 against
 * an amplicon of such codes whose scores over them are two-valued (a match score, a mismatch score) */
int  c2b_diag_popcount_reads(c2b_engine *e, int64_t *reads);

/* replaces: the count vectors / counters built by the quantification loop (CRISPRessoCORE.py:3841-3907,
 * :3964-4115).  Layout above.  c2b_counts_device exposes the block for an NCCL all-reduce.            */
int  c2b_counts_layout(const c2b_engine *e, int32_t *n_refs, int32_t *n_vec, int32_t *stride, int32_t *n_scal);
/* histogram section of each reference's chunk: C2B_NHIST rows of hstride buckets; hist_zero = bucket of key 0 in the
 * two frame rows */
int  c2b_counts_hist_layout(const c2b_engine *e, int32_t *n_hist, int32_t *hstride, int32_t *hist_zero);
int  c2b_counts_reset(c2b_engine *e);
int  c2b_counts_read(c2b_engine *e, int64_t *out, size_t n_int64);
int  c2b_counts_device(c2b_engine *e, void **d_ptr, size_t *n_int64);

/* replaces: CRISPResso2Align.global_align (Align.pyx:101-434), one pair, forward strand only.
 * score_rows as in c2b_ref.  out_read/out_ref need read_len+ref_len bytes; returns C2B_OK or a status.  */
int  c2b_global_align(c2b_engine *e, const char *read, int32_t read_len, const char *ref, int32_t ref_len,
                      const char *alphabet, int32_t nq, const int64_t *score_rows, const int64_t *gap_incentive,
                      int32_t gap_open, int32_t gap_extend,
                      char *out_read, char *out_ref, int32_t *aln_len, int32_t *n_match);

/* replaces: CRISPRessoCOREResources.find_indels_substitutions (COREResources.pyx:68-187) for ONE aligned
 * pair that obeys the aligner's invariants (no column with two gaps, no insertion column adjacent to a
 * deletion column).  Runs the same row-classification kernel as the batch path.  Reconfigures the engine.
 * edits must hold n_cols+1 entries.  Returns C2B_E_ARG when the pair violates the invariants.        */
int  c2b_classify_aligned(c2b_engine *e, const char *read_al, const char *ref_al, int32_t n_cols,
                          const char *alphabet, int32_t nq, const int64_t *include_idx, int32_t n_include,
                          c2b_aln_rec *out, c2b_edit *edits);
/* the same with engine flags: C2B_F_LEGACY_INS selects find_indels_substitutions_legacy (COREResources.pyx:190-315) */
int  c2b_classify_aligned_flags(c2b_engine *e, const char *read_al, const char *ref_al, int32_t n_cols,
                                const char *alphabet, int32_t nq, const int64_t *include_idx, int32_t n_include,
                                uint32_t flags, c2b_aln_rec *out, c2b_edit *edits);

/* replaces: the FASTQ read + de-duplication loop of process_fastq (CRISPRessoCORE.py:1820-1849): four lines per
 * record (text-mode universal newlines), sequence = line 2 stripped of surrounding whitespace, identical sequences
 * counted, unique sequences kept in first-seen order.  Host code (threads), exact (hash placement + byte compare).
 * The result is in the packed layout c2b_align_batch takes: seqs/offsets[n_unique+1]/counts[n_unique].
 * path ending in ".gz" is inflated with zlib.  n_threads <= 0: all hardware threads.                  */
typedef struct c2b_fastq c2b_fastq;
int  c2b_fastq_dedup(const char *path, int32_t n_threads, c2b_fastq **out);
int  c2b_fastq_dedup_buffer(const uint8_t *data, size_t n_bytes, int32_t n_threads, c2b_fastq **out);
int64_t c2b_fastq_n_reads(const c2b_fastq *f);            /* num_reads of :1830 */
int64_t c2b_fastq_n_unique(const c2b_fastq *f);
int32_t c2b_fastq_max_len(const c2b_fastq *f);
const uint8_t *c2b_fastq_seqs(const c2b_fastq *f);
const int64_t *c2b_fastq_offsets(const c2b_fastq *f);
const int32_t *c2b_fastq_counts(const c2b_fastq *f);
const int64_t *c2b_fastq_first_index(const c2b_fastq *f); /* record index of each unique sequence's first occurrence */
void c2b_fastq_free(c2b_fastq *f);
const char *c2b_fastq_last_error(void);
/* the same front end ON the GPU (csrc/c2b_fastq_gpu.cu): the file's bytes cross PCIe once; line index, per-record strip + hash,
 * exact de-duplication in a device hash table (byte compare on a hash match), first-seen order by a radix sort of the groups'
 * first records.  Same c2b_fastq result, same semantics (CRISPRessoCORE.py:1820-1849), gzip inflated on the host first. */
int  c2b_fastq_gpu_available(void);              /* 1 in the CUDA build; 0 in the CPU emulator test build (no device front end) */
int  c2b_fastq_dedup_gpu(const char *path, int32_t device, c2b_fastq **out);
int  c2b_fastq_dedup_gpu_buffer(const uint8_t *data, size_t n_bytes, int32_t device, c2b_fastq **out);
/* replaces: the pass-1 loop of process_bam (CRISPRessoCORE.py:2047-2057) over the text of `samtools view -F <flags> <bam>
 * [<region>]`: one record per line (text-mode universal newlines), its sequence is line.rstrip().split("\t")[9], identical
 * sequences counted in first-seen order.  Same c2b_fastq result and accessors (n_reads = lines).  A line with fewer than 10
 * fields returns C2B_E_LIMIT (IndexError in the reference), a non-ASCII byte C2B_E_ARG (out of contract); the first bad line
 * is named in c2b_fastq_last_error.  _gpu_buffer: line index, one warp per line, exact dedup on the device (C2B_E_STATE in the
 * emulator build); _buffer: host threads (n_threads <= 0: all). */
int  c2b_sam_dedup_gpu_buffer(const uint8_t *data, size_t n_bytes, int32_t device, c2b_fastq **out);
int  c2b_sam_dedup_buffer(const uint8_t *data, size_t n_bytes, int32_t n_threads, c2b_fastq **out);

/* replaces: the reverse-complement count transfer at the head of the quantification loop (CRISPRessoCORE.py:3964-3975) for
 * packed unique reads in first-seen order: weights[k] = the count read k ends up with (0 for a read absorbed by an earlier
 * reverse complement; doubled for a palindrome, as in the reference).  member (NULL = all): reads still in the cache
 * (aligned ones).  Host threads (n_threads <= 0: all).                                                          */
int  c2b_rc_merge_weights(const uint8_t *seqs, const int64_t *offsets, int64_t n, const int32_t *counts,
                          const uint8_t *member, int32_t *weights, int32_t n_threads);

/* Reads the engine cannot take (empty, longer than max_len, a symbol other than A C G T N): out[k] = 1.  Host threads.
 * Returns their number.  (The reference indexes its score table with whatever byte arrives -- lower case out of bounds,
 * Align.pyx:212 -- and its quantification loop raises KeyError on IUPAC codes, CRISPRessoCORE.py:4081.)             */
int64_t c2b_screen_reads(const uint8_t *seqs, const int64_t *offsets, int64_t n, int32_t max_len, uint8_t *out, int32_t n_threads);

/* replaces: the statistics loop of the serial process_fastq branch (CRISPRessoCORE.py:1956-1999) over a batch's records:
 * out[11] = N_TOT_READS, N_CACHED_ALN, N_CACHED_NOTALN, N_COMPUTED_ALN, N_COMPUTED_NOTALN, N_GLOBAL_SUBS, N_SUBS_OUTSIDE_WINDOW,
 * N_MODS_IN_WINDOW, N_MODS_OUTSIDE_WINDOW, N_READS_IRREGULAR_ENDS, READ_LENGTH; aligned[k] = best_match_score > 0.  Host threads. */
int  c2b_serial_stats(const c2b_read_rec *recs, const c2b_aln_rec *alns, const int32_t *counts, int64_t n, int32_t nr,
                      int64_t *out, uint8_t *aligned, int32_t n_threads);

/* replaces: filterFastqs.filterFastqs for single-end input (CRISPResso2/filterFastqs.py:29-229, called at
 * CRISPRessoCORE.py:3716-3717): keep a record iff min(q) >= min_bp_qual_in_read and mean(q) >= min_av_read_qual (each when
 * non-zero), mask bases with q < min_bp_qual_or_N as 'N'; q = byte - 33 (uint8).  Same record/line rules as the reference's
 * binary-mode reader; ".gz" in/out handled.  Returns C2B_E_LIMIT for an empty quality line under the min filter (ValueError in
 * the reference) and C2B_E_ARG for a sequence/quality length mismatch under masking (IndexError in the reference).          */
int  c2b_fastq_filter(const char *path_in, const char *path_out, int32_t min_bp_qual_in_read, int32_t min_av_read_qual,
                      int32_t min_bp_qual_or_N, int32_t n_threads, int64_t *n_in, int64_t *n_out);

/* ---- allele-level consumers (host code, csrc/c2b_alleles.cpp): SURVEY.md section 8(f) rank 2 ----------------------------
 * replaces: the allele table of CRISPRessoCORE.py:3909-3959 + :4298-4303 (rows, %Reads, sort), the text of
 * Alleles_frequency_table.txt (:4498-4535) and CRISPRessoShared.get_dataframe_around_cut[_asymmetrical] (CRISPRessoShared.py:
 * 1513-1531), for alignments held in the compact form of c2b_align_batch_compact.  Row i = one (unique read, reference)
 * alignment: row_read[i] indexes reads/offsets, row_slot[i] indexes ops (NW words per slot) / meta, row_ref[i] the reference,
 * row_count[i] = #Reads.  comp256: byte -> complement byte (reads aligned as their reverse complement).             */
typedef struct c2b_alleles c2b_alleles;
int  c2b_alleles_build(const uint8_t *reads, const int64_t *offsets, const uint64_t *ops, const uint32_t *meta, int32_t NW,
                       int64_t n_rows, const int64_t *row_read, const int64_t *row_slot, const int32_t *row_ref,
                       const int64_t *row_count, int32_t n_refs, const char *const *ref_seqs, const int32_t *ref_lens,
                       const uint8_t *comp256, int32_t n_threads, c2b_alleles **out);
void c2b_alleles_free(c2b_alleles *a);
int64_t        c2b_alleles_n(const c2b_alleles *a);
const int64_t *c2b_alleles_order(const c2b_alleles *a);    /* rows by (#Reads desc, Aligned_Sequence, Reference_Sequence), stable (:4303) */
const uint8_t *c2b_alleles_arena(const c2b_alleles *a);    /* row i: aligned read at arena[offsets[i]], aligned reference right after it */
const int64_t *c2b_alleles_offsets(const c2b_alleles *a);  /* n + 1 */
const int32_t *c2b_alleles_lengths(const c2b_alleles *a);  /* alignment columns per row */
/* header + one line per row of `rows`; name_id / status_id / pct_id index the caller's (small) string tables */
int  c2b_alleles_write_tsv(const c2b_alleles *a, const char *path, int64_t n_sel, const int64_t *rows,
                           const int32_t *name_id, const char *const *names, const int32_t *status_id, const char *const *statuses,
                           const int32_t *n_deleted, const int32_t *n_inserted, const int32_t *n_mutated,
                           const int32_t *pct_id, const char *const *pcts, int32_t n_threads);
/* per-row arrays are indexed by row id; `rows` lists the rows of the (sorted, filtered) DataFrame in its order.
 * -> number of groups, C2B_E_LIMIT when a row's alignment lacks reference position cut_point (ValueError in the reference) */
int64_t c2b_alleles_around_cut(c2b_alleles *a, int64_t n_sel, const int64_t *rows, int32_t cut_point, int32_t plot_left,
                               int32_t plot_right, const uint8_t *unedited, const int32_t *n_deleted, const int32_t *n_inserted,
                               const int32_t *n_mutated, const double *pct);
int32_t c2b_alleles_cut_width(const c2b_alleles *a);
int  c2b_alleles_cut_fetch(const c2b_alleles *a, uint8_t *seq, uint8_t *ref, int32_t *wlen, uint8_t *unedited, int32_t *n_deleted,
                           int32_t *n_inserted, int32_t *n_mutated, int64_t *reads, double *pct);

/* ---- annotated outputs: --fastq_output / --bam_output (csrc/c2b_annotate.cuh on the device, writers in csrc/c2b_fastq.cpp) ----
 * replaces: the per-read annotation of process_fastq_write_out (CRISPRessoCORE.py:2302-2343) and
 * process_single_fastq_write_bam_out (:2399-2497): ALN / ALN_SCORES / ALN_DETAILS / CLASS / MODS / DEL / INS / SUB / ALN_REF /
 * ALN_SEQ text per unique read, and the SAM CIGAR (CRISPRessoShared.CIGAR_LOOKUP + unexplode_cigar, CRISPRessoShared.py:426-434,
 * 561-582), flag and MAPQ of its first aligned reference.  Unique read u (reads / offsets) is batch read bidx[u] of the compact
 * outputs (recs / alns: [n][R], ops: [n][R][NW], meta: [n][R], edits: [n][R][edit_cap], complete lists), or -1 when it was
 * not in the batch (outside the engine's contract: "ALN=NA" with no scores).  Per batch read, decided by the host:
 * amask = slots listed in aln_ref_names (ascending; 0 = not aligned), aname = name id of the one listed slot when it is
 * re-labelled (prime-editing scaffold), else -1, label = class_name id.  names[0..R) are the references' own names;
 * name_rev[id] = refs[name]['aln_strand'] == '-'.  ref_seqs are the R amplicons as aligned.  Uniques go through the device in
 * chunks of `chunk` (<= 0: 65536) through pinned buffers on the engine's stream.  flags: C2B_F_LEGACY_INS, and
 * C2B_ANN_SAM_OPTIONAL for the form of process_bam (:2217-2234): "c2:Z:" instead of the leading space, no ALN_SCORES /
 * ALN_DETAILS for aligned reads (not-aligned reads and reads outside the contract keep them). */
#define C2B_ANN_SAM_OPTIONAL  (1u << 16)
typedef struct c2b_annotation c2b_annotation;
int  c2b_annotate_build(c2b_engine *e, const uint8_t *reads, const int64_t *offsets, int64_t n_unique, const int32_t *bidx,
                        int32_t R, int32_t NW, int32_t edit_cap, const c2b_read_rec *recs, const c2b_aln_rec *alns,
                        const uint64_t *ops, const uint32_t *meta, const c2b_edit *edits,
                        const uint32_t *amask, const int16_t *aname, const int32_t *label,
                        int32_t n_names, const char *const *names, const uint8_t *name_rev,
                        int32_t n_labels, const char *const *labels,
                        const char *const *ref_seqs, const int32_t *ref_lens, const uint8_t *comp256, uint32_t flags,
                        int64_t chunk, c2b_annotation **out);
void c2b_annotate_free(c2b_annotation *a);
int64_t        c2b_annotate_n(const c2b_annotation *a);
const uint8_t *c2b_annotate_arena(const c2b_annotation *a);          /* annotation u: arena[offsets[u] .. offsets[u+1]), leading space */
const int64_t *c2b_annotate_offsets(const c2b_annotation *a);        /* n + 1 */
const uint8_t *c2b_annotate_cigar_arena(const c2b_annotation *a);
const int64_t *c2b_annotate_cigar_offsets(const c2b_annotation *a);
const uint8_t *c2b_annotate_flags(const c2b_annotation *a);          /* SAM flag, 255 = not aligned */
const int32_t *c2b_annotate_mapq(const c2b_annotation *a);
const int16_t *c2b_annotate_first(const c2b_annotation *a);          /* name id of the first aligned reference, -1 */
/* after c2b_annotate_write_sam: record index of each unique read's last SAM line (-1: none), and its id / quality at
 * arena[off[2u] .. off[2u+1]) / arena[off[2u+1] .. off[2u+2]) */
const int64_t *c2b_annotate_last_record(const c2b_annotation *a);
const uint8_t *c2b_annotate_record_arena(const c2b_annotation *a);
const int64_t *c2b_annotate_record_offsets(const c2b_annotation *a);
/* replaces: the record loop of process_fastq_write_out (:2293-2346).  The input is read again (plain, gzip, blocked gzip),
 * split by text-mode readline() rules, every record matched to its unique read (seqs / offsets, the handle's order) by exact
 * sequence; out_path is gzip, one member per thread and 32 MB of text.  C2B_E_ARG: non-ASCII input or a sequence that is in
 * no table.  Host threads (n_threads <= 0: all). */
int  c2b_annotate_write_fastq(const c2b_annotation *a, const uint8_t *seqs, const int64_t *offsets, int64_t n_unique,
                              const char *in_path, const char *out_path, int32_t n_threads);
/* replaces: the record loop of process_single_fastq_write_bam_out (:2387-2502) up to the samtools call: header, then one
 * SAM line per record; chr / pos / rev per name id = refs[name]['aln_chr'], str(refs[name]['aln_start']), aln_strand == '-'. */
int  c2b_annotate_write_sam(c2b_annotation *a, const uint8_t *seqs, const int64_t *offsets, int64_t n_unique,
                            const char *in_path, const char *sam_path, const char *header, int32_t n_names,
                            const char *const *chr, const char *const *pos, const uint8_t *rev, int32_t n_threads);
/* replaces: the pass-2 loop of process_bam (:2251-2262) over the text of `samtools view <bam> [<region>]`: every line whose
 * field 10 is one of the handle's unique reads (seqs / offsets) is appended to sam_path (the caller opened it and wrote the
 * header) as rstrip(line) + "\t" + annotation + "\n", in input order; other lines are dropped.  The annotations should be built
 * with C2B_ANN_SAM_OPTIONAL.  Same line rules and errors as c2b_sam_dedup_buffer.  Host threads (n_threads <= 0: all). */
int  c2b_annotate_write_sam_passthrough(const c2b_annotation *a, const uint8_t *seqs, const int64_t *offsets, int64_t n_unique,
                                        const uint8_t *text, size_t n_bytes, const char *sam_path, int32_t n_threads);

/* replaces: filterFastqs.filterFastqs for paired input (CRISPResso2/filterFastqs.py:230-407, the seven run_*_pair variants): both
 * files in lockstep, a pair kept iff both mates pass; mate 2 strictly above the threshold when only the min or only the mean
 * filter is set (:262, :284); same error mapping as c2b_fastq_filter.                                              */
int  c2b_fastq_filter_pair(const char *path1_in, const char *path2_in, const char *path1_out, const char *path2_out,
                           int32_t min_bp_qual_in_read, int32_t min_av_read_qual, int32_t min_bp_qual_or_N,
                           int32_t n_threads, int64_t *n_in, int64_t *n_out);

/* ---- --vcf_output edit counts (csrc/c2b_vcf.cuh on the device, the sum in csrc/c2b_fastq.cpp) ----
 * replaces: build_edit_counts (CRISPResso2/writers/vcf.py:172-212) over the rows of df_alleles that have edits: every deletion,
 * insertion and substitution of a row becomes one (chrom, pos, REF, ALT) key, deletions and insertions left-normalised
 * (_left_normalize_deletion / _left_normalize_insertion, :9-40, :79-112), and equal keys sum the rows' #Reads.  The rows come
 * packed: per row chrom id (< 0: its Reference_Name is not in amplicon_positions), pos (the amplicon's 1-based start), #Reads,
 * Reference_Sequence / Aligned_Sequence bytes at ref_off / aln_off, ref_positions at rp_off, deletion_coordinates and
 * insertion_coordinates as (a, b) int64 pairs at del_off / ins_off (offsets counted in pairs), insertion_sizes at isz_off and
 * substitution_positions at sub_off (every offset array n_rows + 1 long, starting at 0).  Rows go through the device in chunks
 * of `chunk` rows (<= 0: 16384) through pinned buffers on the engine's stream.
 * Result: the distinct keys in the order the reference's dict has them (first record in row order, then deletions, insertions,
 * substitutions), key i at keys[key_off[i] .. key_off[i+1]) as chrom id (int32 LE) | pos (int64 LE) | len(REF) (int32 LE) |
 * REF | ALT, with its summed #Reads.  When a row raises in the reference, returns C2B_E_ARG with err[0..2] = row, kind
 * (C2B_VCF_E_*), value (the argument of the failed ref_positions.index() for C2B_VCF_E_NOT_IN_LIST): the first such row, and
 * in it the first exception in the reference's order.  err[0] = -1 otherwise.  C2B_E_LIMIT: a sum leaves int64.         */
#define C2B_VCF_E_KEY           1   /* KeyError(Reference_Name) */
#define C2B_VCF_E_NOT_IN_LIST   2   /* ValueError: <value> is not in list */
#define C2B_VCF_E_STRING_INDEX  3   /* IndexError: string index out of range */
#define C2B_VCF_E_EMPTY_MAX     4   /* ValueError: max() iterable argument is empty */
typedef struct c2b_vcf_counts c2b_vcf_counts;
int  c2b_vcf_edit_counts(c2b_engine *e, int64_t n_rows, const int32_t *chrom, const int64_t *pos, const int64_t *reads,
                         const uint8_t *ref, const int64_t *ref_off, const uint8_t *aln, const int64_t *aln_off,
                         const int64_t *rp, const int64_t *rp_off, const int64_t *del, const int64_t *del_off,
                         const int64_t *ins, const int64_t *ins_off, const int64_t *isz, const int64_t *isz_off,
                         const int64_t *sub, const int64_t *sub_off, int64_t chunk, int64_t *err, c2b_vcf_counts **out);
void c2b_vcf_free(c2b_vcf_counts *v);
int64_t        c2b_vcf_n(const c2b_vcf_counts *v);             /* distinct keys */
const uint8_t *c2b_vcf_keys(const c2b_vcf_counts *v);
const int64_t *c2b_vcf_key_offsets(const c2b_vcf_counts *v);   /* n + 1 */
const int64_t *c2b_vcf_reads(const c2b_vcf_counts *v);         /* summed #Reads per key */
int64_t        c2b_vcf_n_records(const c2b_vcf_counts *v);     /* records before the sum */
/* wall time of the call's device pass with its copies, and of the host sum, in ms */
int  c2b_vcf_timings(const c2b_vcf_counts *v, double *device_ms, double *sum_ms);

/* ---- paired-end merge mode (csrc/c2b_paired.cpp) ----
 * get_consensus_alignment_from_pairs (CRISPRessoCORE.py:829-985, get_greater_qual_nuc :801-826): the two mates' alignments to one
 * amplicon (aligned read, aligned amplicon, score, quality string of the read's bases) merged column by column into one aligned
 * read / amplicon / quality triple.  out_* hold at least `cap` >= n1 + n2 bytes.  n_match / n_cols give the homology
 * (round(100 * n_match / n_cols, 3) on the caller's side); caching_is_ok = 0 when a base was chosen by quality.
 * C2B_E_LIMIT: a quality string (or an aligned read) shorter than what the walk over the amplicon strings consumes (IndexError in
 * the reference); C2B_E_STATE: nothing but
 * amplicon gaps (IndexError there too). */
int  c2b_consensus_from_pairs(const char *aln_seq_r1, int32_t ns1, const char *aln_ref_r1, int32_t n1, double score_r1, const char *qual_r1, int32_t nq1,
                              const char *aln_seq_r2, int32_t ns2, const char *aln_ref_r2, int32_t n2, double score_r2, const char *qual_r2, int32_t nq2,
                              char *out_aln, char *out_qual, char *out_ref, int32_t cap,
                              int32_t *n_cols, int32_t *n_qual, int32_t *n_match, int32_t *caching_is_ok);

/* pinned host memory (cudaHostAlloc) for callers that want full-speed host<->device copies */
void *c2b_host_alloc(size_t n_bytes);
void  c2b_host_free(void *p);

#ifdef __cplusplus
}
#endif
#endif

// c2b_fastq_int.h -- result object shared by the host (c2b_fastq.cpp) and GPU (c2b_fastq_gpu.cu) FASTQ front ends.
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

struct c2b_fastq {
    std::unique_ptr<uint8_t[]> seqs;                        // packed unique sequences (uninitialised storage: every byte is written by emit)
    std::vector<int64_t> offsets;
    std::vector<int32_t> counts;
    std::vector<int64_t> first_index;
    int64_t n_reads = 0;
    int32_t max_len = 0;
    std::string err;
};

// byte buffer whose resize() leaves new bytes uninitialised (a whole FASTQ is read or inflated into it: no memset pass first)
template <class T> struct c2b_noinit_alloc : std::allocator<T> {
    template <class U> struct rebind { using other = c2b_noinit_alloc<U>; };
    template <class U> void construct(U *p) { ::new ((void *)p) U; }
    template <class U, class A, class... As> void construct(U *p, A &&a, As &&...as) { ::new ((void *)p) U(std::forward<A>(a), std::forward<As>(as)...); }
};
using c2b_bytes = std::vector<uint8_t, c2b_noinit_alloc<uint8_t>>;

// Read annotations of --fastq_output / --bam_output (built by c2b_annotate_build in c2b_engine.cu, written out by
// c2b_annotate_write_fastq / _sam in c2b_fastq.cpp).  Per unique read u: annotation text ann[ann_off[u] .. ann_off[u+1]) (the
// FASTQ form, with its leading space), CIGAR of the first aligned reference, SAM flag (255: not aligned), MAPQ, name id of the
// first aligned reference.
struct c2b_annotation {
    int64_t n = 0;
    c2b_bytes ann, cig;
    std::vector<int64_t> ann_off, cig_off;
    std::vector<uint8_t> flag;
    std::vector<int32_t> mapq;
    std::vector<int16_t> first;
    // set by c2b_annotate_write_sam: id and quality of each unique read's last record (rec[rec_off[2u] .. rec_off[2u+1]) and
    // rec[rec_off[2u+1] .. rec_off[2u+2])), last_rec[u] = -1 when no record of it was written
    std::vector<int64_t> last_rec, rec_off;
    std::string rec;
};

// --vcf_output edit counts (built by c2b_vcf_edit_counts in c2b_engine.cu): the distinct record keys in first-seen order, key i
// at keys[key_off[i] .. key_off[i+1]), and the summed #Reads of each
struct c2b_vcf_counts {
    std::unique_ptr<uint8_t[]> keys;
    std::vector<int64_t> key_off, reads;
    int64_t n_records = 0;
    double device_ms = 0, sum_ms = 0;
};
// the records rec[i] = arena[off[i] .. off[i+1]) with weights w[i], equal records summed (the exact hash of the FASTQ front end);
// false when a sum leaves int64.  w may be nullptr (no sums); index (optional): index[i] = the number of record i's key
bool c2b_vcf_sum_records(const uint8_t *arena, const int64_t *off, const int64_t *w, int64_t n, c2b_vcf_counts *out,
                         int64_t *index = nullptr);

// One row, or one group, of the tables around the cut before pandas' groupby (get_dataframe_around_cut_asymmetrical,
// get_base_edit_dataframe_around_cut): Aligned_Sequence seq[0 .. len) and Reference_Sequence ref[0 .. len), the other key columns,
// #Reads and %Reads (comp: the Kahan compensation of a group's sum)
struct c2b_cut_group {
    const uint8_t *seq, *ref; int64_t len;
    uint8_t unedited; int64_t ndel, nins, nmut;
    int64_t reads; double pct, comp;
};
// groupby over the six key columns with .sum() in row order, sorted as the reference sorts the result (c2b_alleles.cpp)
std::vector<c2b_cut_group> c2b_group_around_cut(const std::vector<c2b_cut_group> &rows);

// whole file into memory (c2b_fastq.cpp): plain read / gzip inflate (blocked gzip: all host threads)
bool c2b_fastq_read_gz(const char *path, c2b_bytes &buf, std::string &err);
void c2b_fastq_set_error(const std::string &m);
// error of a SAM text line (0-based `line`; kind 0: a non-ASCII byte -> C2B_E_ARG, 1: fewer than 10 fields -> C2B_E_LIMIT)
int c2b_sam_line_error(int64_t line, int kind);

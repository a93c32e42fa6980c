# Small batches through every kernel path, meant to run under compute-sanitizer (memcheck / racecheck / synccheck):
#   compute-sanitizer --tool memcheck python tools/sanitize_check.py
import os, sys, numpy as np
sys.path.insert(0, '.')
from crispresso2_b200 import synth, _lib
from crispresso2_b200.engine import Engine
from oracle import oracle as O
m = O.make_matrix()
rng = np.random.default_rng(3)
amp = synth.random_amplicon(rng, 250)
ref = synth.amplicon_setup(amp)
eng = Engine(0)
# single amplicon: ring path, pair path (mixed lengths), 32-bit path (long reads)
reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, 1200, 250, sub_rate=0.01, rc_frac=0.1, n_rate=0.002, cut=ref['cut_point'])]
reads += [r[:200] for r in reads[:64]] + [(r + r)[:300] for r in reads[:40]]
eng.configure({'Reference': ref}, ['Reference'], m, -20, -2, 5, 2, 0, 'ACGTN', 8)
eng.counts_reset()
res = eng.align(reads)
print('single', eng.path_counts(), eng.ring_counts(), int((res.recs['best_score_milli'] > 0).sum()))
# HDR: three amplicons (multi-reference ring path), ref1 re-projection
hdr = amp[:120] + 'TGA' + amp[123:127] + 'ACGTAC' + amp[127:]
refs = {'WT': ref, 'HDR': synth.amplicon_setup(hdr)}
eng.configure(refs, ['WT', 'HDR'], m, -20, -2, 5, 2, _lib.F_HDR_REF1, 'ACGTN', 8)
eng.counts_reset()
res = eng.align(reads[:600])
print('hdr', eng.path_counts(), eng.ring_counts())
# Pooled: per-read amplicon id, compact outputs
refs, names, rr, rid = {}, [], [], []
for k in range(5):
    a = synth.random_amplicon(rng, 180 + 20 * k)
    refs['a%d' % k] = synth.amplicon_setup(a, guide_start=80)
    names.append('a%d' % k)
    rr += [r.tobytes().decode() for r in synth.synth_reads(rng, a, 100, len(a), cut=refs['a%d' % k]['cut_point'])]
    rid += [k] * 100
eng.configure(refs, names, m, -20, -2, 5, 2, 0, 'ACGTN', 8)
eng.counts_reset()
from crispresso2_b200.engine import pack_reads
buf, off = pack_reads(rr)
res = eng.align_packed(buf, off, ref_id=np.asarray(rid, dtype=np.int32))
print('pooled', eng.path_counts(), eng.ring_counts())
# streamed host batch (one persistent launch fed chunk by chunk)
big = synth.synth_reads_fast(rng, amp, 70000, 250, cut=ref['cut_point'])
eng.configure({'Reference': ref}, ['Reference'], m, -20, -2, 5, 2, 0, 'ACGTN', 8)
eng.counts_reset()
res = eng.align_packed(big.reshape(-1), np.arange(70001, dtype=np.int64) * 250)
print('streamed', eng.path_counts(), int((res.recs['best_score_milli'] > 0).sum()))
# compact outputs with the narrow first tier + legacy insertion quantification
eng.configure({'Reference': ref}, ['Reference'], m, -20, -2, 5, 2, _lib.F_LEGACY_INS, 'ACGTN', 8)
eng.counts_reset()
buf, off = pack_reads(reads[:1200])
res = eng.align_packed(buf, off, compact=True)
print('compact+legacy', eng.path_counts(), eng.ring_counts(), res.strings_block(0, 4).shape)
# diagonal tier with routing: bench-mix batches of 16, 17, 33 and 100 reads (partial units on the narrow and tier-2 lists),
# routing on, off and on for every unproved read
eng.configure({'Reference': ref}, ['Reference'], m, -20, -2, 5, 2, 0, 'ACGTN', 8)
for sw in (None, 'C2B_NO_ROUTE', 'C2B_ROUTE_ALL'):
    if sw:
        os.environ[sw] = '1'
    for nb in (16, 17, 33, 100):
        eng.counts_reset()
        buf, off = pack_reads(reads[:nb])
        res = eng.align_packed(buf, off, compact=True)
        print('route', sw, nb, eng.diag_counts(), eng.route_counts())
    os.environ.pop(sw or 'C2B_NO_ROUTE', None)
# FASTQ front end on the GPU: mixed line ends, blank tail, duplicates
from crispresso2_b200 import fastq
recs = []
for k, s in enumerate(reads[:3000] + reads[:500]):
    e = [b"\n", b"\r\n", b"\r"][k % 3]
    recs.append(b"@r%d" % k + e + s.encode() + e + b"+" + e + b"I" * len(s) + e)
data = b"".join(recs) + b"\n\n"
dd = fastq.dedup_bytes(data, device=0)
hh = fastq.dedup_bytes(data)
assert dd.n_reads == hh.n_reads and np.array_equal(dd.buf, hh.buf) and np.array_equal(dd.counts, hh.counts)
print('gpu ingest', dd.n_reads, len(dd.counts))
# three amplicons whose seed tests disagree for 8 % of the reads (per-reference both-strand alignment inside ALIGN, r02y)
import bench
w3 = bench.Workload("hdr", 2048, 0)
eng.configure(w3.refs, w3.ref_names, m, -20, -2, 5, 2, w3.flags, 'ACGTN', 8)
eng.counts_reset()
res = eng.align_packed(w3.buf, w3.off, compact=True)
print('hdr3', eng.path_counts(), eng.ring_counts(), int((res.recs['best_score_milli'] > 0).sum()))
# read annotations of --fastq_output / --bam_output: size / scan / write kernels over HDR compact results, several chunks
import tempfile, types
from crispresso2_b200 import annotate, core
d = tempfile.mkdtemp(prefix='c2b_sanitize_')
fq = os.path.join(d, 'hdr.fastq')
synth.write_fastq_fast(fq, w3.buf.reshape(w3.n, -1))
a = types.SimpleNamespace(**vars(w3.params))
a.use_legacy_insertion_quantification = False
a.prime_editing_pegRNA_scaffold_seq = a.prime_editing_pegRNA_extension_seq = ''
a.needleman_wunsch_aln_matrix_loc = 'EDNAFULL'
a.n_processes = '1'
cache = {}
core.process_fastq(fq, cache, w3.ref_names, w3.refs, a, [], d, engine=eng, aln_matrix=m)
A = annotate.Annotation(cache, w3.refs, chunk=700)
A.write_fastq(fq, os.path.join(d, 'out.fastq.gz'))
print('annotate', A.n, int(A.ann_off[-1]))
# --bam_input: the SAM front end (k_sam_records, one warp per line) and the process_bam annotation form, several chunks
sam = b"".join(b"r%d\t%d\tc\t1\t42\t250M\t*\t0\t0\t%s\tII\tAS:i:0%s" % (k, 16 * (k & 1), s.encode(), [b"\n", b"\r\n", b"\r"][k % 3])
               for k, s in enumerate(reads[:3000] + reads[:500])) + b"r\t0\tc\t1\t0\t*\t*\t0\t0\tACGT"
ds, hs = fastq.dedup_sam(sam, device=0), fastq.dedup_sam(sam)
assert ds.n_reads == hs.n_reads and np.array_equal(ds.buf, hs.buf) and np.array_equal(ds.counts, hs.counts)
B = annotate.Annotation(cache, w3.refs, chunk=700, sam_optional=True)
print('sam ingest', ds.n_reads, len(ds.counts), 'annotate sam form', B.n, int(B.ann_off[-1]))
import shutil; shutil.rmtree(d, ignore_errors=True)

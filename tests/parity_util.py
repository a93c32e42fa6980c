"""Parity checks shared by the CPU-emulator tests (-m "not gpu") and the GPU tests (-m gpu): the same
assertions run against either build of the engine."""
import types

import numpy as np

import golden_util as G
from crispresso2_b200 import core
from oracle import oracle as O


def edits_canonical(res, r=0):
    """Edit lists of reference slot r in canonical order -- by (type, position); the C ABI promises increasing position per
    type only, and the two-kernel form emits in column order where the general kernel emits per 32-position block --
    entries past n_edits zeroed.  -> (EDIT_DTYPE [n, cap], mask of reads whose list is complete)"""
    ed = res.edits[:, r].copy()
    ne = res.alns[:, r]["n_edits"].astype(np.int64)
    cap = ed.shape[1]
    idx = np.arange(cap)[None, :]
    valid = idx < ne[:, None]
    key = np.where(valid, ed["type"].astype(np.int64) * 100000 + ed["a"], 1 << 40)
    ed = np.take_along_axis(ed, np.argsort(key, axis=1, kind="stable"), axis=1)
    ed[~valid] = 0
    return ed, ne <= cap


def args_from(params):
    a = types.SimpleNamespace(**params)
    a.use_legacy_insertion_quantification = bool(params.get("use_legacy_insertion_quantification", False))
    a.prime_editing_pegRNA_scaffold_seq = params.get("prime_editing_pegRNA_scaffold_seq", "") or ""
    a.needleman_wunsch_aln_matrix_loc = "EDNAFULL"
    a.n_processes = "1"
    if not hasattr(a, "expected_hdr_amplicon_seq"):
        a.expected_hdr_amplicon_seq = ""
    a.prime_editing_pegRNA_extension_seq = params.get("prime_editing_pegRNA_extension_seq", "") or ""
    a.prime_editing_pegRNA_scaffold_min_match_length = params.get("prime_editing_pegRNA_scaffold_min_match_length", 1)
    return a


ALLELE_COLS = ["#Reads", "Aligned_Sequence", "Reference_Sequence", "n_inserted", "n_deleted", "n_mutated", "Reference_Name",
               "Read_Status", "Aligned_Reference_Names", "Aligned_Reference_Scores", "ref_positions", "%Reads"]


def check_alleles(engine, case, tmp_path):
    """Allele-level consumers (crispresso2_b200/alleles.py) against what the UNMODIFIED reference produced for the same FASTQ
    (tests/golden/gen_golden.py): df_alleles as main() handed it to CorePlotContext (every column, the row order and the index),
    the text of Alleles_frequency_table.txt, and the reference's own get_dataframe_around_cut_asymmetrical for every reference,
    guide and two window shapes -- compared as the text pandas writes, byte for byte."""
    from crispresso2_b200 import alleles
    rec = G.load(case)
    refs = G.refs_from(rec)
    fq = tmp_path / (case + ".fastq")
    with open(fq, "w") as fh:
        for k, s in enumerate(rec["reads"]):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    args = args_from(rec["params"])
    if rec.get("ref1", {}).get("ref1_all_deletion_count_vectors") and not args.prime_editing_pegRNA_extension_seq:
        args.expected_hdr_amplicon_seq = refs[rec["ref_names"][1]]["sequence"]
    cache = {}
    core.process_fastq(str(fq), cache, rec["ref_names"], refs, args, [], str(tmp_path), engine=engine, aln_matrix=O.make_matrix())
    t = alleles.AlleleTable(cache)
    want = rec["alleles"]
    assert t.n_total == want["n_total"]
    df = t.to_dataframe()
    assert [int(x) for x in df.index] == want["index"]
    assert {c: str(df[c].dtype) for c in ALLELE_COLS} == want["dtypes"]
    assert df.loc[:, ALLELE_COLS].to_csv(sep="\t", header=True, index=None) == want["tsv"]
    # Alleles_frequency_table.txt (CRISPRessoCORE.py:4514: the nine crispresso2Cols columns of the same frame)
    out = tmp_path / "Alleles_frequency_table.txt"
    t.write_frequency_table(str(out))
    text = out.read_text()
    assert text == df.loc[:, alleles.CRISPRESSO2_COLS].to_csv(sep="\t", header=True, index=None)
    z = tmp_path / "Alleles_frequency_table.zip"
    t.write_frequency_zip(str(z))                           # zips the text file and removes it, as CRISPRessoCORE.py:4529-4531
    import zipfile
    with zipfile.ZipFile(z) as zf:
        assert zf.namelist() == ["Alleles_frequency_table.txt"] and zf.read("Alleles_frequency_table.txt").decode() == text
    assert not out.exists()
    assert want["around_cut"]
    for key, text in want["around_cut"].items():
        rn, cut, pl, pr = key.split("|")
        got = alleles.get_dataframe_around_cut_asymmetrical(df.loc[df["Reference_Name"] == rn], int(cut), int(pl), int(pr))
        assert got.to_csv(sep="\t", header=True) == text, key
    return len(df)


REF1_KEYS = {"ref1_all_insertion_count_vectors": "ref1_all_insertion_count",
             "ref1_all_insertion_left_count_vectors": "ref1_all_insertion_left_count",
             "ref1_all_deletion_count_vectors": "ref1_all_deletion_count",
             "ref1_all_substitution_count_vectors": "ref1_all_substitution_count",
             "ref1_all_indelsub_count_vectors": "ref1_all_indelsub_count"}


def check_golden_case(engine, case, tmp_path, max_reads=None):
    """process_fastq on the fixture's reads must reproduce the reference's variantCache, aln_stats and count files."""
    rec = G.load(case)
    refs = G.refs_from(rec)
    reads = rec["reads"] if max_reads is None else rec["reads"][:max_reads]
    fq = tmp_path / (case + ".fastq")
    with open(fq, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    args = args_from(rec["params"])
    hdr = bool(rec.get("ref1", {}).get("ref1_all_deletion_count_vectors"))
    if hdr and not args.prime_editing_pegRNA_extension_seq:
        args.expected_hdr_amplicon_seq = refs[rec["ref_names"][1]]["sequence"]
    cache = {}
    stats, lost = core.process_fastq(str(fq), cache, rec["ref_names"], refs, args, [], str(tmp_path), engine=engine,
                                     aln_matrix=O.make_matrix())
    if max_reads is None:
        assert stats == rec["aln_stats"]
        assert list(cache.keys()) == list(rec["variants"].keys())
        assert set(lost) == set(rec["not_aligned"])
    for s, got in cache.items():
        want = rec["variants"][s]
        for k in ("aln_ref_names", "aln_scores", "best_match_score", "class_name", "best_match_name"):
            assert got[k] == want[k], (s, k, got[k], want[k])
        if max_reads is None:
            assert got["count"] == want["count"]
        assert [list(d) for d in got["ref_aln_details"]] == want["ref_aln_details"], s
        for r in want["aln_ref_names"]:
            bad = G.payload_equal(want["variant_" + r], got["variant_" + r])
            assert not bad, (s, r, bad, {b: (want["variant_" + r][b], got["variant_" + r][b]) for b in bad})
    for s, got in lost.items():
        assert got["aln_scores"] == rec["not_aligned"][s]["aln_scores"]
    if max_reads is not None:
        return
    block = core.quantify(cache)
    if args.prime_editing_pegRNA_scaffold_seq:              # the reference appended by main() after process_fastq (:3759-3764)
        assert block.ref_names == rec["ref_names"] + ["Scaffold-incorporated"]
        assert any(v["class_name"] == "Scaffold-incorporated" for v in cache.values())
    want_classes = {}
    for s, v in rec["variants"].items():                    # counts as process_fastq left them; the rc merge moves none across classes here
        want_classes[v["class_name"]] = want_classes.get(v["class_name"], 0) + v["count"]
    assert block.class_counts() == want_classes
    for r, seq in zip(block.ref_names, block.ref_seqs):
        V = block.vectors(r)
        tot = block.scalar(r, "TOTAL")
        assert G.mod_count_text(seq, V, tot) == G.file_for(rec, r, "Modification_count_vectors.txt")
        assert G.qw_count_text(seq, V, tot) == G.file_for(rec, r, "Quantification_window_modification_count_vectors.txt")
        nf = G.nuc_freq_rows(G.file_for(rec, r, "Nucleotide_frequency_table.txt"))
        for b in "ACGTN-":
            assert (nf[b] == V["all_base_count_" + b]).all(), (r, b)
        if hdr and max_reads is None:               # ref1_* vectors captured from the reference's CorePlotContext
            R1 = block.vectors_ref1(r)
            for gk, mk in REF1_KEYS.items():
                assert R1[mk].tolist() == rec["ref1"][gk][r], (r, gk)
            for b in "ACGTN-":
                assert R1["ref1_all_base_count_" + b].tolist() == rec["ref1"]["ref1_all_base_count_vectors"][r + "_" + b], (r, b)


def check_against_oracle(engine, refs, ref_names, params, reads, matrix):
    """Engine vs oracle on arbitrary reads: per-read variants, aln_stats, every count vector and counter."""
    import tempfile, os
    cache_o, stats_o, lost_o = O.process_reads(reads, refs, ref_names, params, matrix)
    d = tempfile.mkdtemp()
    fq = os.path.join(d, "r.fastq")
    with open(fq, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    args = args_from({k: getattr(params, k) for k in vars(params)})
    cache = {}
    stats, lost = core.process_fastq(fq, cache, ref_names, refs, args, [], d, engine=engine, aln_matrix=matrix)
    assert stats == stats_o
    assert list(cache.keys()) == list(cache_o.keys())
    assert set(lost) == set(lost_o)
    for s, want in cache_o.items():
        got = cache[s]
        for k in ("count", "aln_ref_names", "aln_scores", "best_match_score", "class_name", "best_match_name"):
            assert got[k] == want[k], (s, k, got[k], want[k])
        assert [tuple(x) for x in got["ref_aln_details"]] == [tuple(x) for x in want["ref_aln_details"]], s
        for r in want["aln_ref_names"]:
            bad = G.payload_equal(want["variant_" + r], got["variant_" + r])
            assert not bad, (s, r, bad)
    extras = {}
    vec, sca, classes, total = O.count_vectors(cache_o, refs, ref_names, params, extras)
    block = core.quantify(cache)
    assert block.class_counts() == classes, (block.class_counts(), classes)
    for r in ref_names:
        V = block.vectors(r)
        for name in O.VECTOR_NAMES:
            assert (V[name] == vec[r][name]).all(), (r, name, np.nonzero(V[name] != vec[r][name]))
        S = block.scalars(r)
        for name in O.SCALAR_NAMES:
            assert S[name] == sca[r][name], (r, name, S[name], sca[r][name])
        H = block.size_histograms(r)
        for name in ("inserted_n", "deleted_n", "substituted_n", "effective_len"):
            assert dict(H[name]) == dict(extras[r][name]), (r, name, H[name], extras[r][name])
        inframe, frameshift = block.frame_histograms(r)
        assert dict(inframe) == dict(extras[r]["hists_inframe"]), (r, inframe, extras[r]["hists_inframe"])
        assert dict(frameshift) == dict(extras[r]["hists_frameshift"]), (r, frameshift, extras[r]["hists_frameshift"])
    if getattr(params, "expected_hdr_amplicon_seq", ""):
        want = O.ref1_vectors(cache_o, refs, ref_names, params)
        for r in ref_names[1:]:
            R1 = block.vectors_ref1(r)
            for name, v in want[r].items():
                assert (R1[name] == v).all(), (r, name)


def check_seed_disagreement(engine, n=1536):
    """Reads whose seed tests disagree across the candidate amplicons (forward for two, both strands for the third -- 8 % of the
    HDR bench workload; plus constructed forward / reverse-complement conflicts): ALIGN gives such a reference its own both-strand
    alignment instead of sending the pair to the general kernel (r02y).  Every field and the count block against the oracle."""
    import bench
    w = bench.Workload("hdr", n, 0)
    reads = [r.tobytes().decode() for r in w.buf.reshape(-1, 250)]
    # conflicts: the front of a forward read joined to the reverse complement of its back half hits forward AND reverse seeds
    reads += [reads[k][:125] + O.reverse_complement(reads[k])[:125] for k in range(0, 64, 2)]
    reads += [O.reverse_complement(reads[k]) for k in range(1, 64, 2)]
    modes = [tuple(O._strand_choice(w.params, s, w.refs[r]) for r in w.ref_names) for s in reads]
    assert sum(1 for m in modes if len(set(m)) > 1) > n // 40
    check_against_oracle(engine, w.refs, w.ref_names, w.params, reads, O.make_matrix())
    return sum(1 for m in modes if len(set(m)) > 1)


def check_pooled(engine, n_amplicons=6, reads_per=40, seed=21, amp_len=(120, 200), matrix=None, go=-20, ge=-2):
    """Config-4 shape (post-demultiplex Pooled): every read carries the index of its single amplicon (ref_id).
    Each (amplicon, read) must equal what the oracle computes with that amplicon alone; the count block of
    amplicon k must equal the oracle's single-amplicon quantification of k's reads.  matrix / go / ge replace EDNAFULL, -20 / -2."""
    from crispresso2_b200 import synth, core
    from crispresso2_b200.engine import pack_reads
    rng = np.random.default_rng(seed)
    m = O.make_matrix() if matrix is None else matrix
    refs, names, reads, rid = {}, [], [], []
    for k in range(n_amplicons):
        L = int(rng.integers(amp_len[0], amp_len[1] + 1))
        amp = synth.random_amplicon(rng, L)
        nm = "amp%d" % k
        refs[nm] = synth.amplicon_setup(amp, guide_start=L // 2 - 10)
        names.append(nm)
        rr = synth.synth_reads(rng, amp, reads_per, L, sub_rate=0.01, rc_frac=0.1, cut=refs[nm]["cut_point"])
        reads += [r.tobytes().decode() for r in rr]
        rid += [k] * reads_per
    order = rng.permutation(len(reads))
    reads = [reads[i] for i in order]
    rid = [rid[i] for i in order]
    engine.configure(refs, names, m, go, ge, 5, 2, 0, "ACGTN", 64)
    engine.counts_reset()
    buf, off = pack_reads(reads)
    res = engine.align_packed(buf, off, ref_id=np.asarray(rid, dtype=np.int32))
    params = O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge)
    per_amp = {k: [] for k in range(n_amplicons)}
    for i, s in enumerate(reads):
        k = rid[i]
        per_amp[k].append(s)
        want = O.new_variant(params, s, {names[k]: refs[names[k]]}, [names[k]], m)
        a = res.alns[i, 0]                              # compact Pooled layout: [read][0]
        assert int(res.recs[i]["best_ref"]) == (k if want["best_match_score"] > 0 else -1)
        assert (res.pair(i, 0)[0], res.pair(i, 0)[1], res.score(i, 0)) == tuple(want["ref_aln_details"][0][1:]), (i, k)
        aligned = want["best_match_score"] > 0
        assert (res.recs[i]["best_score_milli"] > 0) == aligned
        if aligned:
            p = want["variant_" + names[k]]
            assert (int(a["insertion_n"]), int(a["deletion_n"]), int(a["substitution_n"])) == (p["insertion_n"], p["deletion_n"], p["substitution_n"])
            assert bool(a["modified"]) == (p["classification"] == "MODIFIED")
    blk = engine.counts()
    for k in range(n_amplicons):
        nm = names[k]
        cache, stats, lost = O.process_reads(per_amp[k], {nm: refs[nm]}, [nm], params, m)
        # instance-level weights here (no dedup, no rc-merge): compare against the oracle's vectors built the same way
        for s in cache:
            cache[s]["count_keep"] = cache[s]["count"]
        vec, sca, classes, total = O.count_vectors({s: v for s, v in cache.items()}, {nm: refs[nm]}, [nm], params)
        V = blk.vectors(nm)
        # rc-merge only moves weight between a read and its reverse complement, which align identically here
        for name in ("all_deletion_count", "all_substitution_count", "all_insertion_count", "deletion_count", "insertion_count"):
            assert (V[name] == vec[nm][name]).all(), (nm, name)
        assert blk.scalar(nm, "TOTAL") == sca[nm]["counts_total"]


def check_band_fallback(engine, n=24, seed=31):
    """Packed path with the banded traceback slab: alignments that wander off the diagonal (40-60 bp deletions, random
    reads) must trigger the full-slab re-run and still equal the oracle."""
    from crispresso2_b200 import synth
    rng = np.random.default_rng(seed)
    amp = synth.random_amplicon(rng, 250)
    ref = synth.amplicon_setup(amp)
    reads = []
    for k in range(n):
        if k % 3 == 0:
            d = int(rng.integers(40, 61)); a = int(rng.integers(60, 150))
            s = amp[:a] + amp[a + d:] + "".join(rng.choice(list("ACGT"), d))
        elif k % 3 == 1:
            s = "".join(rng.choice(list("ACGT"), 250))
        else:
            s = amp
        reads.append(s[:250])
    import os
    os.environ["C2B_NO_SPLIT"] = "1"                       # the general kernel alone: its packed path keeps a banded slab
    try:
        check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(), reads, O.make_matrix())
        pairs, singles = engine.path_counts()
        assert pairs > 0 and engine.band_reruns() > 0
    finally:
        del os.environ["C2B_NO_SPLIT"]
    # the two-kernel form sends the same pairs to the general kernel with the full slab straight away
    check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(), reads, O.make_matrix())
    engine.path_counts()
    assert engine.band_reruns() == 0


def check_leftover_singles(engine, n=43, seed=77):
    """Left-over list of the ALIGN kernel with single reads on it: pairs in which ONE read fails the ring bound (a random
    read beside an amplicon-like one) put single entries on the list, and an odd read count puts the last read there alone;
    the general kernel takes the list two entries at a time, so a read listed twice would be classified -- and counted --
    twice (r02c: device aln_stats 3 above the per-read records on a 947 601-read batch)."""
    from crispresso2_b200 import synth
    rng = np.random.default_rng(seed)
    amp = synth.random_amplicon(rng, 250)
    ref = synth.amplicon_setup(amp)
    base = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, n, 250, sub_rate=0.01, cut=ref["cut_point"])]
    acgt = list("ACGT")
    reads = []
    for k, s in enumerate(base):
        if k % 7 in (1, 4):                                 # unrelated read: fails the bound, its pair partner passes
            s = "".join(rng.choice(acgt, 250))
        elif k % 11 == 5:                                   # 45-bp deletion: leaves the band
            s = (amp[:80] + amp[125:] + "".join(rng.choice(acgt, 45)))[:250]
        reads.append(s)
    assert len(reads) % 2 == 1
    check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(), reads, O.make_matrix())
    engine.path_counts()
    kept, sent = engine.ring_counts()
    assert kept > 0 and sent > 0, (kept, sent)


def check_legacy(engine, n=120, seed=17):
    """--use_legacy_insertion_quantification (find_indels_substitutions_legacy, COREResources.pyx:190-315) through the whole path,
    one amplicon and HDR mode (the ref1 re-projection uses the legacy function too, CRISPRessoCORE.py:4244-4247): insertions with
    ONE flank in the window, deletions that start at reference position 0 / 1 or reach the last position."""
    from crispresso2_b200 import synth
    rng = np.random.default_rng(seed)
    acgt = list("ACGT")
    amp = synth.random_amplicon(rng, 200)
    ref = synth.amplicon_setup(amp, guide_start=90, window_size=3)
    cut = ref["cut_point"]
    lo, hi = int(min(ref["include_idxs"])), int(max(ref["include_idxs"]))
    reads = [r.tobytes().decode() for r in synth.synth_reads(rng, amp, n, 200, sub_rate=0.01, cut=cut)]
    extra = [amp[1:], amp[2:] + "AC", amp[:-1], amp[:-3] + "GGT", amp[:1] + amp[3:],                       # end rules of the deletion coordinates
             amp[:lo] + "TTTT" + amp[lo:], amp[:hi + 1] + "GG" + amp[hi + 1:], amp[:lo - 1] + "CA" + amp[lo - 1:],   # one flank / both / none in the window
             amp[:hi + 2] + "ACG" + amp[hi + 2:], amp[:cut - 20] + amp[cut + 15:]]
    reads += [(e + "".join(rng.choice(acgt, 200)))[:200] for e in extra]
    check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(use_legacy_insertion_quantification=True), reads,
                         O.make_matrix())
    hdr = amp[:cut - 2] + "TGA" + amp[cut + 1:cut + 4] + "ACGTAC" + amp[cut + 4:]
    ref2 = synth.amplicon_setup(hdr, guide_start=90, window_size=3)
    r2 = [r.tobytes().decode() for r in synth.synth_reads(rng, hdr, 60, 200, del_frac=0.1, ins_frac=0.05, cut=ref2["cut_point"])]
    P = O.Params(use_legacy_insertion_quantification=True, expected_hdr_amplicon_seq=hdr)
    check_against_oracle(engine, {"Reference": ref, "HDR": ref2}, ["Reference", "HDR"], P, reads[:60] + r2 + reads[-10:], O.make_matrix())


def check_narrow_equals_wide(engine, n=640, I=250, seed=59, oracle_subset=0, matrix=None, go=-20, ge=-2, gap_incentive=None):
    """Narrow first tier of the ALIGN kernel (sixteen reads per warp, band of 36 slots, result kept iff the score beats that
    band's bound; everything else re-queued for the 72-slot ring / the full matrix) against the same batch with the tier
    switched off (C2B_NO_NARROW): identical records, op streams, strings, edit lists and count block.  Reads straddle the narrow
    bound: deletions of 1..24 bp, insertions of 1..16 bp, 0..40 substitutions, reverse-complemented and both-strand reads.
    matrix / go / ge / gap_incentive (an I + 1 array) replace EDNAFULL, -20 / -2 and the cut-site incentive.
    -> diag_counts() of the run with the tier"""
    import os
    from crispresso2_b200 import synth
    from crispresso2_b200.engine import pack_reads
    rng = np.random.default_rng(seed)
    amp = synth.random_amplicon(rng, I)
    ref = synth.amplicon_setup(amp, guide_start=max(1, I // 2 - 10))
    m = O.make_matrix() if matrix is None else matrix
    if gap_incentive is not None:
        ref["gap_incentive"] = np.asarray(gap_incentive, dtype=np.int64)
    acgt = list("ACGT")
    comp = {"A": "T", "C": "G", "G": "C", "T": "A", "N": "N"}
    reads = []
    for k in range(n):
        kind = k % 8
        if kind == 0:
            d = int(rng.integers(1, 25)); a = int(rng.integers(20, I - d - 20))
            s = amp[:a] + amp[a + d:] + "".join(rng.choice(acgt, d))
        elif kind == 1:
            d = int(rng.integers(1, 17)); a = int(rng.integers(20, I - 20))
            s = amp[:a] + "".join(rng.choice(acgt, d)) + amp[a:]
        elif kind == 2:
            s = list(amp)
            for p in rng.choice(I, int(rng.integers(0, 41)), replace=False):
                s[p] = acgt[int(rng.integers(0, 4))]
            s = "".join(s)
        elif kind == 3:
            s = "".join(comp[c] for c in reversed(amp))                     # reverse complement
        elif kind == 4:
            s = amp[:40] + "".join(rng.choice(acgt, I - 80)) + amp[-40:]         # few seeds left: both strands tried
        else:
            s = synth.synth_reads(rng, amp, 1, I, sub_rate=0.01, cut=ref["cut_point"])[0].tobytes().decode()
        reads.append(s[:I].ljust(I, "A"))
    buf, off = pack_reads(reads)
    out = []
    for off_switch in (None, "1"):
        if off_switch:
            os.environ["C2B_NO_NARROW"] = off_switch
        try:
            engine.configure({"Reference": ref}, ["Reference"], m, go, ge, 5, 2, 0, "ACGTN", 48)
            engine.counts_reset()
            res = engine.align_packed(buf, off)
            dc = engine.diag_counts()
            cres = engine.align_packed(buf, off, compact=True, count=np.zeros(n, dtype=np.int32), qweight=np.zeros(n, dtype=np.int32))
            out.append((res, engine.counts_raw(), cres, dc))
        finally:
            os.environ.pop("C2B_NO_NARROW", None)
    (a, ca, xa, da), (b, cb, xb, _) = out
    assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
    assert ((xa.meta & 0xffffff) == (xb.meta & 0xffffff)).all() and (((xa.meta >> 24) != 0) == ((xb.meta >> 24) != 0)).all()   # columns, strand; the state byte names the kernel that aligned
    W = a.W
    cols = np.arange(W)[None, :] >= (W - a.alns[:, 0]["aln_len"].astype(np.int64))[:, None]
    assert ((a.strings[:, 0] == b.strings[:, 0]) | ~cols[:, None, :]).all()
    (ea, fa), (eb, fb) = edits_canonical(a), edits_canonical(b)
    assert (fa == fb).all() and (ea[fa] == eb[fb]).all()
    nw = (xa.meta.reshape(-1) & 0xffff).astype(np.int64)                      # op words in use per alignment
    for k in range(n):
        used = (int(nw[k]) + 31) // 32
        assert (xa.ops.reshape(n, -1)[k, :used] == xb.ops.reshape(n, -1)[k, :used]).all(), k
    if oracle_subset:
        check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge),
                             reads[:oracle_subset], m)
    return da


def check_long_pairs(engine, n=40, seed=91):
    """Pairs whose alignment can exceed 512 columns (I + J > 512): since r02g the ALIGN kernel takes them on the packed 16-bit
    path with two op-stream words per lane and half (up to 1024 columns; amplicons of two row blocks included); before, they fell
    to the one-read-per-warp 32-bit path of the general kernel."""
    from crispresso2_b200 import synth
    rng = np.random.default_rng(seed)
    acgt = list("ACGT")
    for I, J in ((300, 290), (450, 300), (280, 250), (500, 312)):
        amp = synth.random_amplicon(rng, I)
        ref = synth.amplicon_setup(amp, guide_start=I // 2 - 10)
        reads = []
        for k in range(n):
            s = synth.synth_reads(rng, amp, 1, I, sub_rate=0.02, cut=ref["cut_point"])[0].tobytes().decode()
            if k % 5 == 1:                                   # a long insertion: many gap columns, alignment well past 512 columns
                p = int(rng.integers(40, I - 60))
                s = s[:p] + "".join(rng.choice(acgt, 60)) + s[p:]
            elif k % 5 == 2:                                 # a read that starts inside the amplicon: long leading gap
                s = s[int(rng.integers(30, 90)):]
            reads.append((s + "".join(rng.choice(acgt, J)))[:J])
        check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(), reads, O.make_matrix())
        pairs, singles = engine.path_counts()
        assert singles <= 8 and pairs > 0, (I, J, pairs, singles)      # the last, incomplete group of eight goes to the general kernel


def check_ring_equals_full(engine, n=96, I=250, seed=41, oracle_subset=0, matrix=None, go=-20, ge=-2, gap_incentive=None):
    """Ring-banded DP (four pairs per warp, only a diagonal band computed, result kept iff the score beats the
    out-of-band bound) against the full-matrix packed path: identical records, alignments, strings, edit lists and
    count block.  Reads are built to straddle the bound: deletions of 1..48 bp, insertions of 1..40 bp, heavy
    substitution loads, random reads.  matrix / go / ge / gap_incentive (an I + 1 array) replace EDNAFULL, -20 / -2 and the
    cut-site incentive."""
    from crispresso2_b200 import synth, _lib
    from crispresso2_b200.engine import pack_reads
    rng = np.random.default_rng(seed)
    amp = synth.random_amplicon(rng, I)
    ref = synth.amplicon_setup(amp, guide_start=max(1, I // 2 - 10))
    m = O.make_matrix() if matrix is None else matrix
    if gap_incentive is not None:
        ref["gap_incentive"] = np.asarray(gap_incentive, dtype=np.int64)
    acgt = list("ACGT")
    reads = []
    for k in range(n):
        kind = k % 6
        if kind == 0:
            d = int(rng.integers(1, 49)); a = int(rng.integers(20, max(21, I - d - 20)))
            s = amp[:a] + amp[a + d:] + "".join(rng.choice(acgt, d))
        elif kind == 1:
            d = int(rng.integers(1, 41)); a = int(rng.integers(20, I - 20))
            s = amp[:a] + "".join(rng.choice(acgt, d)) + amp[a:]
        elif kind == 2:
            s = list(amp)
            for p in rng.choice(I, int(rng.integers(5, 60)), replace=False):
                s[p] = acgt[int(rng.integers(0, 4))]
            s = "".join(s)
        elif kind == 3:
            s = "".join(rng.choice(acgt, I))
        elif kind == 4:
            d = int(rng.integers(25, 40)); a = int(rng.integers(20, I // 2))      # long deletion and long insertion
            s = amp[:a] + amp[a + d:I - 30] + "".join(rng.choice(acgt, d)) + amp[I - 30:]
        else:
            s = synth.synth_reads(rng, amp, 1, I, sub_rate=0.01, cut=ref["cut_point"])[0].tobytes().decode()
        reads.append(s[:I].ljust(I, "A"))
    buf, off = pack_reads(reads)
    out = []
    for flags in (0, _lib.F_NO_RING):
        engine.configure({"Reference": ref}, ["Reference"], m, go, ge, 5, 2, flags, "ACGTN", 40)
        engine.counts_reset()
        res = engine.align_packed(buf, off)
        pc = engine.path_counts()
        out.append((res, engine.counts_raw(), pc, engine.ring_counts()))
    (a, ca, pa, ra), (b, cb, pb, rb) = out
    assert ra[0] > 0 and ra[1] > 0, ra                    # both the ring result and the full-matrix fallback occurred
    assert rb == (0, 0)
    assert (a.recs == b.recs).all() and (a.alns == b.alns).all() and (ca == cb).all()
    W = a.W
    cols = np.arange(W)[None, :] >= (W - a.alns[:, 0]["aln_len"].astype(np.int64))[:, None]
    assert ((a.strings[:, 0] == b.strings[:, 0]) | ~cols[:, None, :]).all()
    (ea, fa), (eb, fb) = edits_canonical(a), edits_canonical(b)
    assert (fa == fb).all() and (ea[fa] == eb[fb]).all()
    if oracle_subset:
        check_against_oracle(engine, {"Reference": ref}, ["Reference"], O.Params(needleman_wunsch_gap_open=go, needleman_wunsch_gap_extend=ge),
                             reads[:oracle_subset], m)
    return ra


def check_coding_seq(engine, n_reads=60, seed=9):
    """--coding_seq quantification (CRISPRessoCORE.py:4083-4180): exon / splicing position sets, a second reference
    whose exons changed length (tot_exon_len_mod != 0), wide window so that window edits fall in and out of the exons."""
    from crispresso2_b200 import synth
    rng = np.random.default_rng(seed)
    amp = synth.random_amplicon(rng, 160)
    hdr = amp[:70] + "TG" + amp[70:]                       # HDR allele: 2-bp insertion inside the first exon
    wt = synth.amplicon_setup(amp, guide_start=55, window_size=25)
    hd = synth.amplicon_setup(hdr, guide_start=55, window_size=25)
    exon = list(range(40, 82)) + list(range(110, 130))
    wt.update(contains_coding_seq=True, exon_positions=exon, exon_len_mods=[0, 0],
              splicing_positions=[38, 39, 82, 83, 108, 109, 130, 131])
    exon_h = list(range(40, 84)) + list(range(112, 132))
    hd.update(contains_coding_seq=True, exon_positions=exon_h, exon_len_mods=[2, 0],
              splicing_positions=[38, 39, 84, 85, 110, 111, 132, 133])
    refs = {"WT": wt, "HDR": hd}
    reads = []
    for a, cut in ((amp, wt["cut_point"]), (hdr, hd["cut_point"])):
        reads += [r.tobytes().decode() for r in synth.synth_reads(rng, a, n_reads, len(a), sub_rate=0.02, rc_frac=0.1,
                                                                    del_frac=0.35, ins_frac=0.25, cut=cut)]
    m = O.make_matrix()
    for kw in ({"expected_hdr_amplicon_seq": hdr}, {"expected_hdr_amplicon_seq": hdr, "ignore_substitutions": True},
               {"expected_hdr_amplicon_seq": hdr, "discard_indel_reads": True},
               {"expected_hdr_amplicon_seq": hdr, "ignore_insertions": True, "ignore_deletions": True}):
        check_against_oracle(engine, refs, ["WT", "HDR"], O.Params(**kw), reads, m)
    far = {"WT": dict(wt, exon_positions=list(range(5, 30)) + list(range(135, 150)), splicing_positions=[3, 4, 30, 31, 62, 63])}
    check_against_oracle(engine, far, ["WT"], O.Params(), reads[:n_reads], m)    # edits near the cut touch no exon
    nc = {"WT": dict(wt, contains_coding_seq=False, exon_positions=[], exon_len_mods=[], splicing_positions=[])}
    check_against_oracle(engine, {"WT": wt}, ["WT"], O.Params(), reads[:n_reads], m)
    check_against_oracle(engine, nc, ["WT"], O.Params(), reads[:n_reads], m)


def check_random_config(engine, seed):
    """One random configuration against the oracle: 1-3 amplicons (WT / HDR-like / SNP allele), random guide position, window
    size and excluded ends, optional coding-sequence masks with exon length changes, 3-70 reads of assorted lengths drawn from
    the alleles (deletions, insertions, substitutions, N, reverse complements), random ignore / discard / ambiguity / HDR flags."""
    from crispresso2_b200 import synth
    m = O.make_matrix()
    rng = np.random.default_rng(seed)
    L = int(rng.integers(60, 270))
    amp = synth.random_amplicon(rng, L)
    nref = int(rng.integers(1, 4))
    gs = int(rng.integers(20, max(21, L - 45)))
    wsize = int(rng.choice([1, 1, 3, 10, 25]))
    refs, names, seqs = {}, [], []
    for k in range(nref):
        s = list(amp)
        if k == 1:                                   # HDR-like: small substitution + insertion
            p = gs + 10
            s[p] = "A" if s[p] != "A" else "C"
            ins = "".join(rng.choice(list("ACGT"), int(rng.integers(0, 7))))
            s = s[:p + 2] + list(ins) + s[p + 2:]
        elif k == 2:                                 # a few SNPs
            for p in rng.choice(len(s), size=4, replace=False):
                s[p] = "G" if s[p] != "G" else "T"
        s = "".join(s)
        nm = "R%d" % k
        refs[nm] = synth.amplicon_setup(s, guide_start=min(gs, len(s) - 40), window_size=wsize,
                                        exclude_left=int(rng.integers(0, 16)), exclude_right=int(rng.integers(0, 16)))
        if rng.random() < 0.4:
            ex = sorted(set(rng.integers(0, len(s), size=int(rng.integers(5, 60))).tolist()))
            refs[nm].update(contains_coding_seq=True, exon_positions=ex, splicing_positions=sorted(set(rng.integers(0, len(s), size=6).tolist())),
                            exon_len_mods=[int(rng.choice([0, 0, 0, 2, -3]))])
        names.append(nm); seqs.append(s)
    reads = []
    nreads = int(rng.integers(3, 70))
    for _ in range(nreads):
        k = int(rng.integers(0, nref))
        s = seqs[k]
        rl = int(rng.choice([len(s), len(s), len(amp), int(rng.integers(30, 300))]))
        r = synth.synth_reads(rng, s, 1, rl, sub_rate=float(rng.choice([0.0, 0.01, 0.05])), del_frac=0.3, ins_frac=0.2,
                              rc_frac=float(rng.choice([0.0, 0.3])), n_rate=float(rng.choice([0.0, 0.01])), cut=refs[names[k]]["cut_point"])[0].tobytes().decode()
        reads.append(r)
    kw = {}
    for f in ("ignore_substitutions", "ignore_insertions", "ignore_deletions", "discard_indel_reads"):
        if rng.random() < 0.2: kw[f] = True
    if nref > 1:
        u = rng.random()
        if u < 0.3: kw["expand_ambiguous_alignments"] = True
        elif u < 0.5: kw["assign_ambiguous_alignments_to_first_reference"] = True
        if rng.random() < 0.6: kw["expected_hdr_amplicon_seq"] = seqs[1]
    check_against_oracle(engine, refs, names, O.Params(**kw), reads, m)

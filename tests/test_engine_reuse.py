"""Results read after their engine is reused.  process_fastq leaves lazy variantCache entries and compact op streams that are
spelled on first read, and engines are shared and reconfigured all the time: another sample, get_new_variant_object,
global_align, classify_pair, AlignmentMemo, the annotation and VCF passes all run on the same engine.  Every case here runs a
sample A, makes one intervening call on the same engine, and only then reads what A left behind -- entries, not-aligned dict,
count block, allele table and a compact batch -- against the oracle and against a twin of A read at once on a fresh engine.
Then the order and lifetime edges (half read before and half after, the reverse order, Engine.close(), the release of a
cache's results) and the device state across a scripted sequence of batches on one engine.  Runs on the CPU warp emulator;
with -m gpu the same checks run through the sm_90a library on cuda:0."""
import copy
import functools
import gc
import os
import sys
import weakref

import numpy as np
import pytest

import golden_util as G
import parity_util as PU
from crispresso2_b200 import _lib, alleles, core, lazy, synth
from crispresso2_b200.engine import Engine, EngineError, pack_reads
from oracle import oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module", params=["emu", pytest.param("gpu", marks=pytest.mark.gpu)])
def lib(request):
    """library path of the warp-emulator build; None (the sm_90a library on cuda:0) with -m gpu"""
    if request.param == "gpu":
        return None
    sys.path.insert(0, os.path.join(HERE, "emu"))
    import build_emu
    return build_emu.build()


@pytest.fixture(scope="module")
def eng(lib):
    """the one engine every case reuses"""
    return Engine(0, lib_path=lib)


# ------------------------------------------------------------------------------------------------------------ runs
class Run:
    """one sample: amplicons, arguments, reads, and what it must give (oracle, or the reference's golden record)"""

    def __init__(self, refs, names, reads, params, matrix=None, rec=None):
        self.refs, self.names, self.reads, self.params = refs, list(names), reads, params
        self.matrix = O.make_matrix() if matrix is None else matrix
        self.rec = rec
        self.args = PU.args_from(rec["params"] if rec else vars(params))
        if rec is None and getattr(params, "expected_hdr_amplicon_seq", ""):
            self.args.expected_hdr_amplicon_seq = params.expected_hdr_amplicon_seq
        if rec is not None and rec.get("ref1", {}).get("ref1_all_deletion_count_vectors") and not self.args.prime_editing_pegRNA_extension_seq:
            self.args.expected_hdr_amplicon_seq = refs[names[1]]["sequence"]


def _amplicons(rng, lens, window_size=1):
    refs, names = {}, []
    for k, L in enumerate(lens):
        amp = synth.random_amplicon(rng, L)
        refs["amp%d" % k] = synth.amplicon_setup(amp, guide_start=L // 2 - 10, window_size=window_size)
        names.append("amp%d" % k)
    return refs, names


def _reads(rng, refs, names, per, **kw):
    out = []
    for nm in names:
        s = refs[nm]["sequence"]
        kw2 = dict(dict(sub_rate=0.02, rc_frac=0.2, del_frac=0.2, ins_frac=0.15, cut=refs[nm]["cut_point"]), **kw)
        out += [r.tobytes().decode() for r in synth.synth_reads(rng, s, per, len(s), **kw2)]
    return out


def _junk(rng, n, L=150):
    return ["".join(rng.choice(list("ACGT"), L)) for _ in range(n)]


def run_one():
    rng = np.random.default_rng(5)
    refs, names = _amplicons(rng, [200])
    reads = _reads(rng, refs, names, 50, n_rate=0.003)
    return Run(refs, names, reads + reads[:10] + _junk(rng, 2), O.Params())


def run_hdr3():
    """three amplicons, the second the HDR allele: ALIGN, CLASSIFY and the general kernel, the ref1 re-projection"""
    rng = np.random.default_rng(6)
    amp = synth.random_amplicon(rng, 200)
    hdr = amp[:98] + "TGA" + amp[101:104] + "ACGTAC" + amp[104:]
    snp = "".join(("G" if c != "G" else "T") if k in (30, 150, 170) else c for k, c in enumerate(amp))
    refs = {"WT": synth.amplicon_setup(amp, guide_start=90), "HDR": synth.amplicon_setup(hdr, guide_start=90),
            "SNP": synth.amplicon_setup(snp, guide_start=90)}
    names = ["WT", "HDR", "SNP"]
    reads = _reads(rng, refs, names, 25)
    return Run(refs, names, reads + reads[:6] + _junk(rng, 1), O.Params(expected_hdr_amplicon_seq=hdr))


def run_six():
    rng = np.random.default_rng(7)
    refs, names = _amplicons(rng, [120, 200, 150, 180, 140, 210])
    return Run(refs, names, _reads(rng, refs, names, 8), O.Params())


def run_coding():
    rng = np.random.default_rng(9)
    amp = synth.random_amplicon(rng, 160)
    hdr = amp[:70] + "TG" + amp[70:]
    wt = synth.amplicon_setup(amp, guide_start=55, window_size=25)
    hd = synth.amplicon_setup(hdr, guide_start=55, window_size=25)
    wt.update(contains_coding_seq=True, exon_positions=list(range(40, 82)) + list(range(110, 130)), exon_len_mods=[0, 0],
              splicing_positions=[38, 39, 82, 83, 108, 109, 130, 131])
    hd.update(contains_coding_seq=True, exon_positions=list(range(40, 84)) + list(range(112, 132)), exon_len_mods=[2, 0],
              splicing_positions=[38, 39, 84, 85, 110, 111, 132, 133])
    refs = {"WT": wt, "HDR": hd}
    reads = _reads(rng, refs, ["WT", "HDR"], 30, del_frac=0.35, ins_frac=0.25, rc_frac=0.1)
    return Run(refs, ["WT", "HDR"], reads, O.Params(expected_hdr_amplicon_seq=hdr))


def run_legacy():
    rng = np.random.default_rng(17)
    refs, names = _amplicons(rng, [200], window_size=3)
    amp = refs["amp0"]["sequence"]
    lo, hi = int(min(refs["amp0"]["include_idxs"])), int(max(refs["amp0"]["include_idxs"]))
    extra = [amp[1:] + "A", amp[:lo] + "TTTT" + amp[lo:-4], amp[:hi + 1] + "GG" + amp[hi + 1:-2], amp[:1] + amp[3:] + "CA"]
    return Run(refs, names, _reads(rng, refs, names, 50) + extra, O.Params(use_legacy_insertion_quantification=True))


def run_overflow():
    """reads with more edits than the batch's cap of 12: process_fastq re-runs them with complete lists (the `fix` results)"""
    rng = np.random.default_rng(23)
    refs, names = _amplicons(rng, [200])
    return Run(refs, names, _reads(rng, refs, names, 20, sub_rate=0.02) + _reads(rng, refs, names, 20, sub_rate=0.12), O.Params())


def run_prime():
    """the prime-editing fixture with a scaffold sequence: scaffold passes of core._batch, reads re-labelled
    'Scaffold-incorporated'; checked against the reference's own outputs"""
    rec = G.load("fanc_pe_scaffold")
    return Run(G.refs_from(rec), rec["ref_names"], rec["reads"], None, rec=rec)


RUNS = {"one": run_one, "hdr3": run_hdr3, "six": run_six, "coding": run_coding, "legacy": run_legacy, "overflow": run_overflow,
        "prime": run_prime}
_memo = {}


def the_run(name):
    if name not in _memo:
        _memo[name] = RUNS[name]()
    return _memo[name]


def fastq(tmp, reads, name):
    p = os.path.join(str(tmp), name)
    with open(p, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))
    return p


def process(engine, tmp, run, name="a.fastq", args=None, cache=None, **kw):
    cache = {} if cache is None else cache
    st, lost = core.process_fastq(fastq(tmp, run.reads, name), cache, run.names, run.refs, args or run.args, [], str(tmp),
                                  engine=engine, aln_matrix=run.matrix, **kw)
    return cache, lost, st


# ------------------------------------------------------------------------------------------------------------ reading
def unique_reads(run):
    seen = {}
    for s in run.reads:
        seen[s] = 1
    return list(seen)


def compact_batch(engine, run):
    """a compact batch of A's unique reads on the engine as A's process_fastq configured it"""
    core.configure_engine(engine, run.args, run.refs, run.names, run.matrix)
    buf, off = pack_reads(unique_reads(run))
    n = len(off) - 1
    return engine.align_packed(buf, off, count=np.zeros(n, dtype=np.int32), qweight=np.zeros(n, dtype=np.int32), compact=True)


def _canon(v):
    out = {}
    for k in v:
        x = v[k]
        if k.startswith("variant_"):
            out[k] = {f: G._norm(x[f]) for f in x.__slots__ if hasattr(x, f)}
        elif k == "ref_aln_details":
            out[k] = [list(d) for d in x]
        else:
            out[k] = G._norm(x)
    return out


def read_all(cache, lost, res, run):
    """everything A left behind, spelled now: entries, not-aligned dict, count block, allele table, compact pairs"""
    block = core.quantify(cache)
    blk = {"classes": block.class_counts(), "raw": block.raw.tolist(), "names": list(block.ref_names)}
    for r in block.ref_names:
        blk["v_" + r] = {k: np.asarray(x).tolist() for k, x in block.vectors(r).items()}
        blk["s_" + r] = dict(block.scalars(r))
    df = alleles.AlleleTable(cache).to_dataframe()
    nr = res.alns.shape[1]
    pairs = [[res.pair(i, r) if int(res.meta[i, r]) >> 24 else None for r in range(nr)] for i in range(len(res.recs))]
    return {"cache": {s: _canon(v) for s, v in cache.items()}, "lost": {s: _canon(v) for s, v in lost.items()},
            "keys": list(cache), "block": blk, "alleles": df.loc[:, PU.ALLELE_COLS].to_csv(sep="\t", index=None), "pairs": pairs}


def oracle_of(run):
    if not hasattr(run, "want"):
        if run.rec is not None:
            run.want = None
        else:
            cache_o, st_o, lost_o = O.process_reads(run.reads, run.refs, run.names, run.params, run.matrix)
            extras = {}
            cc = copy.deepcopy(cache_o)
            vec, sca, classes, _ = O.count_vectors(cc, run.refs, run.names, run.params, extras)
            run.want = (cache_o, st_o, lost_o, vec, sca, classes)
    return run.want


def check_oracle(run, st, got):
    """the spelled results against the oracle (or, for the golden fixture, the reference's recorded outputs)"""
    if run.rec is not None:
        rec = run.rec
        assert st == rec["aln_stats"]
        assert got["keys"] == list(rec["variants"])
        assert set(got["lost"]) == set(rec["not_aligned"])
        for s, want in rec["variants"].items():
            v = got["cache"][s]
            for k in ("aln_ref_names", "aln_scores", "best_match_score", "class_name", "best_match_name", "count"):
                assert v[k] == G._norm(want[k]), (s, k)
            assert v["ref_aln_details"] == want["ref_aln_details"], s
            for r in want["aln_ref_names"]:
                assert not G.payload_equal(want["variant_" + r], v["variant_" + r]), (s, r)
        for s, want in rec["not_aligned"].items():
            assert got["lost"][s]["aln_scores"] == want["aln_scores"]
        classes = {}
        for v in rec["variants"].values():
            classes[v["class_name"]] = classes.get(v["class_name"], 0) + v["count"]
        assert got["block"]["classes"] == classes
        for r in got["block"]["names"]:
            V = {k: np.asarray(x) for k, x in got["block"]["v_" + r].items()}
            seq = run.refs[r if r in run.refs else core.PE_REF]["sequence"]
            assert G.mod_count_text(seq, V, got["block"]["s_" + r]["counts_total"]) == G.file_for(rec, r, "Modification_count_vectors.txt")
        return
    cache_o, st_o, lost_o, vec, sca, classes = oracle_of(run)
    assert st == st_o
    assert got["keys"] == list(cache_o)
    assert set(got["lost"]) == set(lost_o)
    for s, want in cache_o.items():
        v = got["cache"][s]
        assert set(v) == set(want), s
        for k in ("count", "aln_ref_names", "aln_scores", "best_match_score", "class_name", "best_match_name"):
            assert v[k] == G._norm(want[k]), (s, k, v[k], want[k])
        assert v["ref_aln_details"] == [list(d) for d in want["ref_aln_details"]], s
        for r in want["aln_ref_names"]:
            assert not G.payload_equal(want["variant_" + r], v["variant_" + r]), (s, r)
    for s, want in lost_o.items():
        v = got["lost"][s]
        assert set(v) == set(want) and v["count"] == want["count"] and v["aln_scores"] == want["aln_scores"], s
        assert v["ref_aln_details"] == [list(d) for d in want["ref_aln_details"]] and v["best_match_score"] == want["best_match_score"]
    assert got["block"]["classes"] == classes
    for r in run.names:
        for name in O.VECTOR_NAMES:
            assert got["block"]["v_" + r][name] == vec[r][name].tolist(), (r, name)
        for name in O.SCALAR_NAMES:
            assert got["block"]["s_" + r][name] == sca[r][name], (r, name)
    # the compact batch: every (read, amplicon) slot spells the oracle's alignment
    want_all = dict(lost_o, **cache_o)
    for i, s in enumerate(unique_reads(run)):
        if s not in want_all:
            continue
        for r, d in enumerate(want_all[s]["ref_aln_details"]):
            assert got["pairs"][i][r] == (d[1], d[2]), (i, r)


_twins = {}


def twin(lib, tmp, name):
    """A on a fresh engine, read at once"""
    key = (lib, name)
    if key not in _twins:
        e = Engine(0, lib_path=lib)
        run = the_run(name)
        cache, lost, st = process(e, tmp, run, "twin.fastq")
        got = read_all(cache, lost, compact_batch(e, run), run)
        check_oracle(run, st, got)
        _twins[key] = got
        e.close()
    return _twins[key]


# ------------------------------------------------------------------------------------------------------------ intervening calls
def _other_run(n, L, seed):
    rng = np.random.default_rng(seed)
    refs, names = _amplicons(rng, [L] * n)
    return Run(refs, names, _reads(rng, refs, names, max(2, 24 // n)), O.Params())


def _same_amplicons(run, matrix=None, strip_coding=False, **flags):
    refs = run.refs
    if strip_coding:
        refs = {k: dict(v, contains_coding_seq=False) for k, v in refs.items()}
    b = Run(refs, run.names, run.reads[::-1][:40], run.params, matrix=matrix if matrix is not None else run.matrix, rec=run.rec)
    b.args = copy.copy(run.args)
    for k, v in flags.items():
        setattr(b.args, k, v)
    return b


def _pf(run_of):
    def call(engine, tmp, run, ctx):
        b = run_of(run)
        process(engine, tmp, b, "b.fastq")
    return call


def _flag(flag, value=True):
    def call(engine, tmp, run, ctx):
        strip = flag == "use_legacy_insertion_quantification" and any(r.get("contains_coding_seq") for r in run.refs.values())
        process(engine, tmp, _same_amplicons(run, strip_coding=strip, **{flag: value}), "b.fastq")
    return call


def _bam(engine, tmp, run, ctx):
    import bam_util as BU
    from crispresso2_b200 import bam
    b = _other_run(2, 160, 41)
    recs = [dict(qname="q%d" % k, flag=0, rname="*", pos=0, mapq=0, cigar="*", seq=s, qual="F" * len(s), tags=[])
            for k, s in enumerate(b.reads)]
    path = os.path.join(str(tmp), "b.bam")
    BU.write_bam(path, "@HD\tVN:1.0\tSO:unsorted\n@SQ\tSN:chr1\tLN:5000\n", [("chr1", 5000)], recs)
    old, version = os.environ["PATH"], bam._version
    os.environ["PATH"] = BU.fake_samtools(os.path.join(str(tmp), "bin"))
    bam._version = lambda: "0"                                 # the @PG line's version, taken from the reference where installed
    try:
        args = copy.copy(b.args)
        args.samtools_exclude_flags, args.debug = "0", False
        bam.process_bam(path, "", os.path.join(str(tmp), "out.bam"), {}, b.names, b.refs, args, [], str(tmp), engine=engine,
                        aln_matrix=b.matrix)
    finally:
        os.environ["PATH"], bam._version = old, version


def _global_align(engine, tmp, run, ctx):
    from crispresso2_b200 import align
    b = _other_run(1, 330, 43)
    ref = b.refs[b.names[0]]
    s1, s2, sc = align.global_align(b.reads[0], ref["sequence"], b.matrix, ref["gap_incentive"], -20, -2, engine=engine)
    assert (s1, s2, sc) == O.global_align(b.reads[0], ref["sequence"], b.matrix, ref["gap_incentive"], -20, -2)


def _classify_pair(engine, tmp, run, ctx):
    aln, _ = engine.classify_pair("ACGT-ACGTTACGGA", "ACGTTACG-TACGGA", list(range(15)))
    assert (int(aln["deletion_n"]), int(aln["insertion_n"])) == (1, 1) and engine.n_refs == 0


def _new_variant(engine, tmp, run, ctx):
    b = _other_run(2, 260, 47)
    v = core.get_new_variant_object(b.args, b.reads[1], b.refs, b.names, b.matrix, engine=engine)
    want = O.new_variant(b.params, b.reads[1], b.refs, b.names, b.matrix)
    assert [list(d) for d in v["ref_aln_details"]] == [list(d) for d in want["ref_aln_details"]]


def _memo_call(engine, tmp, run, ctx):
    from crispresso2_b200 import paired
    b = _other_run(3, 140, 53)
    m = paired.AlignmentMemo(engine, b.reads, b.refs, b.names, b.matrix, -20, -2)
    ref = b.refs[b.names[0]]
    assert m.global_align(b.reads[0], ref["sequence"], b.matrix, ref["gap_incentive"], -20, -2) == \
        O.global_align(b.reads[0], ref["sequence"], b.matrix, ref["gap_incentive"], -20, -2)


def _annotate(engine, tmp, run, ctx):
    from crispresso2_b200 import annotate
    b = _other_run(1, 240, 59)
    pf = functools.partial(core.process_fastq, engine=engine, aln_matrix=b.matrix)
    annotate.process_fastq_write_out(fastq(tmp, b.reads, "b.fastq"), os.path.join(str(tmp), "b.out.fastq.gz"), {}, b.names, b.refs,
                                     b.args, [], str(tmp), process_fastq=pf)


def _vcf(engine, tmp, run, ctx):
    from crispresso2_b200 import vcf
    b = _other_run(1, 230, 61)
    cache, _, _ = process(engine, tmp, b, "b.fastq")
    import vcf_util as V
    assert vcf.build_edit_counts(V.frame_from_cache(cache), {b.names[0]: ("chr1", 1000)}, engine=engine)


def _shared_twice(engine, tmp, run, ctx):
    for k, (n, L) in enumerate(((1, 200), (4, 150))):
        b = _other_run(n, L, 67 + k)
        core.process_fastq(fastq(tmp, b.reads, "b%d.fastq" % k), {}, b.names, b.refs, b.args, [], str(tmp), engine=None,
                           aln_matrix=b.matrix)


CALLS = {
    "pf_same_length": _pf(lambda run: _other_run(1, len(run.refs[run.names[0]]["sequence"]), 101)),
    "pf_shorter": _pf(lambda run: _other_run(1, 90, 102)),
    "pf_longer": _pf(lambda run: _other_run(1, 420, 103)),
    "pf_1": _pf(lambda run: _other_run(1, 150, 104)),
    "pf_2": _pf(lambda run: _other_run(2, 150, 105)),
    "pf_5": _pf(lambda run: _other_run(5, 150, 106)),
    "pf_32": _pf(lambda run: _other_run(32, 64, 107)),
    "same_gaps": _pf(lambda run: _same_amplicons(run, needleman_wunsch_gap_open=-12, needleman_wunsch_gap_extend=-1)),
    "same_matrix": _pf(lambda run: _same_amplicons(run, matrix=O.make_matrix(3, -2, -1, 0))),
    "same_seeds": _pf(lambda run: _same_amplicons(run, aln_seed_count=2, aln_seed_min=0)),
    "legacy": _flag("use_legacy_insertion_quantification"),
    "discard_indel": _flag("discard_indel_reads"),
    "ignore_substitutions": _flag("ignore_substitutions"),
    "ignore_insertions": _flag("ignore_insertions"),
    "ignore_deletions": _flag("ignore_deletions"),
    "expand_ambiguous": _flag("expand_ambiguous_alignments"),
    "assign_first": _flag("assign_ambiguous_alignments_to_first_reference"),
    "process_bam": _bam,
    "global_align": _global_align,
    "classify_pair": _classify_pair,
    "get_new_variant_object": _new_variant,
    "alignment_memo": _memo_call,
    "annotate": _annotate,
    "build_edit_counts": _vcf,
    "shared_engine_twice": _shared_twice,
}
# every intervening call after the one-amplicon run; calls that move max_I, n_refs and the alphabet after every other run
SHORT = ["pf_longer", "pf_5", "classify_pair"]
CASES = [("one", c) for c in CALLS] + [(r, c) for r in ("hdr3", "six", "coding", "legacy", "overflow", "prime") for c in SHORT]


@pytest.mark.parametrize("run_name,call", CASES)
def test_read_after_reuse(eng, lib, tmp_path, monkeypatch, run_name, call):
    """A, one intervening call on the same engine, then everything A left behind: equal to the oracle and to a twin read at
    once on a fresh engine"""
    want = twin(lib, tmp_path, run_name)
    run = the_run(run_name)
    monkeypatch.setitem(core._engines, (0, None), eng)        # get_engine(): the shared engine is this one
    cache, lost, st = process(None if call == "shared_engine_twice" else eng, tmp_path, run)
    if run_name == "overflow":
        assert core.source_of(cache).parts[0][2]              # reads re-run with complete edit lists
    table_before = alleles.AlleleTable(cache).to_dataframe().loc[:, PU.ALLELE_COLS].to_csv(sep="\t", index=None)
    res = compact_batch(eng, run)
    CALLS[call](eng, tmp_path, run, None)
    got = read_all(cache, lost, res, run)
    assert got["alleles"] == table_before
    check_oracle(run, st, got)
    assert got == want


# ------------------------------------------------------------------------------------------------------------ order and lifetime
def test_half_read_before_half_after(eng, lib, tmp_path):
    run = the_run("hdr3")
    want = twin(lib, tmp_path, "hdr3")
    cache, lost, st = process(eng, tmp_path, run)
    keys = list(cache)
    first = {s: _canon(cache[s]) for s in keys[::2]}
    _pf(lambda r: _other_run(5, 260, 111))(eng, tmp_path, run, None)
    got = {s: _canon(cache[s]) for s in keys[1::2]}
    assert first == {s: want["cache"][s] for s in keys[::2]}
    assert got == {s: want["cache"][s] for s in keys[1::2]}


def test_reverse_order(eng, lib, tmp_path):
    """B stays right after A's entries were read while B's were unread"""
    a, b = the_run("one"), the_run("six")
    wa, wb = twin(lib, tmp_path, "one"), twin(lib, tmp_path, "six")
    ca, la, _ = process(eng, tmp_path, a)
    cb, lb, _ = process(eng, tmp_path, b, "b.fastq")
    assert {s: _canon(v) for s, v in ca.items()} == wa["cache"]
    _pf(lambda r: _other_run(2, 300, 113))(eng, tmp_path, a, None)
    assert {s: _canon(v) for s, v in cb.items()} == wb["cache"] and {s: _canon(v) for s, v in lb.items()} == wb["lost"]


def test_alignment_memo_after_reconfiguration(eng, tmp_path):
    from crispresso2_b200 import paired
    b = _other_run(3, 180, 127)
    m = paired.AlignmentMemo(eng, b.reads, b.refs, b.names, b.matrix, -20, -2)
    process(eng, tmp_path, _other_run(7, 120, 131), "c.fastq")
    eng.classify_pair("ACGTACGT", "ACGTACGT", [3])
    for k in (0, 5, len(b.reads) - 1):
        for nm in b.names:
            ref = b.refs[nm]
            m0 = m.hits
            got = m.global_align(b.reads[k], ref["sequence"], b.matrix, ref["gap_incentive"], -20, -2)
            assert m.hits == m0 + 1                          # answered from the memo's batch
            assert got == O.global_align(b.reads[k], ref["sequence"], b.matrix, ref["gap_incentive"], -20, -2)


def test_close_while_a_lazy_cache_is_alive(lib, tmp_path):
    """after Engine.close() the entries, count block, allele table and compact batch of its runs still read right; the
    annotation pass, which needs the engine's device, raises an EngineError naming the cause"""
    from crispresso2_b200 import annotate
    run = the_run("hdr3")
    want = twin(lib, tmp_path, "hdr3")
    e = Engine(0, lib_path=lib)
    cache, lost, st = process(e, tmp_path, run)
    res = compact_batch(e, run)
    e.close()
    got = read_all(cache, lost, res, run)
    check_oracle(run, st, got)
    assert got == want
    with pytest.raises(EngineError, match="closed"):
        annotate.Annotation(cache, run.refs)


def test_results_are_released_with_the_cache(eng, tmp_path):
    run = the_run("one")
    cache, lost, _ = process(eng, tmp_path, run)
    src = weakref.ref(core.source_of(cache))
    assert core.quantify(cache) is src().block
    cache[next(iter(cache))]["class_name"]                    # one entry materialised, the rest lazy
    del cache, lost
    gc.collect()
    assert src() is None
    for fn in (core.source_of, core.quantify, alleles.AlleleTable):
        with pytest.raises(KeyError):
            fn({})
    # a cache no read aligned to is answered while the call's not-aligned dict holds the results; a cache emptied afterwards
    # holds nothing that leads to them
    junk = Run(run.refs, run.names, _junk(np.random.default_rng(3), 4), O.Params())
    cache, lost, st = process(eng, tmp_path, junk, "junk.fastq")
    assert not cache and len(lost) == 4 and st["N_COMPUTED_NOTALN"] == 4
    src = weakref.ref(core.source_of(cache))
    assert core.quantify(cache).class_counts() == {}
    del lost
    gc.collect()
    assert src() is None
    with pytest.raises(KeyError):
        core.quantify(cache)
    cache, lost, _ = process(eng, tmp_path, run)
    cache.clear()
    with pytest.raises(KeyError):
        core.quantify(cache)


# ------------------------------------------------------------------------------------------------------------ device state
def _batch(engine, refs, names, reads, compact, ref_id=None, cap=24, matrix=None):
    engine.configure(refs, names, O.make_matrix() if matrix is None else matrix, -20, -2, 5, 2, 0, "ACGTN", cap)
    engine.counts_reset()
    buf, off = pack_reads(reads)
    n = len(reads)
    w = np.ones(n, dtype=np.int32)
    res = engine.align_packed(buf, off, count=w, qweight=w, ref_id=ref_id, compact=compact)
    tiers = (engine.path_counts(), engine.diag_counts(), engine.diag_popcount_reads(), engine.ring_counts(), engine.route_counts())
    out = {"recs": res.recs.tobytes(), "alns": res.alns.tobytes(), "counts": engine.counts_raw().tobytes(), "tiers": tiers}
    if res.edits is not None:                                 # entries past a slot's n_edits are not part of the output
        ed = res.edits.copy()
        ed[np.arange(ed.shape[2])[None, None, :] >= res.alns["n_edits"].astype(np.int64)[:, :, None]] = 0
        out["edits"] = ed.tobytes()
    ends = [(0, min(n, 2048)), (max(0, n - 2048), n)]        # strings of the first and last reads (all of a small batch)
    if compact:
        m = res.meta
        out["meta"] = m.tobytes()
        cols = (m & 0xffff).astype(np.int64)
        nw = res.ops.shape[2]
        used = np.arange(nw)[None, None, :] < ((cols + 31) // 32)[:, :, None]
        out["ops"] = np.where(used, res.ops, 0).tobytes()
        out["strings"] = [res.strings_block(a, b).tobytes() for a, b in ends]
    else:
        W = res.W
        live = np.arange(W)[None, None, :] >= (W - res.alns["aln_len"].astype(np.int64))[:, :, None]
        out["strings"] = np.where(live[:, :, None, :], res.strings, 0).tobytes()
    return out


def _scripted(gpu):
    """(label, refs, names, reads, compact, ref_id, cap) batches of assorted sizes, amplicon counts and output forms"""
    rng = np.random.default_rng(71)
    one = _amplicons(rng, [250])
    six = _amplicons(rng, [120, 200, 150, 180, 140, 210])
    big = _amplicons(rng, [330, 90])
    r_one = _reads(rng, *one, 64, sub_rate=0.02)
    r_six = _reads(rng, *six, 12)
    r_big = _reads(rng, *big, 24, sub_rate=0.05)
    rid = np.repeat(np.arange(6, dtype=np.int32), 12)
    sizes = (17, 64 << 10, 1 << 20) if gpu else (17, 48, 120)
    chunk = None if gpu else "40"                              # the emulator's batches are small: the test hook chunks them

    def tile(reads, n):
        return [reads[k % len(reads)] for k in range(n)]
    steps = [("17_one_strings", one, r_one[:17], False, None, 24, None),
             ("mid_six_compact", six, tile(r_six, sizes[1]), True, None, 24, chunk),
             ("large_one_compact", one, tile(r_one, sizes[2]), True, None, 4, chunk),
             ("pooled_six", six, r_six, True, rid, 24, None),
             ("17_six_strings", six, r_six[:17], False, None, 24, None),
             ("mid_two_strings", big, tile(r_big, sizes[1] // 4), False, None, 40, chunk),
             ("17_one_compact", one, r_one[-17:], True, None, 12, None),
             ("pooled_six_chunked", six, r_six[::-1], True, rid[::-1].copy(), 24, "16"),
             ("17_one_strings_again", one, r_one[:17], False, None, 24, None)]
    return steps


def test_device_state_across_batches(eng, lib, monkeypatch):
    """one engine through a scripted sequence of batches: every batch equals the same batch on a fresh engine -- records,
    alignments, op streams, strings, edit lists, count block and the tier counters; batches above the pipeline's chunk
    take the chunked path, the rest the unchunked one"""
    steps = _scripted(lib is None)
    for label, (refs, names), reads, compact, rid, cap, chunk in steps:
        if chunk:
            monkeypatch.setenv("C2B_CHUNK", chunk)
        else:
            monkeypatch.delenv("C2B_CHUNK", raising=False)
        got = _batch(eng, refs, names, reads, compact, rid, cap)
        fresh = Engine(0, lib_path=lib)
        want = _batch(fresh, refs, names, reads, compact, rid, cap)
        fresh.close()
        for k in want:
            assert got[k] == want[k], (label, k)

"""Shared by tests/test_base_edit.py (warp emulator) and tests/test_gpu_base_edit.py (sm_90a): the reference's own
get_upset_plot_counts / get_base_edit_dataframe_around_cut (plots/data_prep.py, CRISPRessoShared.py of the package under
oracle/_ref/install), the frames both are compared on, and the comparisons: the same dict with its key order and item types,
or the same frame under pandas' exact checks, or the same exception type and message."""
import os
import sys
import tempfile

import numpy as np
import pandas as pd

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, HERE):
    if p not in sys.path:
        sys.path.insert(0, p)

HAVE_REF = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "install", "CRISPResso2", "plots", "data_prep.py"))
_REF = {}


def reference():
    """-> (get_upset_plot_counts, get_base_edit_dataframe_around_cut) of the unmodified reference, as first imported"""
    if not _REF:
        from baseline import ref_shim
        ref_shim.load_core()
        from CRISPResso2 import CRISPRessoShared
        from CRISPResso2.plots import data_prep
        _REF["upset"] = data_prep.get_upset_plot_counts
        _REF["quilt"] = CRISPRessoShared.get_base_edit_dataframe_around_cut
    return _REF["upset"], _REF["quilt"]


def _outcome(fn):
    try:
        return "ok", fn()
    except Exception as ex:                                     # noqa: BLE001 -- the exception is the result compared
        return type(ex), str(ex)


def check_upset(df, bp, wt, engine, chunk=0):
    """the drop-in against the reference on one frame -> the reference's outcome"""
    from crispresso2_b200 import base_edit
    want = _outcome(lambda: reference()[0](df, bp, wt))
    got = _outcome(lambda: base_edit.get_upset_plot_counts(df, bp, wt, engine=engine, chunk=chunk))
    assert got[0] == want[0], (got, want)
    if want[0] != "ok":
        assert got[1] == want[1], (got, want)
        return want
    g, w = got[1], want[1]
    assert list(g) == list(w)
    for k in w:
        if k.endswith("_allele_counts"):
            assert type(g[k]) is type(w[k]) and g[k].default_factory is int, k
            assert list(g[k].items()) == list(w[k].items()), k            # first-seen key order
            assert all(type(v) is int for v in g[k].values()), k
        else:
            assert g[k] == w[k], (k, g[k], w[k])
            assert all(type(v) is int for v in (g[k] if isinstance(g[k], list) else [g[k]])), k
    return want


def check_quilt(df, nuc, engine, chunk=0):
    from crispresso2_b200 import base_edit
    want = _outcome(lambda: reference()[1](df, nuc))
    got = _outcome(lambda: base_edit.get_base_edit_dataframe_around_cut(df, nuc, engine=engine, chunk=chunk))
    assert got[0] == want[0], (got, want)
    if want[0] != "ok":
        assert got[1] == want[1], (got, want)
        return want
    if len(df) == 0:
        assert got[1] is df
    else:
        pd.testing.assert_frame_equal(got[1], want[1], check_exact=True, check_index_type=True, check_column_type=True,
                                      check_names=True)
    return want


def row(ref, aln, reads=1, name="A", status=None, n=(0, 0, 0), pct=None):
    """an allele row with the columns both functions read (n = n_inserted, n_deleted, n_mutated)"""
    return {"#Reads": reads, "Aligned_Sequence": aln, "Reference_Sequence": ref, "n_inserted": n[0], "n_deleted": n[1],
            "n_mutated": n[2], "Reference_Name": name,
            "Read_Status": status or ("UNMODIFIED" if aln == ref else "MODIFIED"),
            "%Reads": float(reads) if pct is None else pct}


def frame(rows):
    return pd.DataFrame(rows)


R = "ACGTCCAGTCAGCTA"                                         # positions 0..14


def hand_cases():
    """-> [(label, frame, bp_substitutions_arr, wt_ref_name)] at the edges of get_upset_plot_counts' semantics"""
    bp = [(4, "C", "T"), (5, "C", "T"), (9, "C", "T")]
    out = []
    sub = R[:4] + "T" + R[5:]
    out.append(("substitutions", frame([row(R, sub, 5, n=(0, 0, 1)), row(R, R, 7), row(R, R[:4] + "TT" + R[6:], 3, n=(0, 0, 2)),
                                        row(R, R[:9] + "G" + R[10:], 2, n=(0, 0, 1))]), bp, "A"))
    out.append(("leading_insertion_run", frame([row("--" + R, "GG" + R, 4, n=(2, 0, 0)), row("---" + R, "TTA" + R, 1, n=(3, 0, 0))]),
                [(0, "A", "G"), (1, "C", "T")], "A"))
    out.append(("insertion_after_last_base", frame([row(R + "--", R + "CC", 2, n=(2, 0, 0))]), [(14, "A", "G"), (13, "T", "C")], "A"))
    out.append(("deletion_then_insertion", frame([row(R[:4] + "-" + R[4:], R[:4] + "-T" + R[5:], 3, n=(0, 1, 0)),
                                                  row(R[:5] + "-" + R[5:], R[:4] + "-G" + R[5:], 2, n=(1, 1, 0))]), bp, "A"))
    out.append(("deletion", frame([row(R, R[:4] + "-" + R[5:], 6, n=(0, 1, 0)), row(R, R[:4] + "--" + R[6:], 1, n=(0, 2, 0))]), bp, "A"))
    out.append(("all_gap_reference", frame([row("----", "ACGT", 2), row("-", "AC", 1)]), [(0, "A", "C"), (1, "A", "C")], "A"))
    out.append(("targets_past_and_negative", frame([row(R, R, 2), row(R, sub, 1)]), [(-1, "A", "T"), (15, "A", "T"), (40, "", "T"),
                                                                                 (4, "C", "T")], "A"))
    out.append(("mod_base_gap_and_long", frame([row(R, R[:4] + "-" + R[5:], 3, n=(0, 1, 0)), row(R[:5] + "-" + R[5:], R[:5] + "A" + R[5:], 2)]),
                [(4, "C", "-"), (4, "C", "CA"), (5, "C", "")], "A"))
    out.append(("empty_bp", frame([row(R, sub, 3, n=(0, 0, 1)), row(R, R, 4), row(R, R[:3] + "-" + R[4:], 5, n=(0, 1, 0))]), [], "A"))
    out.append(("other_references", frame([row(R, sub, 3, n=(0, 0, 1)), row("", "", 8, name="B"), row(R, "AC", 2, name="AMBIGUOUS_A"),
                                           row(R, R, 1, name="B"), row(R, R, 5)]), bp, "A"))
    out.append(("no_row_on_reference", frame([row(R, R, 1, name="B")]), bp, "A"))
    out.append(("key_order_ties", frame([row(R, R[:4] + t + R[5:], 2, n=(0, 0, 1)) for t in "TGATGCA"] + [row(R, R, 2)]), bp, "A"))
    out.append(("longer_aligned_sequence", frame([row(R, R + "AAA", 2)]), bp, "A"))
    out.append(("reads_zero_and_negative", frame([row(R, sub, 0, n=(0, 0, 1)), row(R, sub, -3, n=(0, 0, 1)), row(R, R, 2)]), bp, "A"))
    return out


def upset_error_cases():
    """-> [(label, frame, bp, wt)] whose reference call raises: the first failing row in frame order wins"""
    bp = [(4, "C", "T")]
    good = row(R, R, 2)
    return [
        ("empty_reference_sequence", frame([good, row("", "", 1), row(R, "AC", 1)]), bp, "A"),
        ("short_aligned_sequence", frame([good, row("B" + R, R, 1, name="B"), row(R, R[:-1], 3), row("", "", 1)]), bp, "A"),
        ("short_under_leading_gaps", frame([row("---" + R, "GG", 1)]), bp, "A"),
        ("missing_reads", frame([good]).drop(columns=["#Reads"]), bp, "A"),
        ("missing_reference_name", frame([good]).drop(columns=["Reference_Name"]), bp, "A"),
        ("missing_n_deleted", frame([good]).drop(columns=["n_deleted"]), bp, "A"),
        ("missing_aligned_sequence", frame([good]).drop(columns=["Aligned_Sequence"]), bp, "A"),
        ("missing_on_other_reference_only", frame([row(R, R, 1, name="B")]).drop(columns=["Aligned_Sequence", "n_deleted"]), bp, "A"),
    ]


def quilt_cases():
    """-> [(label, frame, conversion_nuc_from)]"""
    rows = [row(R, R, 40, n=(0, 0, 0)), row(R, R[:4] + "T" + R[5:], 25, n=(0, 0, 1)), row(R, R[:4] + "TT" + R[6:], 20, n=(0, 0, 2)),
            row(R[:5] + "-" + R[5:], R[:5] + "A" + R[5:], 7, n=(1, 0, 0)), row(R, R[:4] + "-" + R[5:], 3, n=(0, 1, 0)),
            row(R, R[:2] + "A" + R[3:], 25, n=(0, 0, 1)), row(R, R[:13] + "C" + R[14:], 20, n=(0, 0, 1), status="MODIFIED"),
            row(R, R, 5, name="B")]
    out = [("nuc_" + c, frame(rows), c) for c in "ACGT"]
    out.append(("nuc_CT", frame(rows), "CT"))
    out.append(("nuc_lowercase", frame(rows), "c"))
    # %Reads whose Kahan-compensated sum differs from the naive one
    kahan = [row(R, R, 1, pct=p) for p in (1e16, 1.0, 1.0, 1.0, -1e16, 0.1, 0.2, 0.3)]
    out.append(("kahan", frame(kahan), "C"))
    ties = [row(R, R[:4] + a + R[5:9] + b + R[10:], 3, n=(0, 0, 1), status=s) for a in "TC" for b in "CG" for s in ("MODIFIED", "UNMODIFIED")]
    out.append(("ties", frame(ties + [row(R, R, 3, n=(1, 0, 0))]), "C"))
    out.append(("empty_frame", frame([row(R, R)]).iloc[:0], "C"))
    return out


def quilt_error_cases():
    good = row(R, R, 2)
    return [
        ("short_aligned", frame([good, row(R, R[:3], 1), row(R, R[:1], 1)]), "C"),
        ("short_past_nuc", frame([good, row("AAAA" + R, "AAAA", 1)]), "G"),
        ("missing_reference_sequence", frame([good]).drop(columns=["Reference_Sequence"]), "C"),
        ("missing_status", frame([good]).drop(columns=["Read_Status"]), "C"),
        ("missing_aligned", frame([good]).drop(columns=["Aligned_Sequence"]), "C"),
        ("missing_aligned_unused", frame([row("AAAA", "AAAA", 1)]).drop(columns=["Aligned_Sequence"]), "C"),
        ("missing_aligned_and_status", frame([good]).drop(columns=["Aligned_Sequence", "Read_Status"]), "C"),
    ]


# ------------------------------------------------------------------------------------------------ base-editing reads
FANC_GUIDE = "GGAATCCCTTCTGCAGCACC"


def fanc():
    """the FANC amplicon of tests/golden/gen_golden.py"""
    with open(os.path.join(HERE, "golden", "gen_golden.py")) as fh:
        src = fh.read()
    ns = {}
    for name in ("FANC", "FANC_HDR"):
        start = src.index(name + " = (")
        end = src.index(")\n", start) + 1
        exec(src[start:end], ns)
    return ns["FANC"], ns["FANC_HDR"]


def base_edit_reads(rng, amp, n, guide=FANC_GUIDE, nuc_from="C", nuc_to="T"):
    """FANC.Cas9-like base-editing reads: the guide's conversion_nuc_from bases converted in random combinations, a few reads
    with an indel at the cut, some unedited"""
    g = amp.index(guide)
    cs = [g + i for i, c in enumerate(guide) if c == nuc_from]
    cut = g + len(guide) - 3
    out = []
    for k in range(n):
        s = list(amp)
        kind = k % 10
        if kind < 7:
            for p in cs:
                if rng.random() < 0.5:
                    s[p] = nuc_to
        if kind == 7:                                           # deletion at the cut
            d = int(rng.integers(1, 5))
            s = s[:cut] + s[cut + d:]
        elif kind == 8:                                         # insertion at the cut, with a conversion
            if cs:
                s[cs[0]] = nuc_to
            s = s[:cut] + list("ACGT"[int(rng.integers(0, 4))] * int(rng.integers(1, 3))) + s[cut:]
        out.append("".join(s))
    return out


def write_fastq(path, reads):
    with open(path, "w") as fh:
        for k, s in enumerate(reads):
            fh.write("@r%d\n%s\n+\n%s\n" % (k, s, "I" * len(s)))


def engine_frame(engine, amps, reads):
    """df_alleles of one process_fastq run (AlleleTable.to_dataframe(), as main() sees it) over `reads` against `amps` (named
    A, B, ...)"""
    from crispresso2_b200 import core, synth
    from crispresso2_b200.alleles import AlleleTable
    from oracle import oracle as O
    from parity_util import args_from
    names = [chr(ord("A") + k) for k in range(len(amps))]
    refs = {nm: synth.amplicon_setup(a, guide_start=amps[0].index(FANC_GUIDE), window_size=20) for nm, a in zip(names, amps)}
    params = O.Params()
    d = tempfile.mkdtemp()
    fq = os.path.join(d, "r.fastq")
    write_fastq(fq, reads)
    cache = {}
    core.process_fastq(fq, cache, names, refs, args_from({k: getattr(params, k) for k in vars(params)}), [], d, engine=engine,
                       aln_matrix=O.make_matrix())
    return AlleleTable(cache).to_dataframe(), names


def guide_targets(amp, guide=FANC_GUIDE, nuc_from="C", nuc_to="T"):
    g = amp.index(guide)
    return [(g + i, nuc_from, nuc_to) for i, c in enumerate(guide) if c == nuc_from]

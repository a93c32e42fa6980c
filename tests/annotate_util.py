"""Shared helpers of tests/test_annotate.py (CPU, emulator engine) and tests/test_gpu_annotate.py (sm_90a library): the
reference's own process_fastq_write_out / process_single_fastq_write_bam_out (with its own process_fastq) against
crispresso2_b200.annotate on the same inputs.

The (ref_names, refs, args) a CRISPResso run hands to those functions are captured from the UNMODIFIED reference main()
(oracle/_ref/install) run in a subprocess: `python annotate_util.py capture <out.pickle> -- <CRISPResso argv>`.

TEST INFRASTRUCTURE: needs oracle/_ref/install.
"""
import copy
import functools
import gzip
import os
import pickle
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

import numpy as np  # noqa: E402


def have_reference():
    return os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "install", "CRISPResso2", "CRISPRessoCORE.py"))


def fake_samtools(dirpath):
    """a `samtools` stand-in on PATH: `sort IN -o OUT` copies, `index OUT` touches OUT.bai -> PATH value"""
    os.makedirs(dirpath, exist_ok=True)
    path = os.path.join(dirpath, "samtools")
    with open(path, "w") as fh:
        fh.write('#!/bin/sh\nif [ "$1" = sort ]; then cp "$2" "$4"; exit $?; fi\n'
                 'if [ "$1" = index ]; then : > "$2.bai"; exit 0; fi\nexit 1\n')
    os.chmod(path, 0o755)
    return str(dirpath) + os.pathsep + os.environ.get("PATH", "")


def amplicons():
    with open(os.path.join(HERE, "golden", "gen_golden.py")) as fh:
        src = fh.read()
    ns = {}
    for name in ("FANC", "FANC_HDR"):
        start = src.index(name + " = (")
        exec(src[start:src.index(")\n", start) + 1], ns)
    return ns["FANC"], ns["FANC_HDR"]


def capture(tmp, argv):
    """(ref_names, refs, args) the reference's main() passes to its read loop for this argv (run with --bam_output, so refs
    carry aln_chr / aln_start / aln_strand)"""
    out = os.path.join(str(tmp), "capture_%d.pickle" % abs(hash(tuple(argv))))
    outdir = os.path.join(str(tmp), "capture_run")
    p = subprocess.run([sys.executable, os.path.abspath(__file__), "capture", out, outdir, "--"] + list(argv),
                       capture_output=True, text=True, timeout=600)
    assert p.returncode == 0 and os.path.exists(out), p.stdout[-3000:] + p.stderr[-3000:]
    with open(out, "rb") as fh:
        return pickle.load(fh)


def _capture_main():
    out, outdir = sys.argv[2], sys.argv[3]
    argv = sys.argv[sys.argv.index("--") + 1:]
    from baseline import ref_shim
    CORE = ref_shim.load_core()

    def spy(fastq_input, bam_output, bam_header, variantCache, ref_names, refs, args, files_to_remove, output_directory):
        with open(out, "wb") as fh:
            pickle.dump((list(ref_names), refs, args), fh)
        sys.stdout.flush()
        os._exit(0)

    CORE.process_single_fastq_write_bam_out = spy
    os.makedirs(outdir, exist_ok=True)
    sys.argv = ["CRISPResso"] + argv + ["--bam_output", "--suppress_plots", "--suppress_report", "-o", outdir]
    CORE.main()


def bam_header(ref_names, refs):
    """main()'s header (CRISPRessoCORE.py:3473-3485)"""
    h = "@HD\tVN:1.0\tSO:unknown\n"
    for name in ref_names:
        h += "@SQ\tSN:%s\tLN:%s\n" % (name, refs[name]["sequence_length"])
    return h


def same(a, b, path="v"):
    """equality of two variant dicts as the reference's consumers see them (payload objects compared by their slots)"""
    if type(a).__name__ == "ResultsSlotsDict" or type(b).__name__ == "ResultsSlotsDict":
        # payloads: a slots object, or a plain dict in the reference's legacy mode (COREResources.pyx:298) -- fields compared
        da, db = (x if isinstance(x, dict) else x.__dict__ for x in (a, b))
        assert sorted(da) == sorted(db), (path, sorted(da), sorted(db))
        for k in da:
            same(da[k], db[k], path + "." + k)
        return
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a.keys()) == list(b.keys()), (path, list(a.keys()), list(b.keys()))
        for k in a:
            same(a[k], b[k], path + "[%r]" % (k,))
        return
    if isinstance(a, np.ndarray):
        assert np.array_equal(a, np.asarray(b)) and a.dtype.kind == np.asarray(b).dtype.kind, path
        return
    if isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for k, (x, y) in enumerate(zip(a, b)):
            same(x, y, "%s[%d]" % (path, k))
        return
    assert a == b and type(a) is type(b) or (isinstance(a, (int, float, np.number)) and a == b), (path, a, b)


class Pair:
    """One input through the reference's wrapper and through ours."""

    def __init__(self, CORE, engine, tmp, ref_names, refs, args):
        self.CORE, self.engine, self.tmp = CORE, engine, str(tmp)
        self.ref_names, self.refs, self.args = ref_names, refs, args
        from crispresso2_b200 import core
        loc = args.needleman_wunsch_aln_matrix_loc
        self.matrix = core.read_matrix(loc if os.path.isabs(loc) else os.path.join(CORE._ROOT, loc))
        self.pf = functools.partial(core.process_fastq, engine=engine, aln_matrix=self.matrix)

    def fastq(self, fastq_input, tag="f"):
        from crispresso2_b200 import annotate, lazy
        out_r, out_b = os.path.join(self.tmp, tag + "_ref.fastq.gz"), os.path.join(self.tmp, tag + "_b200.fastq.gz")
        cache_r, cache_b = {}, {}
        res_r = self.CORE.process_fastq_write_out(fastq_input, out_r, cache_r, self.ref_names, copy.deepcopy(self.refs), self.args, [],
                                                  self.tmp)
        res_b = annotate.process_fastq_write_out(fastq_input, out_b, cache_b, self.ref_names, copy.deepcopy(self.refs), self.args, [],
                                                 self.tmp, process_fastq=self.pf)
        lazies = [v for v in cache_b.values() if isinstance(v, lazy.LazyVariant)]
        untouched = all(getattr(v, "_k", -1) >= 0 for v in lazies) and len(lazies) == len(cache_b)
        with gzip.open(out_r, "rb") as fh:
            text_r = fh.read()
        with gzip.open(out_b, "rb") as fh:
            text_b = fh.read()
        return res_r, res_b, cache_r, cache_b, text_r, text_b, untouched

    def sam(self, fastq_input, tag="s", refs=None, debug=True):
        from crispresso2_b200 import annotate
        refs = refs or self.refs
        args = copy.copy(self.args)
        args.debug = debug
        header = bam_header(self.ref_names, refs)
        bam_r, bam_b = os.path.join(self.tmp, tag + "_ref.bam"), os.path.join(self.tmp, tag + "_b200.bam")
        cache_r, cache_b = {}, {}
        res_r = self.CORE.process_single_fastq_write_bam_out(fastq_input, bam_r, header, cache_r, self.ref_names, copy.deepcopy(refs),
                                                             args, [], self.tmp)
        res_b = annotate.process_single_fastq_write_bam_out(fastq_input, bam_b, header, cache_b, self.ref_names, copy.deepcopy(refs),
                                                            args, [], self.tmp, process_fastq=self.pf)
        outs = []
        for p in (bam_r + ".sam", bam_b + ".sam") if debug else (bam_r, bam_b):
            with open(p, "rb") as fh:
                outs.append(fh.read())
        return res_r, res_b, cache_r, cache_b, outs[0], outs[1]


def check_results(res_r, res_b, cache_r, cache_b):
    assert res_r[0] == res_b[0]
    assert list(res_r[1].keys()) == list(res_b[1].keys())
    assert list(cache_r.keys()) == list(cache_b.keys())
    for key in cache_r:
        same(cache_r[key], cache_b[key], "variantCache[%s..]" % key[:12])


def rc(s):
    return s.translate(str.maketrans("ACGTN", "TGCAN"))[::-1]


def fanc_reads(n=None):
    import pe_case
    lines = pe_case.fanc_fastq_text().split("\n")
    reads = [lines[k + 1] for k in range(0, len(lines) - 3, 4)]
    return reads[:n] if n else reads


def write_fastq(path, reads, ends="\n", gz=False):
    text = "".join("@r%d%s%s%s+%s%s%s" % (k, ends, s, ends, ends, "I" * len(s), ends) for k, s in enumerate(reads))
    data = text.encode()
    if gz:
        with gzip.open(path, "wb") as fh:
            fh.write(data)
    else:
        with open(path, "wb") as fh:
            fh.write(data)
    return path


def edited_reads(amp, include_idxs, seed=11, n_random=6):
    """FANC reads plus: reverse complements, reads that align nowhere, insertions right at both window edges, a deletion
    reaching into the window, substitutions inside it"""
    rnd = np.random.default_rng(seed)
    reads = fanc_reads(200)
    reads += [rc(s) for s in reads[:40]]
    reads += ["".join(rnd.choice(list("ACGT"), size=120)) for _ in range(n_random)]
    lo, hi = int(min(include_idxs)), int(max(include_idxs))
    for p in (lo - 1, lo, hi, hi + 1):
        for ins in ("A", "GT", "TTCAG"):
            reads.append(amp[:p + 1] + ins + amp[p + 1:])
    reads.append(amp[:lo - 3] + amp[lo + 2:])
    reads.append(amp[:lo] + ("A" if amp[lo] != "A" else "C") + amp[lo + 1:])
    reads += reads[-10:]                                          # duplicates
    return reads


if __name__ == "__main__" and len(sys.argv) > 1 and sys.argv[1] == "capture":
    _capture_main()

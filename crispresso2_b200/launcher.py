"""CRISPResso-compatible launcher: the reference's own `CRISPResso` main() with its per-read hot path re-bound to the engine.

    python -m crispresso2_b200.launcher -r1 reads.fastq -a AMPLICON -g GUIDE ...      (every CRISPResso argument, unchanged)

also usable as CRISPRessoPooled / CRISPRessoBatch's `--crispresso_command "python -m crispresso2_b200.launcher"`.

What is re-bound (INTEGRATION.md section 2), nothing else of the reference changes:
  * CRISPRessoCORE.process_fastq (module global, resolved by name at CRISPRessoCORE.py:3750; also reached through
    process_fastq_write_out :2285 and process_single_fastq_write_bam_out :2373)   -> crispresso2_b200.core.process_fastq
  * CRISPRessoCORE.process_fastq_write_out / process_single_fastq_write_bam_out (--fastq_output / --bam_output, :3739-3743)
    -> crispresso2_b200.annotate (single process; under torchrun the reference's wrappers stay bound)
  * CRISPRessoCORE.process_bam (--bam_input, :3737-3738)   -> crispresso2_b200.bam.process_bam (single process; under torchrun
    the reference's function stays bound)
  * CRISPRessoCORE.process_paired_fastq (--crispresso_merge, :3744-3748)   -> crispresso2_b200.paired: the reference's loop with its
    global_align calls answered from one GPU batch over every distinct mate sequence
  * filterFastqs.filterFastqs (imported and called at CRISPRessoCORE.py:3716-3717)          -> crispresso2_b200.filter_fastqs.filterFastqs
  * CRISPRessoShared.get_dataframe_around_cut_asymmetrical (plots/data_prep.py:1537)        -> the native grouping of
    crispresso2_b200.alleles when the frame was built by AlleleTable.to_dataframe(), the reference's own function otherwise.
Under torchrun (WORLD_SIZE > 1) every rank runs the same command; process_fastq shards the unique reads over the ranks' GPUs
and merges the count block with one all-reduce (core.process_fastq_sharded); rank 0's output directory is the result.

Needs an importable CRISPResso2 (the user's installation).  The engine library is required: there is no CPU fallback.
"""
import functools
import os
import sys


def _import_reference():
    try:
        from CRISPResso2 import CRISPRessoCORE                      # the user's installed reference
        return CRISPRessoCORE
    except ImportError:
        # this repository's benchmark / test install of the unmodified reference (oracle/_ref/install), when built
        root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
        if root not in sys.path:
            sys.path.insert(0, root)
        try:
            from baseline import ref_shim
        except ImportError:
            raise ImportError("crispresso2_b200.launcher needs an installed CRISPResso2") from None
        return ref_shim.load_core()


def bind(CORE=None, engine=None, lib_path=None):
    """Re-binds the hot path of an imported reference `CRISPRessoCORE` module to the engine; returns the module."""
    from . import alleles, core, filter_fastqs
    CORE = CORE or _import_reference()
    world = int(os.environ.get("WORLD_SIZE", "1"))
    state = {"engine": engine}

    def get_engine():
        if state["engine"] is None:
            dev = int(os.environ.get("LOCAL_RANK", os.environ.get("C2B_DEVICE", "0")))
            state["engine"] = core.get_engine(dev, lib_path)
        return state["engine"]

    def process_fastq(fastq_filename, variantCache, ref_names, refs, args, files_to_remove, output_directory):
        loc = args.needleman_wunsch_aln_matrix_loc
        if not os.path.isabs(loc):
            loc = os.path.join(CORE._ROOT, loc)                     # CRISPRessoCORE.py:1811
        matrix = core.read_matrix(loc)
        fn = core.process_fastq
        if world > 1:
            import torch.distributed as dist
            if not dist.is_initialized():
                os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
                dist.init_process_group("nccl")
            fn = core.process_fastq_sharded
        return fn(fastq_filename, variantCache, ref_names, refs, args, files_to_remove, output_directory,
                  engine=get_engine(), aln_matrix=matrix)

    CORE.process_fastq = process_fastq
    if world == 1:
        # --fastq_output / --bam_output: annotations built on the GPU, records written natively (annotate.py).  Like the
        # reference's wrappers (:2285, :2373) they call the module-global process_fastq as it is bound when they run.
        from . import annotate

        def process_fastq_write_out(fastq_input, fastq_output, variantCache, ref_names, refs, args, files_to_remove, output_directory):
            return annotate.process_fastq_write_out(fastq_input, fastq_output, variantCache, ref_names, refs, args, files_to_remove,
                                                    output_directory, process_fastq=CORE.process_fastq)

        def process_single_fastq_write_bam_out(fastq_input, bam_output, bam_header, variantCache, ref_names, refs, args,
                                               files_to_remove, output_directory):
            return annotate.process_single_fastq_write_bam_out(fastq_input, bam_output, bam_header, variantCache, ref_names, refs,
                                                               args, files_to_remove, output_directory,
                                                               process_fastq=CORE.process_fastq)

        CORE.process_fastq_write_out = process_fastq_write_out
        CORE.process_single_fastq_write_bam_out = process_single_fastq_write_bam_out

        # --bam_input: the SAM front end, the batch and the annotations on the GPU, the pass-through SAM written natively (bam.py)
        from . import bam

        def process_bam(bam_filename, bam_chr_loc, output_bam, variantCache, ref_names, refs, args, files_to_remove, output_directory):
            loc = args.needleman_wunsch_aln_matrix_loc
            if not os.path.isabs(loc):
                loc = os.path.join(CORE._ROOT, loc)                 # CRISPRessoCORE.py:2018
            return bam.process_bam(bam_filename, bam_chr_loc, output_bam, variantCache, ref_names, refs, args, files_to_remove,
                                   output_directory, engine=get_engine(), aln_matrix=core.read_matrix(loc))

        CORE.process_bam = process_bam
    # paired-end merge mode (--crispresso_merge): the reference's own loop over one batch of GPU alignments (paired.py)
    from . import paired
    reference_paired = CORE.process_paired_fastq

    def process_paired_fastq(fastq1_filename, fastq2_filename, variantCache, ref_names, refs, args, files_to_remove, output_directory,
                             fastq_write_out_file=None):
        loc = args.needleman_wunsch_aln_matrix_loc
        if not os.path.isabs(loc):
            loc = os.path.join(CORE._ROOT, loc)
        return paired.process_paired_fastq(reference_paired, CORE.CRISPResso2Align, get_engine(), fastq1_filename, fastq2_filename,
                                           variantCache, ref_names, refs, args, files_to_remove, output_directory,
                                           fastq_write_out_file, aln_matrix=core.read_matrix(loc))

    CORE.process_paired_fastq = process_paired_fastq
    from CRISPResso2 import filterFastqs as FF
    FF.filterFastqs = functools.partial(filter_fastqs.filterFastqs, lib_path=lib_path)
    from CRISPResso2 import CRISPRessoShared as SH
    reference_around_cut = SH.get_dataframe_around_cut_asymmetrical

    def around_cut(df_alleles, cut_point, plot_left, plot_right, collapse_by_sequence=True):
        if getattr(df_alleles, "attrs", {}).get("c2b_allele_table") is not None:
            return alleles.get_dataframe_around_cut_asymmetrical(df_alleles, cut_point, plot_left, plot_right, collapse_by_sequence)
        return reference_around_cut(df_alleles, cut_point, plot_left, plot_right, collapse_by_sequence)

    SH.get_dataframe_around_cut_asymmetrical = around_cut
    return CORE


def main(argv=None):
    CORE = bind()
    if argv is not None:
        sys.argv = ["CRISPResso"] + list(argv)
    else:
        sys.argv[0] = "CRISPResso"
    return CORE.main()


if __name__ == "__main__":
    main()

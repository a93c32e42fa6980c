#!/usr/bin/env python
"""Runs the UNMODIFIED reference `CRISPResso` main() (oracle/_ref/install, loaded by baseline/ref_shim.py) either as-is or through
the shipped launcher's re-binding (crispresso2_b200/launcher.py), for the --bam_input comparisons of tests/test_bam_input.py and
tests/test_gpu_bam_input.py, which diff the two output folders byte for byte.

usage: bam_cli_runner.py <reference|b200> <engine-lib-or-'default'> <outdir> -- <CRISPResso argv>

TEST INFRASTRUCTURE: needs oracle/_ref/install.
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def main():
    mode, lib, outdir = sys.argv[1:4]
    argv = sys.argv[sys.argv.index("--") + 1:]
    from baseline import ref_shim
    CORE = ref_shim.load_core()
    if mode == "b200":
        from crispresso2_b200 import launcher
        from crispresso2_b200.engine import Engine
        lib_path = None if lib == "default" else lib
        launcher.bind(CORE, engine=Engine(lib_path=lib_path), lib_path=lib_path)
        assert CORE.process_bam.__module__ == "crispresso2_b200.launcher"
    os.makedirs(outdir, exist_ok=True)
    os.chdir(outdir)
    sys.argv = ["CRISPResso"] + argv + ["--suppress_plots", "--suppress_report", "-o", outdir]
    try:
        CORE.main()
    except SystemExit as e:
        if e.code not in (0, None):
            raise


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""tests/cli_dropin_runner.py with a count of the calls that reach the --coding_seq drop-in (crispresso2_b200.amino_acids),
written to <outdir>/_amino_acid_calls.json.  Same usage as cli_dropin_runner.py.

TEST INFRASTRUCTURE: needs oracle/_ref/install.
"""
import atexit
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))
sys.path.insert(0, HERE)


def main():
    from crispresso2_b200 import amino_acids
    calls = {"get_amino_acid_dataframe": 0}
    fn = amino_acids.get_amino_acid_dataframe

    def counted(*a, **kw):
        calls["get_amino_acid_dataframe"] += 1
        return fn(*a, **kw)

    amino_acids.get_amino_acid_dataframe = counted
    outdir = sys.argv[3]

    def dump():
        with open(os.path.join(outdir, "_amino_acid_calls.json"), "w") as fh:
            json.dump(calls, fh)

    atexit.register(dump)
    import cli_dropin_runner
    cli_dropin_runner.main()


if __name__ == "__main__":
    main()

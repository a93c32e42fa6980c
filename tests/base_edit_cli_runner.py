#!/usr/bin/env python
"""tests/cli_dropin_runner.py with a count of the calls that reach the --base_editor_output drop-ins
(crispresso2_b200.base_edit), written to <outdir>/_base_edit_calls.json.  Same usage as cli_dropin_runner.py.

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
    from crispresso2_b200 import base_edit
    calls = {"get_upset_plot_counts": 0, "get_base_edit_dataframe_around_cut": 0}
    for name in calls:
        fn = getattr(base_edit, name)

        def counted(*a, _fn=fn, _name=name, **kw):
            calls[_name] += 1
            return _fn(*a, **kw)

        setattr(base_edit, name, counted)
    outdir = sys.argv[3]

    def dump():
        with open(os.path.join(outdir, "_base_edit_calls.json"), "w") as fh:
            json.dump(calls, fh)

    atexit.register(dump)
    import cli_dropin_runner
    cli_dropin_runner.main()


if __name__ == "__main__":
    main()

"""pytest plugin, loaded with `-p amino_acid_standin` by tests/test_amino_acids.py and tests/test_gpu_amino_acids.py when they run
the reference's own amino-acid table unit tests: the reference package under oracle/_ref/install is imported and its
CRISPRessoShared.get_amino_acid_dataframe is replaced by crispresso2_b200.amino_acids' drop-in on the engine library named by
C2B_AMINO_LIB ('default': the sm_90a build)."""
import functools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

_F = {"calls": 0}


def pytest_configure(config):
    from baseline import ref_shim
    ref_shim.load_core()
    from CRISPResso2 import CRISPRessoShared
    from crispresso2_b200 import amino_acids
    from crispresso2_b200.engine import Engine
    lib = os.environ.get("C2B_AMINO_LIB", "default")
    fn = functools.partial(amino_acids.get_amino_acid_dataframe, engine=Engine(lib_path=None if lib == "default" else lib))

    def counted(*a, **kw):
        _F["calls"] += 1
        return fn(*a, **kw)

    CRISPRessoShared.get_amino_acid_dataframe = counted


def pytest_sessionfinish(session, exitstatus):
    assert _F["calls"] > 0, _F

"""pytest plugin, loaded with `-p base_edit_standin` by tests/test_base_edit.py and tests/test_gpu_base_edit.py when they run the
reference's own base-editing unit tests: the reference package under oracle/_ref/install is imported, and its
plots.data_prep.get_upset_plot_counts, CRISPRessoCORE.get_upset_plot_counts and CRISPRessoShared.get_base_edit_dataframe_around_cut
are replaced by crispresso2_b200.base_edit's drop-ins on the engine library named by C2B_BASE_EDIT_LIB ('default': the sm_90a
build).  The test modules import the functions by name, so their module globals are re-bound as they are collected."""
import functools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

_F = {}


def pytest_configure(config):
    from baseline import ref_shim
    CORE = ref_shim.load_core()
    from CRISPResso2 import CRISPRessoShared
    from CRISPResso2.plots import data_prep
    from crispresso2_b200 import base_edit
    from crispresso2_b200.engine import Engine
    lib = os.environ.get("C2B_BASE_EDIT_LIB", "default")
    eng = Engine(lib_path=None if lib == "default" else lib)
    _F["get_upset_plot_counts"] = functools.partial(base_edit.get_upset_plot_counts, engine=eng)
    _F["get_base_edit_dataframe_around_cut"] = functools.partial(base_edit.get_base_edit_dataframe_around_cut, engine=eng)
    _F["calls"] = {"upset": 0, "quilt": 0}

    def upset(*a, **kw):
        _F["calls"]["upset"] += 1
        return _F["get_upset_plot_counts"](*a, **kw)

    def quilt(*a, **kw):
        _F["calls"]["quilt"] += 1
        return _F["get_base_edit_dataframe_around_cut"](*a, **kw)

    data_prep.get_upset_plot_counts = upset
    CORE.get_upset_plot_counts = upset
    CRISPRessoShared.get_base_edit_dataframe_around_cut = quilt
    _F["upset"], _F["quilt"] = upset, quilt


def pytest_collection_modifyitems(session, config, items):
    for item in items:                                         # `from ...data_prep import get_upset_plot_counts` in the test module
        mod = getattr(item, "module", None)
        if mod is not None and hasattr(mod, "get_upset_plot_counts"):
            mod.get_upset_plot_counts = _F["upset"]


def pytest_sessionfinish(session, exitstatus):
    assert _F["calls"]["upset"] > 0 and _F["calls"]["quilt"] > 0, _F["calls"]

"""pytest plugin, loaded with `-p vcf_standin` by tests/test_vcf.py and tests/test_gpu_vcf.py when they run the reference's own
tests/unit_tests/test_writers/test_vcf/*.py: the reference package under oracle/_ref/install is imported, and its
CRISPResso2.writers.vcf.build_edit_counts is replaced by crispresso2_b200.vcf.build_edit_counts on the engine library named by
C2B_VCF_LIB ('default': the sm_90a build)."""
import functools
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    from baseline import ref_shim
    ref_shim.load_core()
    import CRISPResso2.writers.vcf as V
    from crispresso2_b200 import vcf
    from crispresso2_b200.engine import Engine
    lib = os.environ.get("C2B_VCF_LIB", "default")
    V.build_edit_counts = functools.partial(vcf.build_edit_counts, engine=Engine(lib_path=None if lib == "default" else lib))
    V.build_edit_counts.c2b_standin = True


def pytest_sessionfinish(session, exitstatus):
    import CRISPResso2.writers.vcf as V
    assert getattr(V.build_edit_counts, "c2b_standin", False)

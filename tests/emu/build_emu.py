"""Builds the CPU warp-emulator variant of the engine (TEST INFRASTRUCTURE, never loaded by the product)."""
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
SO = os.path.join(HERE, "libc2b200_emu.so")
SRC = [os.path.join(ROOT, "crispresso2_b200", "csrc", f) for f in ("c2b_engine.cu", "c2b_core.cuh", "c2b_fastq.cpp", "c2b_split.cuh", "c2b_alleles.cpp", "c2b_fastq_int.h", "c2b_paired.cpp",
                                                                     "c2b_annotate.cuh")] + \
      [os.path.join(HERE, "warp_emu.h"), os.path.join(ROOT, "include", "c2b200.h")]


def build():
    if os.path.exists(SO) and all(os.path.getmtime(SO) >= os.path.getmtime(s) for s in SRC):
        return SO
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-DC2B_EMU", "-x", "c++", "-shared", "-fPIC",
                           "-I" + os.path.join(ROOT, "include"), "-I" + HERE,
                           "-I" + os.path.join(ROOT, "crispresso2_b200", "csrc"), "-o", SO, SRC[0], SRC[2], SRC[4], SRC[6], "-lz", "-lpthread"])
    return SO

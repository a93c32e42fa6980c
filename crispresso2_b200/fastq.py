"""Native FASTQ ingest + de-duplication (c2b_fastq_dedup of include/c2b200.h) behind the variantCache semantics of
the reference's process_fastq loop (CRISPRessoCORE.py:1820-1849): unique sequences in first-seen order with their
multiplicities.  The packed arrays go straight to Engine.align_packed; Python strings are only made for the keys of
variantCache."""
import ctypes as C

import numpy as np

from . import _lib


class FastqError(RuntimeError):
    pass


class Dedup:
    """uniques: list[str] (first-seen order) | counts: int32[n_unique] | buf/off: packed bytes + int64 offsets |
    n_reads: records in the file | first_index: record index of each unique's first occurrence"""

    def __init__(self, buf, off, counts, first_index, n_reads):
        self.buf, self.off, self.counts, self.first_index, self.n_reads = buf, off, counts, first_index, n_reads
        self._uniques = None

    @property
    def uniques(self):
        if self._uniques is None:
            raw = self.buf.tobytes()
            o = self.off
            try:
                text = raw.decode("ascii")
                self._uniques = [text[o[k]:o[k + 1]] for k in range(len(o) - 1)]
            except UnicodeDecodeError:              # text-mode reading decodes UTF-8; keep the reference's key strings
                self._uniques = [raw[o[k]:o[k + 1]].decode("utf-8", errors="surrogateescape") for k in range(len(o) - 1)]
        return self._uniques


class _Handle:
    """Owns a c2b_fastq result: the arrays handed out are views of its memory (no copy of the packed reads) and keep it alive."""

    def __init__(self, L, h):
        self.L, self.h = L, h

    def __del__(self):
        h, self.h = self.h, None
        if h:
            self.L.c2b_fastq_free(h)

    def view(self, addr, nbytes, dtype):
        if not nbytes:
            return np.zeros(0, dtype=dtype)
        raw = (C.c_uint8 * nbytes).from_address(addr)
        raw._owner = self                                  # ndarray -> ctypes array -> this handle
        return np.frombuffer(raw, dtype=dtype)


def _collect(L, h):
    own = _Handle(L, h)
    nu, nr = int(L.c2b_fastq_n_unique(h)), int(L.c2b_fastq_n_reads(h))
    off = own.view(L.c2b_fastq_offsets(h), (nu + 1) * 8, np.int64)
    if not len(off):
        off = np.zeros(1, dtype=np.int64)
    tot = int(off[-1])
    buf = own.view(L.c2b_fastq_seqs(h), tot, np.uint8)
    counts = own.view(L.c2b_fastq_counts(h), nu * 4, np.int32)
    first = own.view(L.c2b_fastq_first_index(h), nu * 8, np.int64)
    return Dedup(buf, off, counts, first, nr)


GPU_INGEST_MAX_PLAIN = 8 << 30        # the text and its tables (about 3x the file) stay far below one GPU's HBM
GPU_INGEST_MAX_GZ = 1 << 30


def gpu_ingest_device(path, engine_device=None, lib_path=None):
    """Which front end process_fastq uses for `path`: a device index (c2b_fastq_dedup_gpu) or None (c2b_fastq_dedup on the
    host threads).  C2B_GPU_INGEST=1 forces the GPU, =0 the host; unset: the GPU when the library has the device front end
    (not the emulator test build) and the file is small enough to sit in HBM whole."""
    import os
    try:
        size = os.path.getsize(path)
    except OSError:
        size = None
    return _ingest_rule(size, str(path).endswith(".gz"), engine_device, lib_path)


def _ingest_rule(size, gz, engine_device, lib_path):
    """the rule of gpu_ingest_device for `size` bytes of input (None: unknown size -> the host threads unless forced)"""
    import os
    dev = 0 if engine_device is None else int(engine_device)
    env = os.environ.get("C2B_GPU_INGEST", "")
    if env == "0":
        return None
    if env not in ("", "0"):
        return dev
    if not _lib.load(lib_path).c2b_fastq_gpu_available():
        return None
    if size is None:
        return None
    return dev if size <= (GPU_INGEST_MAX_GZ if gz else GPU_INGEST_MAX_PLAIN) else None


def dedup_for_process_fastq(path, engine_device, lib_path=None):
    """The front end process_fastq uses: the GPU one when gpu_ingest_device() picks it (by build and file size), else the host
    threads.  A failure of the chosen one raises -- nothing is retried on the other; C2B_GPU_INGEST=0 / 1 forces either."""
    dev = gpu_ingest_device(path, engine_device, lib_path)
    try:
        return dedup_file(path, lib_path=lib_path, device=dev)
    except FastqError as ex:
        if dev is not None:
            raise FastqError("%s (GPU FASTQ front end; C2B_GPU_INGEST=0 selects the host threads)" % ex) from None
        raise


def dedup_file(path, n_threads=0, lib_path=None, device=None):
    """device=None: the host front end (c2b_fastq_dedup, n_threads workers); device=k: parse + de-duplicate on GPU k
    (c2b_fastq_dedup_gpu) -- same result object either way."""
    L = _lib.load(lib_path)
    h = C.c_void_p()
    if device is not None:
        rc = L.c2b_fastq_dedup_gpu(str(path).encode(), int(device), C.byref(h))
        name = "c2b_fastq_dedup_gpu"
    else:
        rc = L.c2b_fastq_dedup(str(path).encode(), int(n_threads), C.byref(h))
        name = "c2b_fastq_dedup"
    if rc != 0:
        raise FastqError("%s failed (%d): %s" % (name, rc, L.c2b_fastq_last_error().decode()))
    return _collect(L, h)


def dedup_bytes(data, n_threads=0, lib_path=None, device=None):
    L = _lib.load(lib_path)
    h = C.c_void_p()
    arr = np.frombuffer(data, dtype=np.uint8)
    ptr = arr.ctypes.data if len(arr) else None
    if device is not None:
        rc = L.c2b_fastq_dedup_gpu_buffer(ptr, len(arr), int(device), C.byref(h))
    else:
        rc = L.c2b_fastq_dedup_buffer(ptr, len(arr), int(n_threads), C.byref(h))
    if rc != 0:
        raise FastqError("c2b_fastq_dedup%s_buffer failed (%d): %s" % ("_gpu" if device is not None else "", rc, L.c2b_fastq_last_error().decode()))
    return _collect(L, h)


def dedup_sam(data, n_threads=0, lib_path=None, device=None):
    """Pass 1 of process_bam over SAM text (bytes): one record per line, its read is line.rstrip().split("\t")[9]; same result
    object as dedup_file.  device=None: host threads (c2b_sam_dedup_buffer); device=k: on GPU k (c2b_sam_dedup_gpu_buffer).
    A line with fewer than 10 fields raises IndexError, as the reference's loop does; a non-ASCII byte raises FastqError."""
    L = _lib.load(lib_path)
    h = C.c_void_p()
    arr = np.frombuffer(data, dtype=np.uint8)
    ptr = arr.ctypes.data if len(arr) else None
    if device is not None:
        rc = L.c2b_sam_dedup_gpu_buffer(ptr, len(arr), int(device), C.byref(h))
        name = "c2b_sam_dedup_gpu_buffer"
    else:
        rc = L.c2b_sam_dedup_buffer(ptr, len(arr), int(n_threads), C.byref(h))
        name = "c2b_sam_dedup_buffer"
    if rc == _lib.E_LIMIT:
        raise IndexError("list index out of range: %s" % L.c2b_fastq_last_error().decode())
    if rc != 0:
        raise FastqError("%s failed (%d): %s" % (name, rc, L.c2b_fastq_last_error().decode()))
    return _collect(L, h)


def dedup_for_process_bam(data, engine_device, lib_path=None):
    """The front end process_bam uses for its pass-1 text: the GPU one by the rule of dedup_for_process_fastq (build and size;
    C2B_GPU_INGEST=0 / 1 forces either), else the host threads.  A failure of the chosen one raises."""
    dev = _ingest_rule(len(data), False, engine_device, lib_path)
    try:
        return dedup_sam(data, lib_path=lib_path, device=dev)
    except FastqError as ex:
        if dev is not None:
            raise FastqError("%s (GPU SAM front end; C2B_GPU_INGEST=0 selects the host threads)" % ex) from None
        raise

"""Lazy unique-read table behind the reference's variantCache contract.

The reference's process_fastq leaves one dict per unique read in variantCache (CRISPRessoCORE.py:709-798: count, aln_scores,
ref_aln_details, aln_ref_names, class_name, best_match_name, variant_<ref> payloads with ~30 list fields each).  Building
those eagerly costs ~35 us of Python per unique read -- three orders of magnitude more than aligning it.  Here the batch's
results stay in the engine's compact arrays (`BatchSource`) and every cache entry is a `LazyVariant`: a genuine dict
(subclass) that holds only 'count' until something reads another key, at which point it fills itself with exactly the
dict the reference would have built (`core._variant_from`) and behaves as a plain dict from then on.

Contract notes (SURVEY.md section 7, "Payload shape is part of the contract"): after materialisation every value is a
genuine Python list / tuple / int / str / np.array of 1-char str, so `row['ref_positions'].index(...)`, `str()` of lists,
the JSON encoder and VCF iteration see what they see with the reference.  Subscript access (`v[key]`, the only access the
reference's own consumers use) goes through dict's C fast path plus `__missing__` on the first miss; the rarer mapping
methods are overridden to materialise first.
"""
import numpy as np

try:
    from . import _c2b_pyext as _ext
except ImportError:                                    # the helper is optional glue (pure-Python equivalents below)
    _ext = None


class LazyVariant(dict):
    __slots__ = ("_k",)
    _src = None                                        # per-batch subclass attribute: the BatchSource

    # no Python-level __init__: instances are created half a million at a time (c2b_pyext.fill_cache); `_k` is the read's
    # index k in the batch until the entry is materialised, -2 - k afterwards (-1: unset)

    # -- materialisation ---------------------------------------------------------------------------------------
    def _fill(self):
        k = getattr(self, "_k", -1)
        if k >= 0:
            self._k = -2 - k
            src = type(self)._src
            full = src.variant(k)
            full["count"] = dict.__getitem__(self, "count") if dict.__contains__(self, "count") else int(src.counts[k])
            dict.update(self, full)
            src.n_filled += 1
            for key, value_of in src.extra_keys:       # keys the annotated-output writers set (annotate.py): last, as there
                v = value_of(k)
                if v is not None:
                    dict.__setitem__(self, key, v)

    def __missing__(self, key):
        k = getattr(self, "_k", -1)
        if k < 0:
            raise KeyError(key)
        if key == "count":                             # the dedup multiplicity: answered from the batch's count array
            c = int(type(self)._src.counts[k])
            dict.__setitem__(self, "count", c)
            return c
        self._fill()
        return dict.__getitem__(self, key)

    def __setitem__(self, key, value):
        if key != "count":
            self._fill()
        dict.__setitem__(self, key, value)

    def __delitem__(self, key):
        self._fill()
        dict.__delitem__(self, key)

    def __contains__(self, key):
        self._fill()
        return dict.__contains__(self, key)

    def __iter__(self):
        self._fill()
        return dict.__iter__(self)

    def __len__(self):
        self._fill()
        return dict.__len__(self)

    def __eq__(self, other):
        self._fill()
        if isinstance(other, LazyVariant):
            other._fill()
        return dict.__eq__(self, other)

    def __ne__(self, other):
        return not self.__eq__(other)

    __hash__ = None

    def __repr__(self):
        self._fill()
        return dict.__repr__(self)

    def __reduce__(self):                              # pickles / copies as the plain dict it stands for
        self._fill()
        return (dict, (dict(self),))

    def __copy__(self):
        self._fill()
        return dict(self)

    def __deepcopy__(self, memo):
        import copy
        self._fill()
        return copy.deepcopy(dict(self), memo)

    def get(self, key, default=None):
        self._fill()
        return dict.get(self, key, default)

    def keys(self):
        self._fill()
        return dict.keys(self)

    def values(self):
        self._fill()
        return dict.values(self)

    def items(self):
        self._fill()
        return dict.items(self)

    def copy(self):
        self._fill()
        return dict(self)

    def pop(self, *a):
        self._fill()
        return dict.pop(self, *a)

    def popitem(self):
        self._fill()
        return dict.popitem(self)

    def setdefault(self, key, default=None):
        self._fill()
        return dict.setdefault(self, key, default)

    def update(self, *a, **kw):
        self._fill()
        dict.update(self, *a, **kw)

    def __or__(self, other):
        self._fill()
        return dict(self) | other

    def __ror__(self, other):
        self._fill()
        return other | dict(self)


class BatchSource:
    """One batch's results + what is needed to spell any read's variant dict: the engine's compact outputs (BatchResult),
    the read strings (keys), reference names.  `fix` maps a read index to (BatchResult, index) of a re-run with complete
    edit lists (reads whose list overflowed the batch's edit cap).  `parts` (multi-GPU): [(first read index, BatchResult,
    fix)] per rank, contiguous shards in read order."""

    def __init__(self, res, keys, ref_names, refs, counts, ref_id=None, fix=None, parts=None):
        self.keys, self.ref_names, self.refs, self.ref_id = keys, list(ref_names), refs, ref_id
        self.counts = counts                               # dedup multiplicity per read (variant['count'])
        self.parts = parts if parts is not None else [(0, res, fix or {})]
        self.starts = [p[0] for p in self.parts]
        self.n_filled = 0                                  # entries materialised so far
        self.extra_keys = []                               # [(key, value_of(k) -> value or None)], see LazyVariant._fill

    def variant(self, k):
        import bisect
        from . import core
        lo, res, fix = self.parts[bisect.bisect_right(self.starts, k) - 1]
        rr, kk = fix.get(k - lo, (res, k - lo))
        names = self.ref_names if self.ref_id is None else [self.ref_names[int(self.ref_id[k])]]
        return core._variant_from(rr, kk, self.keys[k], names, self.refs)

    def lazy_class(self):
        return type("LazyVariant", (LazyVariant,), {"__slots__": (), "_src": self})


def make_keys(buf, off):
    """packed unique reads -> list of str (what the reference's text-mode reader would have produced)"""
    buf = np.ascontiguousarray(buf, dtype=np.uint8)
    off = np.ascontiguousarray(off, dtype=np.int64)
    if _ext is not None:
        return _ext.make_keys(buf, off)
    raw = buf.tobytes()
    try:
        text = raw.decode("ascii")
        o = off.tolist()
        return [text[o[k]:o[k + 1]] for k in range(len(o) - 1)]
    except UnicodeDecodeError:
        return [raw[off[k]:off[k + 1]].decode("utf-8", errors="surrogateescape") for k in range(len(off) - 1)]


def fill_cache(cache, keys, sel, counts, cls, value=1):
    """cache[keys[k]] = cls() with ._k = k, for every k with sel[k] == value, in k order (counts: see LazyVariant.__missing__)"""
    sel = np.ascontiguousarray(sel, dtype=np.uint8)
    counts = np.ascontiguousarray(counts, dtype=np.int32)
    if _ext is not None:
        return _ext.fill_cache(cache, keys, sel, counts, cls, int(value))
    n = 0
    for k in np.nonzero(sel == value)[0].tolist():
        o = cls()
        o._k = k
        cache[keys[k]] = o
        n += 1
    return n

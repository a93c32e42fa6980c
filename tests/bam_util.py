"""BAM / SAM helpers of the --bam_input tests (tests/test_bam_input.py, tests/test_gpu_bam_input.py) and tools/bam_bench.py.

  * write_bam(path, header, refs, records): a BGZF-compressed BAM (zlib only) of synthetic records;
  * read_bam(path) -> (header text, [(name, length)], [SAM line of every record, flag, contig, 0-based start, end]);
  * fake_samtools(dirpath): a `samtools` stand-in on PATH -- `view` with -H, -c, -F / -f (decimal, 0x hex, 0 octal) and a
    region ("chr", "chr:beg", "chr:beg-end"; a linear scan, overlap by the record's CIGAR span, unmapped records never match),
    SAM text of the aux types A c C s S i I f Z H B; `sort` (copy) and `index` (an empty .bai).  Input may also be a ".sam" text
    file, filtered the same way (lines kept byte for byte), for texts no BAM can hold.

The reference and the drop-in both read what the stand-in prints, so a comparison of the two measures the drop-in only.

TEST INFRASTRUCTURE.
"""
import gzip
import os
import shutil
import struct
import sys
import zlib

HERE = os.path.dirname(os.path.abspath(__file__))

SEQ_CODES = "=ACMGRSVTWYHKDBN"
CIGAR_OPS = "MIDNSHP=X"
REF_CONSUMING = set("MDN=X")


# ------------------------------------------------------------------------------------------------ BGZF
def _bgzf_block(data):
    c = zlib.compressobj(6, zlib.DEFLATED, -15)
    body = c.compress(data) + c.flush()
    bsize = 18 + len(body) + 8 - 1
    head = b"\x1f\x8b\x08\x04\x00\x00\x00\x00\x00\xff\x06\x00BC\x02\x00" + struct.pack("<H", bsize)
    return head + body + struct.pack("<II", zlib.crc32(data) & 0xffffffff, len(data))


BGZF_EOF = bytes.fromhex("1f8b08040000000000ff0600424302001b0003000000000000000000")


def bgzf(data):
    out = [_bgzf_block(data[i:i + 65280]) for i in range(0, len(data), 65280)]
    return b"".join(out) + BGZF_EOF


# ------------------------------------------------------------------------------------------------ BAM writer
def _reg2bin(beg, end):
    end -= 1
    for shift, off in ((14, 4681), (17, 585), (20, 73), (23, 9), (26, 1)):
        if beg >> shift == end >> shift:
            return off + (beg >> shift)
    return 0


def _cigar(cigar):
    if cigar in ("*", ""):
        return []
    ops, num = [], ""
    for ch in cigar:
        if ch.isdigit():
            num += ch
        else:
            ops.append((int(num), ch))
            num = ""
    return ops


def _aux_bytes(tags):
    out = b""
    for tag, typ, val in tags:
        out += tag.encode()
        if typ == "i":                                          # stored as C when it fits, as samtools does; prints back as 'i'
            out += b"C" + struct.pack("<B", int(val)) if 0 <= int(val) <= 255 else b"i" + struct.pack("<i", int(val))
            continue
        out += typ.encode()
        if typ == "A":
            out += val.encode()
        elif typ == "f":
            out += struct.pack("<f", float(val))
        elif typ in "ZH":
            out += val.encode() + b"\0"
        else:
            raise ValueError(typ)
    return out


def write_bam(path, header, refs, records):
    """records: dicts with qname, flag, rname ('*' or a name of refs), pos (1-based, 0 = none), mapq, cigar, seq ('*' or
    bases), qual ('*' or Phred+33), tags [(tag, type, value)] of types A i f Z H"""
    names = [r[0] for r in refs]
    raw = b"BAM\1" + struct.pack("<i", len(header)) + header.encode() + struct.pack("<i", len(refs))
    for name, ln in refs:
        raw += struct.pack("<i", len(name) + 1) + name.encode() + b"\0" + struct.pack("<i", ln)
    for r in records:
        ref_id = names.index(r["rname"]) if r["rname"] != "*" else -1
        pos0 = int(r["pos"]) - 1
        cig = _cigar(r.get("cigar", "*"))
        span = sum(n for n, op in cig if op in REF_CONSUMING) or 1
        seq = "" if r["seq"] == "*" else r["seq"]
        qual = r.get("qual", "*")
        qn = r["qname"].encode() + b"\0"
        body = struct.pack("<iiBBHHHiiii", ref_id, pos0, len(qn), int(r.get("mapq", 255)), _reg2bin(max(pos0, 0), max(pos0, 0) + span),
                           len(cig), int(r["flag"]), len(seq), -1, -1, 0)
        body += qn + b"".join(struct.pack("<I", n << 4 | CIGAR_OPS.index(op)) for n, op in cig)
        codes = [SEQ_CODES.index(c) for c in seq.upper()]
        if len(codes) % 2:
            codes.append(0)
        body += bytes(codes[i] << 4 | codes[i + 1] for i in range(0, len(codes), 2))
        body += b"\xff" * len(seq) if qual == "*" else bytes(ord(c) - 33 for c in qual)
        body += _aux_bytes(r.get("tags", []))
        raw += struct.pack("<i", len(body)) + body
    with open(path, "wb") as fh:
        fh.write(bgzf(raw))
    return path


# ------------------------------------------------------------------------------------------------ BAM reader
def _fmt_float(x):
    return "%g" % x


def _aux_text(b, i, end):
    out = []
    while i < end:
        tag, typ = b[i:i + 2].decode(), chr(b[i + 2])
        i += 3
        if typ == "A":
            out.append("%s:A:%s" % (tag, chr(b[i])))
            i += 1
        elif typ in "cCsSiI":
            fmt = {"c": "<b", "C": "<B", "s": "<h", "S": "<H", "i": "<i", "I": "<I"}[typ]
            v = struct.unpack_from(fmt, b, i)[0]
            i += struct.calcsize(fmt)
            out.append("%s:i:%d" % (tag, v))
        elif typ == "f":
            out.append("%s:f:%s" % (tag, _fmt_float(struct.unpack_from("<f", b, i)[0])))
            i += 4
        elif typ in "ZH":
            j = b.index(b"\0", i)
            out.append("%s:%s:%s" % (tag, typ, b[i:j].decode()))
            i = j + 1
        elif typ == "B":
            sub = chr(b[i])
            n = struct.unpack_from("<i", b, i + 1)[0]
            fmt = {"c": "b", "C": "B", "s": "h", "S": "H", "i": "i", "I": "I", "f": "f"}[sub]
            vals = struct.unpack_from("<%d%s" % (n, fmt), b, i + 5)
            i += 5 + n * struct.calcsize(fmt)
            out.append("%s:B:%s" % (tag, sub) + "".join("," + (_fmt_float(v) if sub == "f" else str(v)) for v in vals))
        else:
            raise ValueError("aux type %r" % typ)
    return out


def read_bam(path):
    b = gzip.decompress(open(path, "rb").read())
    assert b[:4] == b"BAM\1"
    lt = struct.unpack_from("<i", b, 4)[0]
    header = b[8:8 + lt].split(b"\0")[0].decode()
    i = 8 + lt
    nref = struct.unpack_from("<i", b, i)[0]
    i += 4
    refs = []
    for _ in range(nref):
        ln = struct.unpack_from("<i", b, i)[0]
        name = b[i + 4:i + 4 + ln - 1].decode()
        refs.append((name, struct.unpack_from("<i", b, i + 4 + ln)[0]))
        i += 8 + ln
    recs = []
    while i < len(b):
        bs = struct.unpack_from("<i", b, i)[0]
        s, e = i + 4, i + 4 + bs
        ref_id, pos, lqn, mapq, _bin, ncig, flag, lseq, nref_id, npos, tlen = struct.unpack_from("<iiBBHHHiiii", b, s)
        p = s + 32
        qname = b[p:p + lqn - 1].decode()
        p += lqn
        cig = [struct.unpack_from("<I", b, p + 4 * k)[0] for k in range(ncig)]
        p += 4 * ncig
        cigar = "".join("%d%s" % (c >> 4, CIGAR_OPS[c & 15]) for c in cig) or "*"
        seq = "".join(SEQ_CODES[(b[p + k // 2] >> (4 * (1 - k % 2))) & 15] for k in range(lseq)) or "*"
        p += (lseq + 1) // 2
        q = b[p:p + lseq]
        qual = "*" if not lseq or q[0] == 0xff else "".join(chr(x + 33) for x in q)
        p += lseq
        rname = refs[ref_id][0] if ref_id >= 0 else "*"
        rnext = "*" if nref_id < 0 else ("=" if nref_id == ref_id else refs[nref_id][0])
        fields = [qname, str(flag), rname, str(pos + 1), str(mapq), cigar, rnext, str(npos + 1), str(tlen), seq, qual]
        fields += _aux_text(b, p, e)
        span = sum((c >> 4) for c in cig if CIGAR_OPS[c & 15] in REF_CONSUMING) or 1
        recs.append(("\t".join(fields) + "\n", flag, rname, pos, pos + span))
        i = e
    return header, refs, recs


def read_sam(path):
    """a SAM text file as read_bam's result; lines kept as they are (any line ending, any content)"""
    data = open(path, "rb").read().decode("latin-1")
    lines = data.splitlines(keepends=True)
    header = "".join(x for x in lines if x.startswith("@"))
    recs = []
    for x in lines:
        if x.startswith("@"):
            continue
        f = x.rstrip("\r\n").split("\t")
        try:
            flag, pos0 = int(f[1]), int(f[3]) - 1
            span = sum(n for n, op in _cigar(f[5]) if op in REF_CONSUMING) or 1
            recs.append((x, flag, f[2], pos0, pos0 + span))
        except (IndexError, ValueError):
            recs.append((x, 0, "*", -1, -1))                     # kept by -F, matches no region
    return header, [], recs


def parse_flags(s):
    if s.lower().startswith("0x"):
        return int(s, 16)
    if len(s) > 1 and s.startswith("0"):
        return int(s, 8)
    return int(s)


def _in_region(rec, region):
    _, flag, rname, beg, end = rec
    if flag & 4 or beg < 0:
        return False
    name, _, span = region.partition(":")
    if rname != name:
        return False
    if not span:
        return True
    lo, _, hi = span.replace(",", "").partition("-")
    lo = int(lo) - 1 if lo else 0
    hi = int(hi) if hi else 1 << 62
    return beg < hi and end > lo


def samtools_main(argv):
    out = sys.stdout.buffer
    if argv[:1] == ["sort"]:                                     # samtools sort IN -o OUT
        shutil.copyfile(argv[1], argv[argv.index("-o") + 1])
        return 0
    if argv[:1] == ["index"]:
        open(argv[1] + ".bai", "wb").close()
        return 0
    if argv[:1] != ["view"]:
        return 1
    args = argv[1:]
    header_only = count = False
    excl = req = 0
    rest = []
    k = 0
    while k < len(args):
        a = args[k]
        if a == "-H":
            header_only = True
        elif a == "-c":
            count = True
        elif a == "-F":
            excl = parse_flags(args[k + 1])
            k += 1
        elif a == "-f":
            req = parse_flags(args[k + 1])
            k += 1
        else:
            rest.append(a)
        k += 1
    path, regions = rest[0], rest[1:]
    header, _, recs = read_sam(path) if path.endswith(".sam") else read_bam(path)
    if header_only:
        out.write(header.encode("latin-1"))
        return 0
    sel = [r for r in recs if not (r[1] & excl) and (r[1] & req) == req and (not regions or any(_in_region(r, g) for g in regions))]
    if count:
        out.write(b"%d\n" % len(sel))
    else:
        out.write("".join(r[0] for r in sel).encode("latin-1"))
    return 0


def fake_samtools(dirpath):
    """the stand-in as `samtools` in dirpath -> a PATH value with dirpath first"""
    os.makedirs(dirpath, exist_ok=True)
    path = os.path.join(dirpath, "samtools")
    with open(path, "w") as fh:
        fh.write("#!%s\nimport sys\nsys.path.insert(0, %r)\nimport bam_util\nsys.exit(bam_util.samtools_main(sys.argv[1:]))\n"
                 % (sys.executable, HERE))
    os.chmod(path, 0o755)
    return str(dirpath) + os.pathsep + os.environ.get("PATH", "")


def sam_text_of(path, excl=0, region=None):
    """what `samtools view [-F excl] path [region]` prints, as bytes"""
    header, _, recs = read_sam(path) if path.endswith(".sam") else read_bam(path)
    sel = [r for r in recs if not (r[1] & excl) and (region is None or _in_region(r, region))]
    return "".join(r[0] for r in sel).encode("latin-1")


def pass1_restated(text):
    """the pass-1 loop of process_bam (CRISPRessoCORE.py:2047-2057) on bytes: {seq: count} in first-seen order, the number of
    lines; raises IndexError on a short line and UnicodeDecodeError on bytes that are not UTF-8"""
    import io
    cache, n = {}, 0
    for line in io.TextIOWrapper(io.BytesIO(text), encoding="utf-8"):
        seq = line.rstrip().split("\t")[9]
        cache[seq] = cache.get(seq, 0) + 1
        n += 1
    return cache, n

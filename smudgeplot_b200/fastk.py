"""FastK ``.ktab`` table files: host-side reader and writer (numpy only).

Layout as the reference reads it (``src/lib/libfastk.c:786-908`` of smudgeplot, Open_Kmer_Stream,
``:1230-1269`` Current_Entry; SURVEY.md Appendix A), all little-endian host ints:

* stub ``<dir>/<root>.ktab``: ``int32 kmer, nparts, minval, ibyte`` then
  ``int64 index[1 << (8*ibyte)]``; ``index[x]`` = number of entries whose first ``ibyte`` bytes
  (big-endian) are ``<= x`` (the END offset of bucket x).
* parts ``<dir>/.<root>.ktab.<p>``, p = 1..nparts: ``int32 kmer; int64 n`` then ``n`` records of
  ``pbyte = kbyte - ibyte + 2`` bytes: the ``kbyte - ibyte`` suffix bytes of the packed k-mer
  followed by an unaligned little-endian ``uint16`` count.

The reader hands the raw record payloads + stub index to the CUDA loader untouched (the
prefix re-attachment and SoA unpack are done on the GPU, see csrc/hm_kernels.cu); `unpack_host`
is only for tests.  The product's C executable has its own parser (host/fastk_table.c).
"""
from __future__ import annotations

import os
import struct
from dataclasses import dataclass, field

import numpy as np

PART_HEADER = 12  # int32 kmer + int64 n   (libfastk.c:860-861)


def split_name(name: str):
    """(dir, root) as PathTo / Root(name, ".ktab") give them (gene_core.c:64-114)."""
    d, base = os.path.split(name)
    if d == "":
        d = "."
    if len(base) > 5 and base.lower().endswith(".ktab"):
        base = base[:-5]
    return d, base


def stub_path(name: str) -> str:
    d, r = split_name(name)
    return os.path.join(d, r + ".ktab")


def part_path(name: str, p: int) -> str:
    d, r = split_name(name)
    return os.path.join(d, f".{r}.ktab.{p}")


@dataclass
class KtabFiles:
    """Parsed stub + raw part payloads of one FastK table (host memory)."""

    kmer: int
    nparts: int
    minval: int
    ibyte: int
    index: np.ndarray                      # int64[1 << 8*ibyte]
    part_nels: list = field(default_factory=list)
    records: list = field(default_factory=list)   # per part: uint8[n*pbyte] (payload, header stripped)
    name: str | None = None                # the table's files (read_ktab / write_ktab), None if built in memory

    @property
    def kbyte(self) -> int:
        return (self.kmer + 3) >> 2

    @property
    def hbyte(self) -> int:
        return self.kbyte - self.ibyte

    @property
    def pbyte(self) -> int:
        return self.kbyte - self.ibyte + 2

    @property
    def nels(self) -> int:
        return int(sum(self.part_nels))

    def all_records(self) -> np.ndarray:
        """All part payloads concatenated (uint8[nels*pbyte])."""
        if len(self.records) == 1:
            return self.records[0]
        if not self.records:
            return np.zeros(0, dtype=np.uint8)
        return np.concatenate(self.records)


def read_ktab(name: str, mmap: bool = False) -> KtabFiles:
    """Open a table the way Open_Kmer_Stream does; raises FileNotFoundError if the stub is absent
    (the reference returns NULL -> "Cannot open k-mer table", PloidyPlot.c:1350-1354)."""
    sp = stub_path(name)
    with open(sp, "rb") as f:
        kmer, nparts, minval, ibyte = struct.unpack("<4i", f.read(16))
        if ibyte not in (1, 2, 3):
            raise ValueError(f"{sp}: unsupported ibyte {ibyte}")
        ixlen = 1 << (8 * ibyte)
        index = np.fromfile(f, dtype="<i8", count=ixlen)
        if index.size != ixlen:
            raise ValueError(f"{sp}: truncated prefix index")
    kt = KtabFiles(kmer, nparts, minval, ibyte, index, name=name)
    for p in range(1, nparts + 1):
        pp = part_path(name, p)
        if not os.path.exists(pp):
            raise FileNotFoundError(f"Table part {pp} is missing ?")     # libfastk.c:851-854
        with open(pp, "rb") as f:
            pk, n = struct.unpack("<iq", f.read(PART_HEADER))
        if pk != kmer:
            raise ValueError(f"Table part {pp} does not have k-mer length matching stub ?")
        if mmap and n > 0:
            rec = np.memmap(pp, dtype=np.uint8, mode="r", offset=PART_HEADER, shape=(n * kt.pbyte,))
        else:
            rec = np.fromfile(pp, dtype=np.uint8, offset=PART_HEADER, count=n * kt.pbyte)
        if rec.size != n * kt.pbyte:
            raise ValueError(f"{pp}: truncated ({rec.size} of {n * kt.pbyte} payload bytes)")
        kt.part_nels.append(int(n))
        kt.records.append(rec)
    return kt


def unpack_host(kt: KtabFiles):
    """CPU unpack (tests only): -> (keys uint8[nels,kbyte] big-endian packed k-mers, cnt uint16[nels])."""
    n, kb, ib, hb = kt.nels, kt.kbyte, kt.ibyte, kt.hbyte
    rec = kt.all_records().reshape(n, kt.pbyte)
    keys = np.zeros((n, kb), dtype=np.uint8)
    # prefix of ordinal i = first bucket b with index[b] > i   (libfastk.c:1174-1175)
    pre = np.searchsorted(kt.index, np.arange(n, dtype=np.int64), side="right")
    for j in range(ib):
        keys[:, j] = (pre >> (8 * (ib - 1 - j))) & 0xFF
    keys[:, ib:] = rec[:, :hb]
    cnt = rec[:, hb].astype(np.uint16) | (rec[:, hb + 1].astype(np.uint16) << 8)
    return keys, cnt


def keys_u64_to_bytes(keys_u64: np.ndarray, kmer: int) -> np.ndarray:
    """left-aligned packed k-mers -> uint8[n,kbyte] big-endian.  uint64[n] for k<=32, or
    uint64[n,2] = (bases 0..31, bases 32..63) for 32 < k <= 64."""
    kb = (kmer + 3) >> 2
    a = np.ascontiguousarray(np.asarray(keys_u64, dtype=np.uint64))
    words = 1 if a.ndim == 1 else a.shape[1]
    be = np.ascontiguousarray(a.reshape(-1, words).astype(">u8")).view(np.uint8).reshape(-1, 8 * words)
    return np.ascontiguousarray(be[:, :kb])


def keys_bytes_to_u64(keys: np.ndarray) -> np.ndarray:
    """uint8[n,kbyte] big-endian -> left-aligned uint64[n] (kbyte<=8) or uint64[n,2] (kbyte<=16)."""
    n, kb = keys.shape
    words = 1 if kb <= 8 else 2
    buf = np.zeros((n, 8 * words), dtype=np.uint8)
    buf[:, :kb] = keys
    out = buf.view(">u8").reshape(n, words).astype(np.uint64)
    return out[:, 0] if words == 1 else out


def write_ktab(name: str, kmer: int, keys: np.ndarray, cnt: np.ndarray, ibyte: int = 3,
               nparts: int = 1, minval: int = 1, cut_on_buckets: bool = True) -> KtabFiles:
    """Write a FastK table.  `keys`: uint8[n,kbyte] big-endian packed k-mers in ascending order
    (or left-aligned uint64[n] for k<=32); `cnt`: uint16[n].  Parts are cut on prefix-bucket
    boundaries unless cut_on_buckets=False (SURVEY.md Appendix A discusses why that matters to
    the reference's on-disk bisection)."""
    if keys.dtype != np.uint8:
        keys = keys_u64_to_bytes(keys, kmer)
    n, kb = keys.shape
    assert kb == (kmer + 3) >> 2
    hb = kb - ibyte
    assert hb >= 0
    cnt = np.asarray(cnt).astype(np.uint16)
    pre = np.zeros(n, dtype=np.int64)
    for j in range(ibyte):
        pre = (pre << 8) | keys[:, j].astype(np.int64)
    ixlen = 1 << (8 * ibyte)
    index = np.cumsum(np.bincount(pre, minlength=ixlen)).astype("<i8")
    rec = np.empty((n, hb + 2), dtype=np.uint8)
    rec[:, :hb] = keys[:, ibyte:]
    rec[:, hb] = (cnt & 0xFF).astype(np.uint8)
    rec[:, hb + 1] = (cnt >> 8).astype(np.uint8)

    cuts = [0]
    for p in range(1, nparts):
        c = (n * p) // nparts
        if cut_on_buckets and n > 0:
            b = pre[min(c, n - 1)]
            c = int(index[b - 1]) if b > 0 else 0     # start of the bucket holding ordinal c
        cuts.append(max(c, cuts[-1]))
    cuts.append(n)

    d, r = split_name(name)
    os.makedirs(d, exist_ok=True)
    with open(stub_path(name), "wb") as f:
        f.write(struct.pack("<4i", kmer, nparts, minval, ibyte))
        index.tofile(f)
    kt = KtabFiles(kmer, nparts, minval, ibyte, index, name=name)
    for p in range(1, nparts + 1):
        lo, hi = cuts[p - 1], cuts[p]
        with open(part_path(name, p), "wb") as f:
            f.write(struct.pack("<iq", kmer, hi - lo))
            rec[lo:hi].tofile(f)
        kt.part_nels.append(hi - lo)
        kt.records.append(rec[lo:hi].reshape(-1))
    return kt


def same_table_files(a: str, a_parts: int, b: str) -> bool:
    """whether writing table `b` would write over a file of table `a` (a_parts parts): its stub or one of its
    parts is one of a's files (any spelling of the name, links included)"""
    mine = [stub_path(a)] + [part_path(a, p) for p in range(1, a_parts + 1)]
    mine = [os.stat(f) for f in mine if os.path.exists(f)]
    ids = {(st.st_dev, st.st_ino) for st in mine}
    theirs = [stub_path(b)] + [part_path(b, p) for p in range(1, max(a_parts, 1) + 1)]
    return any((os.stat(f).st_dev, os.stat(f).st_ino) in ids for f in theirs if os.path.exists(f))


def remove_ktab(name: str) -> None:
    """Delete stub + parts (what FastK's Fastrm does for a table)."""
    try:
        with open(stub_path(name), "rb") as f:
            _, nparts, _, _ = struct.unpack("<4i", f.read(16))
    except FileNotFoundError:
        return
    for p in range(1, nparts + 1):
        try:
            os.remove(part_path(name, p))
        except FileNotFoundError:
            pass
    os.remove(stub_path(name))

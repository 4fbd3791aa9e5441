"""Host-side mirror of the reference's `hetmers` task.

Reference interface (the only one this path has): ``smudgeplot hetmers -L <cutoff> -t <threads>
-o <prefix> [--verbose] [-tmp <dir>] <FastK_Table>`` builds ``["-o<o>", "-e<L>", "-T<t>", ("-v"),
("-P<tmp>" iff tmp != "."), infile]`` and spawns the ``hetmers`` binary
(smudgeplot's src/smudgeplot/cli.py:57-72, 348-361).  `hetmers_args` + `run_hetmers` reproduce
exactly that against OUR executable (smudgeplot_b200/bin/hetmers); `scan_table` / `Scan` are the
in-process route through the same C ABI (include/hetmers_b200.h layer B) for callers that already
hold the table in host memory.  Everything computes on the GPU; there is no fallback.
"""
from __future__ import annotations

import ctypes as C
import os
import re
import shlex
import subprocess
import sys

import numpy as np

from . import _lib
from .fastk import KtabFiles, read_ktab


def get_binary_path(name: str = "hetmers") -> str:
    """bundled binary first, then PATH -- the lookup order of cli.py:18-54"""
    import shutil
    bundled = os.path.join(os.path.dirname(_lib.BIN_PATH), name)
    if os.path.exists(bundled) and os.access(bundled, os.X_OK):
        return bundled
    found = shutil.which(name)
    if found:
        return found
    raise FileNotFoundError(f"Binary '{name}' not found (looked in {os.path.dirname(bundled)} and PATH); run `make`")


def hetmers_args(infile, o="smudgeplot", L=None, t=4, verbose=False, tmp="."):
    """argv tail exactly as cli.py:350-359 builds it (L is required there via argparse)."""
    if L is None:
        raise ValueError("-L (count threshold) is required, as in `smudgeplot hetmers`")
    args = [f"-o{o}", f"-e{L}", f"-T{t}"]
    if verbose:
        args.append("-v")
    if tmp != ".":
        args.append(f"-P{tmp}")
    args.append(str(infile))
    return args


def run_hetmers(infile, o="smudgeplot", L=None, t=4, verbose=False, tmp=".", gpus=None, stdin_text="n\n"):
    """Spawn the drop-in executable like run_binary (cli.py:57-72): raises CalledProcessError on a
    non-zero exit.  Returns the path of the .smu written."""
    cmd = [get_binary_path("hetmers")] + hetmers_args(infile, o, L, t, verbose, tmp)
    sys.stderr.write(f"Calling: {shlex.join(cmd)}\n")
    env = dict(os.environ)
    if gpus is not None:
        env["HETMERS_GPUS"] = str(gpus)
    subprocess.run(cmd, check=True, input=stdin_text, text=True, env=env)
    return f"{o}.smu"


def extract_args(infile, sma, o="kmerpairs", t=4, verbose=False, tmp="."):
    """argv tail of `smudgeplot extract` exactly as cli.py:368-378 builds it"""
    args = [f"-o{o}", f"-T{t}"]
    if verbose:
        args.append("-v")
    if tmp != ".":
        args.append(f"-P{tmp}")
    args.append(str(infile))
    s = str(sma)
    args.append(s[:-4] if s.endswith(".sma") else s)
    return args


def run_extract(infile, sma, o="kmerpairs", t=4, verbose=False, tmp=".", gpus=None, e=None):
    """Spawn our `extract_kmer_pairs` (same boundary as the reference's second binary,
    src/lib/PloidyList.c; cli.py:368-382).  Writes <o>.<a>A<b>B.txt per smudge of the .sma."""
    cmd = [get_binary_path("extract_kmer_pairs")] + extract_args(infile, sma, o, t, verbose, tmp)
    if e is not None:
        cmd.insert(1, f"-e{e}")
    sys.stderr.write(f"Calling: {shlex.join(cmd)}\n")
    env = dict(os.environ)
    if gpus is not None:
        env["HETMERS_GPUS"] = str(gpus)
    subprocess.run(cmd, check=True, env=env)


_WS = "[ \t\n\v\f\r]*"
_INT = _WS + "([+-]?[0-9]+)"
_SMA_LINE = re.compile(_INT + _INT + _WS + "[+-]?[0-9]+" + _INT + "A" + _INT)   # sscanf " %d %d %*d %dA%dB"


def _fgets_lines(data: bytes, size: int = 1000):
    """the pieces fgets(line, size, f) returns one by one: up to and including a newline, at most size - 1 bytes"""
    at = 0
    while at < len(data):
        nl = data.find(b"\n", at, at + size - 1)
        end = nl + 1 if nl >= 0 else min(at + size - 1, len(data))
        yield data[at:end]
        at = end


def read_sma(path):
    """<path>[.sma] as extract_kmer_pairs reads it (read_sma / smudge_label in host/hetmers_main.c): the suffix is
    optional and matched in any case, the header line is skipped, each further line is "covB covA freq <a>A<b>B"
    (sscanf's " %d %d %*d %dA%dB": leading blanks and trailing text are accepted).  Labels are numbered 1, 2, ... in
    order of first appearance; a later line for the same pixel wins.  -> (pixmap uint16[SMAX+1, FMAX+1]: pixel
    (covA+covB, covB) -> label, 0 = none; [(a, b), ...] of labels 1, 2, ...).  The executable's refusals raise
    ValueError with its message."""
    s = str(path)
    root = s[:-4] if len(s) > 4 and s[-4:].lower() == ".sma" else s
    try:
        with open(root + ".sma", "rb") as f:
            data = f.read()
    except OSError:
        raise ValueError(f"Could not open smudge file {root}.sma") from None
    pix = np.zeros((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.uint16)
    labels = []
    lines = _fgets_lines(data)
    next(lines, None)                                   # the header
    for raw in lines:
        line = raw.decode("latin-1")
        m = _SMA_LINE.match(line)
        if m is None:
            raise ValueError(f"Cannot parse line '{line}'")
        covb, cova, a, b = (_c_int(g) for g in m.groups())
        if a <= 0 or b <= 0 or a < b:
            raise ValueError(f"{a}A{b}B is not a valid smudge label")
        if covb < 0 or covb > _lib.FMAX or cova < covb or covb + cova > _lib.SMAX:
            raise ValueError(f"({covb},{cova}) is not a valid pixel coordinate")
        if (a, b) not in labels:
            labels.append((a, b))
        pix[covb + cova, covb] = labels.index((a, b)) + 1
    return pix, labels


def _c_int(text: str) -> int:
    """a %d conversion's value as a 32-bit int (glibc saturates what strtol cannot hold, then truncates to int)"""
    v = max(min(int(text), (1 << 63) - 1), -(1 << 63))
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v >= (1 << 31) else v


# ------------------------------------------------------------------ in-process (C ABI layer B) --

# one record of extract_kmer_pairs' list (hm_pair_rec), as Scan.extract and dist.StreamedShardedScan.extract return it
PAIR_DTYPE = np.dtype([("key_hi", "<u8"), ("key_lo", "<u8"), ("smudge", "<u4"), ("pos", "u1"), ("alt", "u1"),
                       ("pad", "<u2")])


def _host_table(kt: KtabFiles):
    """hm_host_table view over a KtabFiles (keeps the numpy buffers alive via the returned refs)."""
    index = np.ascontiguousarray(kt.index, dtype=np.int64)
    recs = [np.ascontiguousarray(r) if not isinstance(r, np.memmap) else r for r in kt.records]
    nparts = len(recs)
    part_nels = (C.c_int64 * max(nparts, 1))(*[int(x) for x in kt.part_nels])
    part_rec = (C.c_void_p * max(nparts, 1))(*[r.ctypes.data if r.size else None for r in recs])
    ht = _lib.HostTable(kt.kmer, kt.ibyte, nparts, kt.minval, kt.nels,
                        index.ctypes.data_as(C.POINTER(C.c_int64)), part_nels, part_rec, None, None)
    return ht, (index, recs, part_nels, part_rec)


class _OwnedTable:
    """The one-part host table hm_scan_condition_host made.  Every array viewing it holds this object, and it is
    freed (hm_host_table_free) when the last of them and the Scan that owns it have let it go."""

    def __init__(self, ptr):
        self.ptr = ptr
        self._free = _lib.lib().hm_host_table_free

    def _array(self, addr, shape, typestr):
        holder = type("_View", (), {})()
        holder.owner = self
        holder.__array_interface__ = {"shape": shape, "typestr": typestr, "data": (addr, False), "version": 3}
        return np.asarray(holder)

    def ktab(self) -> KtabFiles:
        v = self.ptr.contents
        n, pbyte = int(v.nels), ((v.kmer + 3) >> 2) - v.ibyte + 2
        index = self._array(C.cast(v.index, C.c_void_p).value, (1 << (8 * v.ibyte),), "<i8")
        rec = self._array(v.part_rec[0], (n * pbyte,), "|u1") if n else np.empty(0, dtype=np.uint8)
        return KtabFiles(kmer=v.kmer, nparts=1, minval=v.minval, ibyte=v.ibyte, index=index, part_nels=[n],
                         records=[rec])

    def __del__(self):
        if self.ptr:
            self._free(self.ptr)
            self.ptr = None


class Scan:
    """Device-resident table + both passes (hm_scan_*).  A table whose in-core scan does not fit the device
    budget is streamed through the GPU on every run() instead (residency()); device_budget (bytes per GPU)
    sets that budget for this and later scans of the process (0: free device memory minus a reserve).
    list_host_budget (bytes) lets a streamed run whose candidate records and S list outgrow the device budget keep
    them in host memory instead of refusing (hm_set_list_host_budget: for this and later runs of the process; 0,
    the default, is off); spill_stats() tells what the last run did.
    from_ktab(src, L) scans a raw FastK table as hetmers -e<L> does, conditioning it on the way in."""

    def __init__(self, kt: KtabFiles, gpus: int = 1, devices=None, device_budget: int | None = None, _owned=None,
                 _stream=False, list_host_budget: int | None = None):
        L = _lib.lib()
        self._L = L
        self._h = None
        self._owned = _owned                      # (from_ktab) the conditioned host table (_OwnedTable)
        self.kt = _owned.ktab() if _owned else kt
        self.stats = {}
        if device_budget is not None:
            L.hm_set_device_budget(int(device_budget))
        if list_host_budget is not None:
            L.hm_set_list_host_budget(int(list_host_budget))
        if _owned:
            ht, self._keep = _owned.ptr.contents, None
        else:
            ht, self._keep = _host_table(kt)      # a streamed scan reads these buffers on every run
        self._ht = ht
        self.devices = list(devices) if devices is not None else list(range(gpus))
        arr = (C.c_int * len(self.devices))(*self.devices)
        h = C.c_void_p()
        create = L.hm_scan_create_streamed if _stream else L.hm_scan_create
        rc = create(C.byref(ht), arr, len(self.devices), C.byref(h))
        if rc != 0:
            self.close()
            _lib.check(rc)
        self._h = h

    @classmethod
    def from_ktab(cls, src, L=None, gpus: int = 1, devices=None, device_budget: int | None = None,
                  host_budget: int | None = None, list_host_budget: int | None = None):
        """The scan of the FastK table `src` as hetmers -e<L> scans it, in one process on `gpus` GPUs (or the
        device ids `devices`), for a table of any size, without writing a conditioned copy.  L None, or a table
        hm_scan_examine(L) finds trimmed and symmetric, gives Scan over the source files.  Otherwise the table is
        trimmed and / or symmetrised on the way in, by the one route the sizes allow: in place on the devices
        (hm_scan_condition) when the source is in core and that fits the device budget, else into host memory
        (hm_scan_condition_host on the same devices; an in-core source is first reopened streamed, so that the
        conditioning has the device budget to itself; the source scan is destroyed afterwards) and a scan created
        over that table, in core if it fits, streamed if not.  The scan owns the host table: close() destroys the
        scan, then frees the table unless arrays of self.kt (its records and index) are still held elsewhere, in
        which case they keep it alive.  device_budget: device bytes per GPU, as Scan's; host_budget: host bytes the
        conditioned table may take (None: no cap), checked against the output histogram's bound before the first
        range pass (HetmersError -3 with both sizes).  list_host_budget: as Scan's (host bytes of a streamed run's
        lists), independent of host_budget.  stats["condition"] differs by route: always route ("none",
        "in_place" or "host"), steps ("trim", "symmetrise") and host_bytes (the host table's records and index, 0
        but on the host route); "in_place" adds nels_in, nels_out and ms_total; "host" adds every
        hm_condition_stats field (ranges, passes, peak_bytes, budget_bytes, ...)."""
        import time
        lib = _lib.lib()
        sc = cls(read_ktab(str(src), mmap=True), gpus, devices, device_budget, list_host_budget=list_host_budget)
        st = {"route": "none", "steps": [], "host_bytes": 0}
        sc.stats = {"condition": st}
        try:
            if L is None:
                return sc
            trim, symm = sc.examine(int(L))
            st["steps"] = [name for name, done in (("trim", trim), ("symmetrise", symm)) if not done]
            if not st["steps"]:
                return sc
            if not sc.residency()[0]:
                t0 = time.perf_counter()
                try:                                    # refused (HM_ENOMEM) before the table is touched
                    n = sc.condition(int(L), not trim, not symm)
                    st.update(route="in_place", nels_in=sc.kt.nels, nels_out=n,
                              ms_total=(time.perf_counter() - t0) * 1e3)
                    return sc
                except _lib.HetmersError as e:
                    if e.code != -3:
                        raise
                src_kt, devs = sc.kt, sc.devices        # the resident source goes: conditioning reads the host table
                sc.close()
                sc = cls(src_kt, devices=devs, _stream=True)
            ht = C.POINTER(_lib.HostTable)()
            cs = _lib.ConditionStats()
            was = lib.hm_set_condition_gpus(len(sc.devices))
            try:
                _lib.check(lib.hm_scan_condition_host(sc._h, int(L), int(not trim), int(not symm),
                                                      -1 if host_budget is None else int(host_budget), C.byref(ht),
                                                      C.byref(cs)))
            finally:
                lib.hm_set_condition_gpus(was)
            sc.close()
            out = cls(None, devices=sc.devices, _owned=_OwnedTable(ht))
        except BaseException:
            sc.close()
            raise
        st.update(route="host", **cs.as_dict())
        st["host_bytes"] = cs.bytes_written
        out.stats = {"condition": st}
        return out

    def examine(self, ethresh: int):
        """(trimmed?, symmetric?) as examine_table decides them (PloidyPlot.c:1167-1230)."""
        trim, symm = C.c_int(), C.c_int()
        _lib.check(self._L.hm_scan_examine(self._h, ethresh, C.byref(trim), C.byref(symm)))
        return bool(trim.value), bool(symm.value)

    def condition(self, ethresh: int, trim: bool, symm: bool) -> int:
        """trim (count >= ethresh) and / or symmetrise the device table in place (what the reference
        gets from FastK's Logex / Symmex, PloidyPlot.c:1381-1426); returns the new entry count"""
        n = C.c_int64()
        _lib.check(self._L.hm_scan_condition(self._h, ethresh, int(trim), int(symm), C.byref(n)))
        self.nels = n.value
        return n.value

    def condition_files(self, dst: str, ethresh: int, trim: bool, symm: bool, device_budget: int | None = None,
                        gpus: int | None = None):
        """write the trimmed (count >= ethresh) and / or symmetrised table as the FastK table `dst`, one key range
        at a time on the first GPU, for a table of any size (hm_scan_condition_files); the scan itself is left as
        it was.  A `dst` whose files are the source's (kt.name) is refused (HM_EINVAL) before anything is written.
        device_budget sets the process-wide device budget (bytes per GPU, as Scan's does) for this and later calls;
        an explicit budget counts what the scan already holds on the device.  gpus=n runs this call on the scan's
        first min(n, its GPUs) devices, the ranges dealt round-robin and written at their offsets by a thread per
        GPU (hm_set_condition_gpus; the files are the same); None keeps the process-wide setting (default 1).
        -> stats dict (entries in / out, ranges, passes, peak device bytes, bytes read / written, times, gpus)"""
        from .fastk import same_table_files
        if self.kt.name is not None and same_table_files(self.kt.name, self.kt.nparts, str(dst)):
            raise _lib.HetmersError(-1, f"{dst} names the source table: conditioning writes a new table")
        if device_budget is not None:
            self._L.hm_set_device_budget(int(device_budget))
        st = _lib.ConditionStats()
        was = self._L.hm_set_condition_gpus(int(gpus)) if gpus is not None else None
        try:
            _lib.check(self._L.hm_scan_condition_files(self._h, int(ethresh), int(trim), int(symm), str(dst).encode(),
                                                       C.byref(st)))
        finally:
            if was is not None:
                self._L.hm_set_condition_gpus(was)
        return st.as_dict()

    PATHS = {"auto": 0, "direct": 1, "symm": 2}

    def residency(self):
        """-> (streamed?, peak device bytes per GPU, chunks of the last run)"""
        b, c = C.c_int64(), C.c_int64()
        r = self._L.hm_scan_residency(self._h, C.byref(b), C.byref(c))
        return bool(r), b.value, c.value

    def spill_stats(self):
        """-> dict of hm_spill_stats for the last run: spilled, flushes, d2h_bytes, host_peak_bytes, partitions,
        rounds, h2d_bytes, slice, part, ms_pass1, ms_flush, ms_pass2"""
        st = _lib.SpillStats()
        _lib.check(self._L.hm_scan_spill_stats(self._h, C.byref(st)))
        return st.as_dict()

    def is_symmetric(self) -> bool:
        """whole-table verdict of the symmetry fingerprint (hm_scan_create / hm_scan_condition)"""
        return bool(self._L.hm_scan_is_symmetric(self._h))

    def run(self, path: str = "auto"):
        """-> (plot int64[1001,501], stats dict).  path "auto": the strand-symmetric scan when the table
        is symmetric, else the direct passes; "direct" / "symm" force one (stats["path"]: 1 / 2)"""
        plot = np.zeros(_lib.PLOT_CELLS, dtype=np.int64)
        st = _lib.ScanStats()
        _lib.check(self._L.hm_scan_run_path(self._h, self.PATHS[path], plot.ctypes.data, C.byref(st)))
        return plot.reshape(_lib.SMAX + 1, _lib.PLOT_W), st.as_dict()

    def extract(self, pixmap: np.ndarray):
        """pair list of extract_kmer_pairs: pixmap uint16[1001,501], label 0 = none;
        -> structured array (key_hi, key_lo, smudge, pos, alt) sorted by (smudge, k-mer).  Takes the route
        run() takes: on a symmetric table the pairs are listed from the last symmetric run's candidates (a run is
        done first if there is none), else from the direct passes; HETMERS_PATH=direct|symm forces one."""
        pm = np.ascontiguousarray(pixmap, dtype=np.uint16).reshape(-1)
        assert pm.size == _lib.PLOT_CELLS
        out = C.POINTER(_lib.PairRec)()
        n = C.c_int64()
        _lib.check(self._L.hm_scan_extract(self._h, pm.ctypes.data, C.byref(out), C.byref(n)))
        dt = PAIR_DTYPE
        arr = np.empty(n.value, dtype=dt)
        if n.value:
            C.memmove(arr.ctypes.data, out, n.value * dt.itemsize)
        libc = C.CDLL(None)
        libc.free.argtypes = [C.c_void_p]
        libc.free(out)
        return arr

    def pairs_hist(self, pixmap: np.ndarray):
        """the records of extract()'s list per key prefix (the top min(20, 2k) bits of key_hi), counted by the
        histogram sweep that write_pairs plans with (hm_scan_pairs_hist) -> uint64[2^min(20, 2k)]"""
        pm = np.ascontiguousarray(pixmap, dtype=np.uint16).reshape(-1)
        assert pm.size == _lib.PLOT_CELLS
        h = np.zeros(1 << min(_lib.COND_HIST_BITS, 2 * self.kt.kmer), dtype=np.uint64)
        _lib.check(self._L.hm_scan_pairs_hist(self._h, pm.ctypes.data, h.ctypes.data))
        return h

    def write_pairs(self, sma, out, device_budget: int | None = None):
        """extract_kmer_pairs' files for the smudges of `sma` (parsed as read_sma parses it): <out>.<a>A<b>B.txt per
        label, byte for byte what the executable writes, sorted and formatted on the GPUs (hm_scan_write_pairs,
        DESIGN.md §6c).  device_budget sets the process-wide device budget (bytes per GPU, as Scan's does) for this
        and later calls.  A plan that does not fit raises HetmersError -3 before any file is touched.
        -> stats dict: records, passes, windows, room, lines per label name, peak_bytes (device bytes beyond the
        scan's), budget (device bytes the call may hold beside the scan), path, and the phase times"""
        pix, labels = read_sma(sma)
        if device_budget is not None:
            self._L.hm_set_device_budget(int(device_budget))
        names = [f"{a}A{b}B" for a, b in labels]
        paths = [f"{out}.{n}.txt" for n in names]
        arr = (C.c_char_p * max(len(paths), 1))(*[p.encode() for p in paths])
        st = _lib.PairsStats()
        pm = np.ascontiguousarray(pix, dtype=np.uint16).reshape(-1)
        _lib.check(self._L.hm_scan_write_pairs(self._h, pm.ctypes.data, len(paths), arr, C.byref(st)))
        d = st.as_dict()
        line = self.kt.kmer + 5
        d["lines"] = {n: os.path.getsize(p) // line for n, p in zip(names, paths)}
        return d

    def download(self, deg: bool = True):
        n = getattr(self, "nels", self.kt.nels)
        keys = np.empty(n, dtype=np.uint64)
        klo = np.empty(n, dtype=np.uint64) if self.kt.kmer > 32 else None
        cnt = np.empty(n, dtype=np.uint16)
        d = np.empty(n, dtype=np.uint8) if deg else None
        _lib.check(self._L.hm_scan_download(self._h, keys.ctypes.data, klo.ctypes.data if klo is not None else None,
                                            cnt.ctypes.data, d.ctypes.data if deg else None))
        if klo is not None:
            keys = np.stack([keys, klo], axis=1)          # [n, 2] (hi, lo) words
        return keys, cnt, d

    def close(self):
        if getattr(self, "_h", None):
            self._L.hm_scan_destroy(self._h)
            self._h = None
        if getattr(self, "_owned", None):               # after the scan that reads it
            self._owned = self._ht = None
            self.kt = None

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def scan_table(kt: KtabFiles, gpus: int = 1):
    """one call: H2D + unpack + index + pass 1 + pass 2 + plot D2H (hm_hetmers_host)."""
    L = _lib.lib()
    ht, keep = _host_table(kt)
    devs = (C.c_int * gpus)(*range(gpus))
    plot = np.zeros(_lib.PLOT_CELLS, dtype=np.int64)
    st = _lib.ScanStats()
    _lib.check(L.hm_hetmers_host(C.byref(ht), devs, gpus, plot.ctypes.data, C.byref(st)))
    del keep
    return plot.reshape(_lib.SMAX + 1, _lib.PLOT_W), st.as_dict()


def condition_table(src, dst, L: int, device_budget: int | None = None, gpus: int | None = None):
    """`condition_kmer_table` in process: examine `src` as hetmers does (-e L) and write it trimmed and / or
    symmetrised as needed to `dst`, streaming it through the GPU if it is larger.  device_budget sets the
    process-wide device budget, as Scan's does.  gpus=n scans and conditions on devices 0..n-1 (what
    HETMERS_GPUS=n does for the executable); None keeps one GPU.  -> stats dict, or None when the table needs
    neither step (nothing is written).  A `dst` naming `src` is refused (HM_EINVAL) before anything is written."""
    if device_budget is not None:
        _lib.lib().hm_set_device_budget(int(device_budget))
    with Scan(read_ktab(str(src), mmap=True), gpus=1 if gpus is None else int(gpus)) as sc:
        trim, symm = sc.examine(int(L))
        if trim and symm:
            return None
        return sc.condition_files(dst, int(L), not trim, not symm, gpus=gpus)


def smu_text(plot: np.ndarray) -> str:
    """the .smu rows: "min\\t(sum-min)\\tcount", sum-major, min < 500 (PloidyPlot.c:1612-1615)"""
    p = np.asarray(plot).reshape(_lib.SMAX + 1, _lib.PLOT_W)[:, :_lib.FMAX]
    s, m = np.nonzero(p > 0)
    return "".join(f"{mi}\t{si - mi}\t{p[si, mi]}\n" for si, mi in zip(s.tolist(), m.tolist()))


def write_smu(path: str, plot: np.ndarray) -> None:
    L = _lib.lib()
    a = np.ascontiguousarray(np.asarray(plot, dtype=np.int64).reshape(-1))
    _lib.check(L.hm_write_smu(path.encode(), a.ctypes.data))


def hetmers(infile, o="smudgeplot", L=None, t=4, verbose=False, tmp=".", gpus: int = 1):
    """In-process equivalent of the `hetmers` task: returns the path of the .smu.  Tables that need
    trimming / symmetrising are conditioned on the GPU (hm_scan_condition)."""
    if L is None:
        raise ValueError("-L (count threshold) is required")
    kt = read_ktab(infile, mmap=True)
    with Scan(kt, gpus=gpus) as sc:
        trim, symm = sc.examine(int(L))
        if verbose:
            sys.stderr.write("\n  The input table is %s\n" % (
                ("trimmed and symmetric" if symm else "trimmed but not symmetric") if trim else
                ("untrimmed yet symmetric" if symm else "untrimmed and not symmetric")))
        if not (trim and symm):
            sc.condition(int(L), not trim, not symm)          # on the GPU (the reference: Logex / Symmex)
        plot, _ = sc.run()
    write_smu(f"{o}.smu", plot)
    return f"{o}.smu"

"""CPU tests of the drop-in boundary: the C-ABI library loads and exports every symbol the header
declares, and the `hetmers` executable honours the reference's argv / message / exit-code
contract (PloidyPlot.c:1246-1314,1350-1354; gene_core.h:32-56) for the cases that need no GPU."""
import os
import re
import subprocess
import sys

import pytest

from conftest import GOLDEN, ROOT
from smudgeplot_b200 import _lib, hetmers


def test_library_loads_and_exports_header_symbols(built):
    L = _lib.lib()
    hdr = open(os.path.join(ROOT, "include", "hetmers_b200.h")).read()
    declared = set(re.findall(r"\b(hm_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"hm_last_error"} - {"hm_last_error"}
    assert declared, "no declarations parsed"
    for sym in sorted(declared):
        assert hasattr(L, sym), f"{sym} declared in hetmers_b200.h but not exported"
    assert declared == set(_lib.ABI_SYMBOLS)
    assert L.hm_abi_version() == 1
    assert L.hm_pick_bucket_bits(200_000_000) == 26
    assert L.hm_pick_bucket_bits(1) == 2
    assert L.hm_pick_filter_bits(200_000_000) == 33 and L.hm_pick_filter_bits(2) == 22
    assert L.hm_pick_filter_bits(400_000_000) == 34 and L.hm_pick_filter_bits(370_000_000) == 33 and L.hm_pick_filter_bits(5_000_000_000) == 37
    assert L.hm_filter_words(32) == (1 << 32) // 32


def run(*args, stdin="n\n"):
    return subprocess.run([_lib.BIN_PATH, *args], input=stdin, capture_output=True, text=True)


def test_usage_on_wrong_positional_count(built):
    for argv in ([], ["a", "b"]):
        r = run(*argv)
        assert r.returncode == 1
        assert r.stderr.startswith("\nUsage: hetmers  [-v] [-T<int(4)>] [-P<dir(/tmp)>]\n")
        assert "-e: count threshold below which k-mers are considered erroneous" in r.stderr
        assert r.stdout == ""


def test_illegal_option_and_bad_integers(built):
    r = run("-x", "tab")
    assert (r.returncode, r.stderr) == (1, "hetmers: -x is an illegal option\n")
    r = run("-vq", "tab")
    assert (r.returncode, r.stderr) == (1, "hetmers: -q is an illegal option\n")
    r = run("-eabc", "tab")
    assert (r.returncode, r.stderr) == (1, "hetmers: -e 'abc' argument is not an integer\n")
    r = run("-T0", "tab")
    assert (r.returncode, r.stderr) == (1, "hetmers: Number of threads must be positive (0)\n")
    r = run("-e-3", "tab")
    assert (r.returncode, r.stderr) == (1, "hetmers: Error-mer threshold must be positive (-3)\n")


def test_missing_table_message_and_thread_clamp(built, tmp_path):
    r = run("-T100", "-vklfs", f"-o{tmp_path}/o", str(tmp_path / "absent"))
    assert r.returncode == 1
    assert r.stderr == ("hetmers: Warning, only 64 threads will be used\n"
                        f"hetmers: Cannot open k-mer table {tmp_path}/absent\n")


def test_existing_smu_prompt_reuse(built, tmp_path):
    out = tmp_path / "have"
    (tmp_path / "have.smu").write_text("1\t2\t3\n")
    r = run(f"-o{out}", os.path.join(GOLDEN, "dip_k21", "dip_k21"), stdin="yes please\n")
    assert r.returncode == 0
    assert r.stdout == f"\n  Found het-table {out}.smu, use it? "
    assert r.stderr == "\n  Using the found het-table, done\n"
    assert (tmp_path / "have.smu").read_text() == "1\t2\t3\n"          # untouched


def test_missing_part_file_is_reported(built, tmp_path):
    import shutil
    d = tmp_path / "g"
    shutil.copytree(os.path.join(GOLDEN, "trip_k31"), d)
    os.remove(d / ".trip_k31.ktab.3")
    r = run(f"-o{tmp_path}/o", str(d / "trip_k31"))
    assert r.returncode == 1 and "Table part" in r.stderr and "is missing ?" in r.stderr


def run_x(*args):
    exe = os.path.join(os.path.dirname(_lib.BIN_PATH), "extract_kmer_pairs")
    return subprocess.run([exe, *args], capture_output=True, text=True)


def test_extract_kmer_pairs_cli_contract(built, tmp_path):
    """argv / .sma parsing / messages of PloidyList.c:1207-1352 (cases that need no GPU)"""
    r = run_x("only_one")
    assert r.returncode == 1 and r.stderr.startswith("\nUsage: extract_kmer_pairs  [-v] [-T<int(4)>] [-P<dir(/tmp)>]\n")
    assert "<source>[.ktab] <smudges>[.sma]" in r.stderr
    r = run_x(f"-o{tmp_path}/o", "tab", str(tmp_path / "missing"))
    assert (r.returncode, r.stderr) == (1, f"\nextract_kmer_pairs: Could not open smudge file {tmp_path}/missing.sma")
    sma = tmp_path / "s.sma"
    for body, msg in (("5\t9\t3\tAB\n", "extract_kmer_pairs: Cannot parse line '5\t9\t3\tAB\n'\n"),
                      ("5\t9\t3\t1A2B\n", "extract_kmer_pairs: 1A2B is not a valid smudge label'\n"),
                      ("9\t5\t3\t1A1B\n", "extract_kmer_pairs: (9,5) is not a valid pixel coordinate\n")):
        sma.write_text("covB\tcovA\tfreq\tsmudge\n" + body)
        r = run_x(f"-o{tmp_path}/o", "tab", str(sma))
        assert (r.returncode, r.stderr) == (1, msg)
    # a good .sma: the per-smudge files are created before the table is opened, like the reference
    sma.write_text("covB\tcovA\tfreq\tsmudge\n5\t9\t3\t1A1B\n6\t9\t1\t2A1B\n7\t9\t1\t1A1B\n")
    r = run_x(f"-o{tmp_path}/o", str(tmp_path / "absent"), str(tmp_path / "s"))
    assert (r.returncode, r.stderr) == (1, f"extract_kmer_pairs: Cannot open k-mer table {tmp_path}/absent\n")
    assert sorted(f.name for f in tmp_path.glob("o.*.txt")) == ["o.1A1B.txt", "o.2A1B.txt"]
    assert hetmers.extract_args("t.ktab", "x.sma", o="kp", t=8, verbose=True, tmp="/s") == \
        ["-okp", "-T8", "-v", "-P/s", "t.ktab", "x"]                                   # cli.py:368-378


def test_cli_argv_mirror_of_reference_cli():
    # cli.py:350-359
    assert hetmers.hetmers_args("t.ktab", o="out", L=12, t=4) == ["-oout", "-e12", "-T4", "t.ktab"]
    assert hetmers.hetmers_args("t", o="o", L=3, t=8, verbose=True, tmp="/scratch") == \
        ["-oo", "-e3", "-T8", "-v", "-P/scratch", "t"]
    with pytest.raises(ValueError):
        hetmers.hetmers_args("t")


def test_no_gpu_means_loud_failure(built, tmp_path):
    L = _lib.lib()
    if L.hm_device_count() > 0:
        pytest.skip("a GPU is visible here")
    r = run(f"-o{tmp_path}/o", os.path.join(GOLDEN, "dip_k21", "dip_k21"))
    assert r.returncode == 1 and "no CUDA device" in r.stderr and not (tmp_path / "o.smu").exists()
    from smudgeplot_b200 import fastk
    with pytest.raises(_lib.HetmersError):
        hetmers.scan_table(fastk.read_ktab(os.path.join(GOLDEN, "dip_k21", "dip_k21")))


# ---------------------------------------------------------------- layer C on the CPU (plain C) ----

def _open_table(path):
    import ctypes as C
    L = _lib.lib()
    h = C.c_void_p()
    rc = L.hm_table_open(path.encode(), C.byref(h))
    return rc, h


def test_layer_c_parser_matches_python_reader_on_goldens(built):
    """hm_table_open (host/fastk_table.c) against smudgeplot_b200.fastk.read_ktab on every golden
    table: header fields, part sizes, prefix index and the mapped payload bytes"""
    import ctypes as C
    import numpy as np
    from conftest import golden_cases
    from smudgeplot_b200 import fastk
    L = _lib.lib()
    for name in golden_cases():
        path = os.path.join(GOLDEN, name, name)
        kt = fastk.read_ktab(path)
        rc, h = _open_table(path + ".ktab")                    # suffix accepted, like the reference
        assert rc == 0, L.hm_last_error()
        v = L.hm_table_view(h).contents
        assert (v.kmer, v.ibyte, v.nparts, v.nels) == (kt.kmer, kt.ibyte, kt.nparts, kt.nels)
        idx = np.ctypeslib.as_array(v.index, shape=(1 << (8 * kt.ibyte),))
        assert np.array_equal(idx, kt.index)
        for p in range(kt.nparts):
            assert v.part_nels[p] == kt.part_nels[p]
            nbytes = kt.part_nels[p] * kt.pbyte
            if nbytes:
                raw = (C.c_uint8 * nbytes).from_address(v.part_rec[p])
                assert bytes(raw) == kt.records[p].tobytes()
            assert v.part_fd[p] >= 0 and v.part_fd_off[p] == 12      # kept open for the pread loader
        L.hm_table_close(h)


def test_layer_c_error_codes(built, tmp_path):
    import shutil
    L = _lib.lib()
    rc, _ = _open_table(str(tmp_path / "absent"))
    assert rc == -4 and L.hm_last_error().decode().startswith("Cannot open k-mer table")      # HM_EIO
    d = tmp_path / "g"
    shutil.copytree(os.path.join(GOLDEN, "trip_k31"), d)
    part = d / ".trip_k31.ktab.2"
    data = part.read_bytes()
    part.write_bytes(data[: len(data) // 2])                       # truncated payload
    rc, _ = _open_table(str(d / "trip_k31"))
    assert rc == -5 and "truncated" in L.hm_last_error().decode()  # HM_EFORMAT (the reference reads garbage)
    part.write_bytes(b"\x15\x00\x00\x00" + data[4:])               # part says k=21, stub says k=31
    rc, _ = _open_table(str(d / "trip_k31"))
    assert rc == -5 and "k-mer length matching stub" in L.hm_last_error().decode()
    stub = d / "trip_k31.ktab"
    sb = stub.read_bytes()
    stub.write_bytes(sb[:100])                                     # truncated prefix index
    rc, _ = _open_table(str(d / "trip_k31"))
    assert rc == -5 and "truncated prefix index" in L.hm_last_error().decode()
    stub.write_bytes(sb[:12] + b"\x07\x00\x00\x00" + sb[16:])      # ibyte = 7
    rc, _ = _open_table(str(d / "trip_k31"))
    assert rc == -5 and "implausible stub header" in L.hm_last_error().decode()


def test_layer_c_smu_writer_matches_oracle_writer(built, tmp_path):
    import ctypes as C
    import numpy as np
    import oracle_util as ou
    rng = np.random.default_rng(5)
    plot = np.zeros((_lib.SMAX + 1, _lib.PLOT_W), dtype=np.int64)
    s = rng.integers(0, _lib.SMAX + 1, size=4000)
    m = np.minimum(rng.integers(0, _lib.PLOT_W, size=4000), s // 2)
    np.add.at(plot, (s, m), rng.integers(1, 10**12, size=4000))
    plot[1000, 500] = 7                                            # computed but never written (i < FMAX)
    out = str(tmp_path / "w.smu")
    assert _lib.lib().hm_write_smu(out.encode(), plot.ctypes.data) == 0
    text = open(out).read()
    assert text == ou.smu_text(plot) == hetmers.smu_text(plot)
    assert "500\t500\t" not in text
    rows = [tuple(int(v) for v in ln.split("\t")) for ln in text.splitlines()]
    assert rows == sorted(rows, key=lambda r: (r[0] + r[1], r[0]))   # sum-major, then min (PloidyPlot.c:1612)


# ---- strand-symmetric scan: host-side pieces of the C ABI (no GPU needed) -------------------------

def test_symm_plan_layout_invariants(built):
    import ctypes as C
    from smudgeplot_b200 import _lib
    L = _lib.lib()
    for n, rng, k, seg in ((2, 2, 31, 1), (200_000_000, 200_000_000, 31, 1), (1_600_000_000, 200_000_000, 31, 8),
                           (5_000_000_000, 625_000_000, 40, 8), (1000, 0, 21, 2)):
        lay = _lib.SymmLayout()
        assert L.hm_symm_plan(n, rng, k, seg, C.byref(lay)) == 0
        assert lay.n_seg == seg and lay.range == rng
        assert lay.cand_cap >= rng // 2 + 1 and lay.runs_cap >= rng // 3 + 1
        assert lay.seg_words >= 1024 and lay.seg_words % 64 == 0
        assert lay.seg_words * 32 * seg >= n                    # at least one filter bit per table entry in all
        # regions in order, non-overlapping, 8-byte aligned, inside `bytes`
        regs = [(lay.off_header, 256), (lay.off_bloom, 4 * lay.seg_words * seg), (lay.off_cand_key, 8 * lay.cand_cap)]
        if k > 32:
            regs.append((lay.off_cand_lo, 8 * lay.cand_cap))
        regs += [(lay.off_cand_meta, 8 * lay.cand_cap), (lay.off_runs, 8 * lay.runs_cap)]
        end = 0
        for off, size in regs:
            assert off % 8 == 0 and off >= end
            end = off + size
        assert end <= lay.bytes and lay.bytes % 256 == 0
    lay = _lib.SymmLayout()
    assert L.hm_symm_plan(10, 20, 31, 1, C.byref(lay)) == -1    # range > n
    assert L.hm_symm_plan(10, 5, 31, 0, C.byref(lay)) == -1     # no segment
    assert L.hm_symm_plan(10, 5, 31, _lib.MAX_SHARDS + 1, C.byref(lay)) == -1
    assert b"hm_symm_plan" in L.hm_last_error()


def test_symm_bloom_bits_env_and_multi_gpu_default(built, monkeypatch):
    """one filter bit per entry on one GPU (a filter that fits the L2 the access-policy window holds it in) and on
    several (the segments cross NVLink); HETMERS_BLOOM_BITS overrides both"""
    import ctypes as C
    from smudgeplot_b200 import _lib
    L = _lib.lib()
    monkeypatch.delenv("HETMERS_BLOOM_BITS", raising=False)
    one, many = _lib.SymmLayout(), _lib.SymmLayout()
    n = 64_000_000
    assert L.hm_symm_plan(n, n, 31, 1, C.byref(one)) == 0 and L.hm_symm_plan(8 * n, n, 31, 8, C.byref(many)) == 0
    assert one.seg_words * 32 >= n and one.seg_words * 32 < n + 64 * 32
    assert many.seg_words * 32 >= n and many.seg_words * 32 < n + 64 * 32
    monkeypatch.setenv("HETMERS_BLOOM_BITS", "5")
    five = _lib.SymmLayout()
    assert L.hm_symm_plan(n, n, 31, 1, C.byref(five)) == 0 and five.seg_words * 32 >= 5 * n


def test_symm_seeds_are_drawn_once_per_process(built):
    import ctypes as C
    from smudgeplot_b200 import _lib
    L = _lib.lib()
    a, b = (C.c_uint64 * 2)(), (C.c_uint64 * 2)()
    L.hm_symm_seeds(a)
    L.hm_symm_seeds(b)
    assert (a[0], a[1]) == (b[0], b[1]) and (a[0] != 0 or a[1] != 0) and a[0] != a[1]
    r = subprocess.run([sys.executable, "-c",
                        "import sys; sys.path.insert(0, %r); import ctypes as C; from smudgeplot_b200 import _lib; "
                        "s = (C.c_uint64 * 2)(); _lib.lib().hm_symm_seeds(s); print(s[0], s[1])" % ROOT],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    other = tuple(int(v) for v in r.stdout.split())
    assert other != (a[0], a[1])                                # another process, other seeds

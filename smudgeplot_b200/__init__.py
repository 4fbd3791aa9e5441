"""smudgeplot_b200 -- H100 (sm_90a) implementation of smudgeplot's `hetmers` hot path.

The product is native: `lib/libhetmers_b200.so` (CUDA kernels + C ABI, include/hetmers_b200.h) and
the drop-in executables `bin/hetmers` / `bin/extract_kmer_pairs` (plain C host).  The Python in
this package is the host-side mirror of the reference's interface for that path and test / bench
plumbing:

    hetmers.py   argv of `smudgeplot hetmers|extract` (cli.py:348-382), run_hetmers / run_extract,
                 in-process Scan (C ABI layer B)
    fastk.py     FastK .ktab reader / writer (numpy)
    device.py    C ABI layer A on torch-owned device memory
    dist.py      one-process-per-GPU sharding (torch.distributed: NCCL / gloo; CUDA IPC peer arrays)
    _lib.py      ctypes binding; raises if the library has not been built -- there is no fallback
"""

__version__ = "0.1.0"

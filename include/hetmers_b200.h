/*******************************************************************************************
 * hetmers_b200.h -- C ABI of libhetmers_b200.so, the H100 (sm_90a) implementation of
 * smudgeplot's `hetmers` hot path.
 *
 * The reference has NO in-process API for this path: its boundary is the `hetmers` executable
 * spawned by smudgeplot's CLI (src/smudgeplot/cli.py:57-72,348-361) and the
 * whole computation lives in src/lib/PloidyPlot.c + the Kmer_Stream part of src/lib/libfastk.c.
 * The drop-in therefore is our own `hetmers` executable (smudgeplot_b200/host/hetmers_main.c,
 * plain C); this header is the thin layer between that C host (or any FFI: ctypes, cgo, JNI)
 * and the CUDA kernels.  Plain pointers and sizes only; no torch / C++ types.
 *
 * Every entry point names the reference code it replaces (file:line in the reference smudgeplot repository).
 * All functions return 0 on success and a negative HM_E* code on failure; hm_last_error()
 * gives the message (thread-local).  There is NO CPU fallback anywhere behind this ABI.
 *
 * Layers
 *   A. hm_k_*      kernels on caller-owned DEVICE memory, enqueued on a caller stream
 *                  (used by the torch.distributed plumbing in smudgeplot_b200/dist.py and by B)
 *   B. hm_scan_*   whole path from HOST buffers holding raw FastK part payloads: H2D, unpack,
 *                  bucket index, pass 1, pass 2, D2H of the plot (used by hetmers_main.c,
 *                  by smudgeplot_b200.hetmers() and by bench.py's e2e leg)
 *   C. hm_table_*  FastK stub/part parser on the host (plain C, host/fastk_table.c)
 *******************************************************************************************/
#ifndef HETMERS_B200_H
#define HETMERS_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HM_SMAX        1000                 /* max CovA+CovB      (PloidyPlot.c:48) */
#define HM_FMAX         500                 /* max min(CovA,CovB) (PloidyPlot.c:49) */
#define HM_PLOT_W      (HM_FMAX+1)
#define HM_PLOT_CELLS  ((HM_SMAX+1)*(HM_FMAX+1))   /* int64 plot[1001][501] (PloidyPlot.c:1466-1473) */
#define HM_MAX_KMER      64                 /* 1 (k<=32) or 2 (k<=64) 64-bit words per packed k-mer */
#define HM_MAX_SHARDS    16                 /* GPUs one table can be sharded over           */
#define HM_FILTER_MIN_BITS 22               /* prefix-filter width in bits                  */
#define HM_FILTER_MAX_BITS 37

#define HM_OK            0
#define HM_EINVAL       -1                  /* bad argument                                   */
#define HM_ECUDA        -2                  /* CUDA runtime / launch failure                  */
#define HM_ENOMEM       -3                  /* host or device allocation failed               */
#define HM_EIO          -4                  /* cannot open / read a table file                */
#define HM_EFORMAT      -5                  /* malformed FastK table                          */
#define HM_EUNSUPPORTED -6                  /* valid input this build does not handle (k>64)  */

const char *hm_last_error(void);
int         hm_abi_version(void);
/* number of visible CUDA devices (0 if none / no driver) */
int         hm_device_count(void);
/* name, SM count and total memory of device `dev` (for -v / bench provenance) */
int         hm_device_info(int dev, char *name, int name_len, int *sm_count, int64_t *total_mem);

/* ======================= A. kernels on device memory ===================================== *
 * Device table layout (structure of arrays, DESIGN.md §3):
 *   keys  uint64[n]  packed 2-bit k-mer, LEFT aligned (base i in bits 63-2i..62-2i), ascending;
 *                    uint64 order == FastK table order (libfastk.c packing :571-579)
 *   keys_lo uint64[n] bases 32..63 (left aligned) when k > 32, else NULL: order = (keys, keys_lo)
 *   cnt   uint16[n]  k-mer counts
 *   deg   uint8 [n]  incidence array == the reference's `Pair` (PloidyPlot.c:163), allocated
 *                    with size rounded up to a multiple of 4 and 4-byte aligned
 *   bucket           lower-bound offsets of every `bits`-bit key prefix, (1<<bits)+1 entries,
 *                    uint32 if idx64==0 (n < 2^32-1) else uint64
 * `stream` is a cudaStream_t passed as void* (NULL = default stream).                        */

/* FastK part records -> SoA.  Replaces Next_Kmer_Entry/Current_Entry (libfastk.c:1159-1176,
 * :1230-1269): re-attaches the ibyte-byte prefix found from the stub index and splits the
 * unaligned (suffix || uint16 count) record.  d_rec: n records of pbyte=kbyte-ibyte+2 bytes,
 * holding table ordinals [first, first+n); d_stub_index: int64[1<<(8*ibyte)] on the device.   */
int hm_k_unpack_records(const uint8_t *d_rec, int64_t n, int64_t first,
                        const int64_t *d_stub_index, int ibyte, int kmer,
                        uint64_t *d_keys, uint64_t *d_keys_lo, uint16_t *d_cnt, void *stream);

/* Prefix (bucket) index over the sorted keys; takes the place of the stub index + on-disk
 * bisection of GoTo_Kmer_Entry (libfastk.c:1320-1409).                                        */
int hm_k_build_bucket_index(const uint64_t *d_keys, int64_t n, int bits,
                            void *d_bucket, int idx64, void *stream);

/* Prefix presence filter: bit f of d_filter is set iff some key starts with the filter_bits-bit
 * prefix f; hm_filter_words(filter_bits) uint32 words (zeroed here).  It answers "is there any
 * k-mer with this prefix" for pass 1's probes -- the role the 4-way merge's "no list head has
 * this suffix" plays in the reference (PloidyPlot.c:618-643).                                  */
int     hm_k_build_filter(const uint64_t *d_keys, int64_t n, int filter_bits,
                          uint32_t *d_filter, void *stream);
int64_t hm_filter_words(int filter_bits);
int     hm_pick_filter_bits(int64_t n);

/* Sharded incidence array (multi-GPU, DESIGN.md §6).  The table is cut into n_shards contiguous
 * index ranges [off[r], off[r+1]); GPU r owns the incidence bytes of shard r.  deg[r] is GPU r's
 * FULL-LENGTH array as addressable from the calling GPU (peer access in one process, or a CUDA
 * IPC mapping from hm_ipc_open between processes); only its slice r is meaningful.  With such a
 * table pass 1 adds to a foreign partner's byte with a remote atomic over NVLink and pass 2 reads
 * a foreign partner's byte with a remote load, so no collective has to move the array; the caller
 * only orders the phases (all pass 1 kernels done -> pass 2; all pass 2 done -> next zeroing).
 * NULL (or n_shards <= 1) = dense mode: every byte lives in d_deg.                              */
typedef struct hm_shards
  { int32_t  n_shards;
    int32_t  self;                          /* the calling GPU's shard                          */
    int64_t  off[HM_MAX_SHARDS+1];
    uint8_t *deg[HM_MAX_SHARDS];
    void    *scratch;                       /* optional device scratch for pass 2: look-ups of       */
    int64_t  scratch_bytes;                 /*   foreign partners are batched instead of done inline */
  } hm_shards;                              /*   (size: hm_pass2_scratch_bytes)                      */

int64_t hm_pass2_scratch_bytes(int64_t range, int idx64);

/* Pass 1 (PASS1=1 of PloidyPlot.c:1489; analysis_in_core_1 :454-568, analysis_thread_1
 * :168-301, big_window :712-842): for every entry x in [lo,hi) find every one-substitution
 * neighbour y > x in the table; for each such pair with cnt sum <= SMAX add 1 to deg[x] and
 * deg[y] (mod 256, atomically) and remember the pair's upper member in d_up[x-lo]
 * (all-ones = none; d_up is initialised here).  d_deg must be zeroed by the caller before the
 * first call (several ranges / GPUs accumulate into it).                                      */
int hm_k_pass1_degree(const uint64_t *d_keys, const uint64_t *d_keys_lo,
                      const uint16_t *d_cnt, int64_t n,
                      const void *d_bucket, int bits, int idx64,
                      const uint32_t *d_filter, int filter_bits, int kmer,
                      int64_t lo, int64_t hi, uint8_t *d_deg, void *d_up,
                      const hm_shards *shards, void *stream);

/* Pass 2 (PASS1=0; analysis_in_core_2 :570-700, analysis_thread_2 :303-452): for x in [lo,hi)
 * with deg[x]<=1 whose recorded upper partner y has deg[y]<=1: plot[cx+cy][min(cx,cy)] += 1.
 * d_plot: uint64[HM_PLOT_CELLS], accumulated into (caller zeroes it).                        */
int hm_k_pass2_plot(const uint16_t *d_cnt, const uint8_t *d_deg, const void *d_up, int idx64,
                    int64_t lo, int64_t hi, unsigned long long *d_plot,
                    const hm_shards *shards, void *stream);

/* extract_kmer_pairs' pass 2 (src/lib/PloidyList.c:425-450,680-705): every isolated pair whose
 * pixel (sum, min) has a non-zero label in d_pixmap (uint16[HM_PLOT_CELLS], the PLOT array the
 * reference fills from the .sma file, PloidyList.c:1313-1350) is appended to d_out: the k-mer with
 * the higher count, the varying position and the other k-mer's base there.  *d_count (zeroed by
 * the caller) counts all matches, also those beyond `cap`.                                      */
typedef struct hm_pair_rec
  { uint64_t key_hi, key_lo;   /* packed k-mer that print_het prints (left aligned words)       */
    uint32_t smudge;           /* label from the pixmap (index into the .sma smudge list, 1-based) */
    uint8_t  pos, alt;         /* varying base position; base (0..3 = acgt) of the partner there */
    uint16_t pad;
  } hm_pair_rec;

int hm_k_pass2_extract(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                       const uint8_t *d_deg, const void *d_up, int idx64, int64_t lo, int64_t hi,
                       const uint16_t *d_pixmap, hm_pair_rec *d_out, int64_t cap,
                       unsigned long long *d_count, const hm_shards *shards, void *stream);

/* ---- the strand-symmetric scan (csrc/hm_symm.cu): every entry read once ------------------------
 * On a table that holds rc(x) with count(x) for every x -- what the reference demands before it
 * scans (examine_table, PloidyPlot.c:1199-1229; `Symmex` otherwise, :1401-1414) -- the pairs that
 * differ at a low position are mirror images of the pairs that differ at a high position, and those
 * sit in one short run of neighbouring entries.  hm_k_symm_runscan + hm_k_symm_resolve produce the
 * same plot as hm_k_pass1_degree + hm_k_pass2_plot (= the reference's two passes) on such a table;
 * hm_k_symm_fingerprint decides whether a table is one (keyed multiset fingerprints of {(x,cnt)}
 * and {(rc x,cnt)}: acc[0]==acc[2] && acc[1]==acc[3]); anything else must take the direct passes.
 * Replaces, for such tables: analysis_in_core_1/_2 + analysis_thread_1/_2 and the window / recursion
 * drivers around them (PloidyPlot.c:168-700,:712-1084); the fingerprint extends examine_table's
 * one-k-mer symmetry probe (PloidyPlot.c:1199-1229) to the whole table.
 * Side effect: hm_k_symm_runscan puts an access-policy window (persisting L2 lines) over the Bloom
 * filter on `stream` and hm_k_symm_resolve lifts it again (HETMERS_L2_PERSIST=0 disables it).      */
#define HM_SYMM_MIN_KMER 2

typedef struct hm_symm_layout               /* work area of one scan range (hm_symm_plan fills it in)     */
  { int64_t bytes;                          /* device bytes to allocate (256-byte aligned)                */
    int64_t off_header;                     /* uint64[3]: candidate count, status bits (hm_symm_status), runs */
    int64_t off_bloom;                      /* n_seg segments of seg_words uint32: Bloom filter over the  */
    int64_t seg_words;                      /*   entries with a partner in their upper half, per shard    */
    int64_t off_cand_key, off_cand_lo, off_cand_meta;   /* candidate pair records                         */
    int64_t cand_cap;
    int64_t range;
    int64_t off_runs, runs_cap;             /* heads of the runs of three or more entries (uint64 indices) */
    int32_t n_seg, pad;
  } hm_symm_layout;

typedef struct hm_symm_shards               /* several GPUs: shard r scans [off[r], off[r+1]) and fills   */
  { int32_t  n_seg, self;                   /*   Bloom segment r; the segments are all-gathered between   */
    int64_t  off[HM_MAX_SHARDS+1];          /*   the two kernels.  Cuts lie on run boundaries             */
    uint64_t first_key[HM_MAX_SHARDS];      /*   (hm_symm_align_cut); first_key[r] = keys[off[r]]         */
  } hm_symm_shards;

#define HM_SYMM_ASYMMETRIC 1                /* status bit: some rc(x) was not in the table -> result void */
#define HM_SYMM_OVERFLOW   2                /* status bit: candidate list full (cut not on a run boundary) */

int  hm_symm_plan(int64_t n, int64_t range, int kmer, int n_seg, hm_symm_layout *out);
void hm_symm_seeds(uint64_t seed[2]);       /* per-process random seeds for the fingerprint               */
/* adds the fingerprints of entries [i0,i1) to d_acc (device uint64[4], zeroed by the caller)            */
int  hm_k_symm_fingerprint(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                           int64_t i0, int64_t i1, int kmer, const uint64_t seed[2],
                           uint64_t *d_acc, void *stream);
/* "pass 1": run scan of [lo,hi): Bloom segment `self` + candidate records (both initialised here), then
 * hm_k_symm_runs for the runs it only listed (call both, in this order, on the same stream).            */
int  hm_k_symm_runscan(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                       const void *d_bucket, int bits, int idx64, int kmer, int64_t lo, int64_t hi,
                       void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards, void *stream);
int  hm_k_symm_runs(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                    const void *d_bucket, int bits, int idx64, int kmer, int64_t lo, int64_t hi,
                    void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards, void *stream);
/* "pass 2": candidates -> isolated pairs -> d_plot (accumulated into; caller zeroes it)                 */
int  hm_k_symm_resolve(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                       const void *d_bucket, int bits, int idx64, int kmer,
                       void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards,
                       unsigned long long *d_plot, void *stream);
/* extract_kmer_pairs on the same work area, after hm_k_symm_runscan + hm_k_symm_runs (one GPU, or each GPU of an
 * in-core scan with the Bloom segments all-gathered): the isolated pairs among candidates [c0, c1) whose pixel
 * (sum, min) has a non-zero label in d_pixmap are appended to d_out as hm_k_pass2_extract lists them -- each
 * candidate once, and its mirror image (rc y, rc x) too unless the pair differs at the middle base of an odd k
 * (DESIGN.md §4a).  At most 2 (c1-c0) records; *d_count (zeroed by the caller) counts all of them, also those
 * beyond `cap`.  The candidate count is in the work-area header (hm_symm_status); c1 must not exceed it, except
 * that c0 = 0 with a larger c1 lists every candidate.                                                      */
int  hm_k_symm_extract(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                       const void *d_bucket, int bits, int idx64, int kmer,
                       void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards,
                       const uint16_t *d_pixmap, int64_t c0, int64_t c1, hm_pair_rec *d_out, int64_t cap,
                       unsigned long long *d_count, void *stream);
int  hm_symm_status(const void *d_work, const hm_symm_layout *layout, uint64_t *n_cand, uint64_t *status,
                    void *stream);
int  hm_symm_align_cut(const uint64_t *d_keys, int64_t n, int kmer, int64_t cut, int64_t *out);

/* Device memory that can be mapped by the other ranks of a one-process-per-GPU job (CUDA IPC):
 * hm_dev_alloc gives a zeroed base allocation on the current device, hm_ipc_export its 64-byte
 * handle (send it to the peers with any host transport), hm_ipc_open maps a peer's allocation.
 * hm_p2p_native_atomics: 1 iff devices a and b can do remote atomics on each other (NVLink).    */
int hm_dev_alloc(int64_t bytes, void **dptr);
int hm_dev_free(void *dptr);
int hm_ipc_export(void *dptr, unsigned char handle[64]);
int hm_ipc_open(const unsigned char handle[64], void **dptr);
int hm_ipc_close(void *dptr);
int hm_p2p_native_atomics(int dev_a, int dev_b);

/* examine_table (PloidyPlot.c:1167-1197): smallest count v>=1 (read as int16) in [frst,last);
 * *d_min (device int) must be preset to 0x8000.                                               */
int hm_k_min_count(const uint16_t *d_cnt, int64_t frst, int64_t last, int *d_min, void *stream);

/* exact-match lookup of nq packed k-mers: d_pos[q] = table index or -1.  Replaces
 * GoTo_Kmer_Entry's "return 1 iff exact hit" use (libfastk.c:1320-1409; PloidyPlot.c:1213). */
int hm_k_find_keys(const uint64_t *d_keys, const uint64_t *d_keys_lo, int64_t n,
                   const void *d_bucket, int bits, int idx64,
                   const uint64_t *d_query, const uint64_t *d_query_lo, int64_t nq,
                   int64_t *d_pos, void *stream);

/* choice of bucket-index width for a table of n entries (DESIGN.md §4) */
int hm_pick_bucket_bits(int64_t n);

/* ======================= B. whole path from host buffers ================================= */

typedef struct hm_host_table
  { int32_t         kmer;        /* k                                                   */
    int32_t         ibyte;       /* prefix bytes folded into the stub index (1..3)      */
    int32_t         nparts;
    int32_t         minval;
    int64_t         nels;        /* sum of part_nels                                    */
    const int64_t  *index;       /* int64[1 << (8*ibyte)] bucket END offsets            */
    const int64_t  *part_nels;   /* [nparts]                                            */
    const uint8_t **part_rec;    /* [nparts] payloads: part_nels[p]*pbyte bytes each    */
    const int32_t  *part_fd;     /* optional [nparts]: open descriptor of the part file (or -1);  */
    const int64_t  *part_fd_off; /*   payload starts at this offset.  When given, the loader       */
                                 /*   pread()s with its host threads instead of touching part_rec  */
  } hm_host_table;

typedef struct hm_scan_stats
  { int64_t nels;
    int32_t n_gpus;
    int32_t bucket_bits;
    int32_t filter_bits;
    int32_t path;                /* HM_PATH_DIRECT or HM_PATH_SYMM: which scan produced the plot */
    double  ms_h2d_unpack;       /* H2D copies + unpack + bucket index (T_load, device part) */
    double  ms_pass1;
    double  ms_pass2;
    double  ms_scan;             /* pass1 + exchange + pass2 + plot reduce (T_scan)          */
    double  ms_total;            /* wall clock of the call                                   */
    int64_t kernel_launches;     /* kernels of ours launched by the call                     */
    double  ms_alloc;            /* of ms_h2d_unpack: context + device allocations           */
    double  ms_records;          /*                   host staging + H2D + unpack            */
    double  ms_index;            /*                   shard exchange + bucket index + filter */
  } hm_scan_stats;

typedef struct hm_scan hm_scan;   /* opaque: device-resident table + work buffers            */

/* Load a table onto `n_gpus` devices (ids dev[0..n_gpus-1]; every device holds a full replica,
 * work is sharded by contiguous index range, DESIGN.md §6).  Replaces Open_Kmer_Stream +
 * Clone_Kmer_Stream + the 4 GiB cache fill (libfastk.c:786-951; PloidyPlot.c:954-964).       */
int  hm_scan_create(const hm_host_table *t, const int *dev, int n_gpus, hm_scan **out);
/* hm_scan_create, streamed whatever the table's size (what HETMERS_STREAM=1 does, for this call): nothing of the
 * table is resident, so a call that reads the host table itself (hm_scan_condition_host) has the device budget
 * to itself.  Scan.from_ktab conditions through such a scan when in-place conditioning does not fit.          */
int  hm_scan_create_streamed(const hm_host_table *t, const int *dev, int n_gpus, hm_scan **out);
/* Optional: start CUDA (driver + primary contexts of the first n_gpus visible devices, 0 = all) and
 * the pinned staging buffers on a background thread and return at once; hm_scan_create waits for
 * it.  Lets a short-lived process overlap CUDA start-up with opening its table files.             */
void hm_prewarm(int n_gpus);
/* host threads used to stage pageable (e.g. mmap'ed) part payloads into pinned memory during
 * hm_scan_create; 0 = min(16, cores).  The executable passes its -T here.                      */
void hm_set_io_threads(int n);
void hm_scan_destroy(hm_scan *s);
/* examine_table decisions (PloidyPlot.c:1167-1230) computed on the device */
int  hm_scan_examine(hm_scan *s, int ethresh, int *trim, int *symm);
/* Condition the device-resident table in place: trim = drop entries with count < ethresh (what
 * `Logex '...=A[<L>-]'` does), symm = add the reverse complement of every k-mer with the same
 * count (what `Symmex` does; the original wins where both are present) -- PloidyPlot.c:1381-1426
 * shells out to those FastK tools; here the table never leaves the GPU.  *nels_out = entries
 * afterwards.  Each GPU conditions its replica a key range at a time (DESIGN.md §4d) into new
 * arrays, which replace the old ones only when the whole call succeeds; the index is rebuilt and
 * the fingerprint verdict taken again.  The table, the new arrays and one range's working set must
 * fit the device budget: else HM_ENOMEM before anything is touched ("... needs N device bytes (M in
 * one range) ...": N is the least budget under which the call succeeds).  A failure on GPU 0 leaves
 * the old table usable; on a later GPU the scan is marked unusable.  A streamed scan refuses
 * (HM_EUNSUPPORTED).                                                                             */
int  hm_scan_condition(hm_scan *s, int ethresh, int do_trim, int do_symm, int64_t *nels_out);
/* both passes; plot: host int64[HM_PLOT_CELLS]; stats optional.  Tables that hm_scan_create found
 * strand-symmetric (fingerprint over the whole table) take the symmetric scan of csrc/hm_symm.cu,
 * all others the direct passes; both give the reference's plot.  hm_scan_run_path forces one
 * (HM_PATH_SYMM on a table that is not symmetric is an error); HETMERS_PATH=direct|symm overrides
 * HM_PATH_AUTO.                                                                                  */
#define HM_PATH_AUTO   0
#define HM_PATH_DIRECT 1
#define HM_PATH_SYMM   2
int  hm_scan_run(hm_scan *s, int64_t *plot, hm_scan_stats *stats);
int  hm_scan_run_path(hm_scan *s, int path, int64_t *plot, hm_scan_stats *stats);
int  hm_scan_is_symmetric(const hm_scan *s);
/* the pair list of extract_kmer_pairs for a pixel->smudge map (host uint16[HM_PLOT_CELLS]); *out is malloc'ed
 * (caller frees), sorted by (smudge, k-mer).  The route follows hm_scan_run's rule: on a table the fingerprint
 * found strand-symmetric (k >= HM_SYMM_MIN_KMER) the pairs are listed from the candidates of the last symmetric
 * run (hm_k_symm_extract, one launch per GPU and slice) -- a symmetric run is done first when the last run left
 * none with a clean status, and one that fails its checks falls back to the direct route; other tables take the
 * direct passes' results (the direct passes run first if the last run did not leave them).  HETMERS_PATH=
 * direct|symm forces a route as it does for a run (symm on a table that is not symmetric is an error).  Either
 * route gives the same list.  The symmetric route's record buffer on each GPU is what the device budget leaves
 * beyond the scan's arrays (HM_ENOMEM, before any launch, if that is less than HM_EXTRACT_MIN_BYTES); the
 * candidates pass through it in slices.  A streamed scan refuses (HM_EUNSUPPORTED).                          */
#define HM_EXTRACT_MIN_BYTES (2ll*HM_PLOT_CELLS + (1ll << 16))   /* device pixmap + 64 KiB of records */
int  hm_scan_extract(hm_scan *s, const uint16_t *pixmap, hm_pair_rec **out, int64_t *n_out);
/* ---- extract_kmer_pairs' pair files from an in-core scan on 1..G GPUs (DESIGN.md §6c) ----------------------
 * hm_scan_write_pairs writes what extract_kmer_pairs writes -- hm_scan_extract's list, one print_het line per
 * record, label s's lines in the file paths[s-1] -- without the records leaving the GPUs: a histogram sweep
 * counts the records per key prefix (the top min(HM_COND_HIST_BITS, 2k) bits of key_hi) on every GPU, the
 * prefixes are cut into windows as dist.pair_windows cuts them for world = G under the smallest room of the GPUs
 * (window j: pass j / G, GPU j mod G), and per pass every GPU lists its share of each window again from the scan
 * (into the owner's buffer, peer-copied at the offset the histograms give), the owner sorts, counts lines per
 * label and formats them, and one writer thread pwrites the text at its offsets.  The route follows
 * hm_scan_extract's rule.  The room of a GPU is the device budget (hm_set_device_budget, else the scan's) less
 * what the scan holds, the pixmap and counters, in records of hm_pairs_bytes' sort and format terms.  HM_ENOMEM
 * with the sizes when that room is below the fixed part or one prefix alone exceeds it: then no file has been
 * touched and st->planned is 0.  After the plan every label file is created or truncated; on any later failure
 * all of them are removed.  A streamed scan refuses (HM_EUNSUPPORTED), a scan left invalid by a failed
 * conditioning too (HM_EINVAL).  st is optional.                                                              */
typedef struct hm_pairs_stats
  { int64_t records;                        /* lines written, over every label                                */
    int64_t passes, windows;
    int64_t room;                           /* records one window may hold (the smallest room of the GPUs)    */
    int64_t peak_bytes;                     /* most device bytes held on one GPU beyond the scan's at the start */
    int64_t budget;                         /* device bytes the call may hold on a GPU beside the scan (least) */
    int32_t path;                           /* HM_PATH_SYMM or HM_PATH_DIRECT: the route the pairs came from   */
    int32_t planned;                        /* 1 once the plan fitted: an HM_ENOMEM is then not the plan's     */
    double  ms_hist;                        /* route, histogram sweep and plan                                */
    double  ms_list, ms_sort, ms_format;    /* window sweeps (with peer copies); sort + label bounds; format  */
    double  ms_d2h;                         /* the text to the pinned pieces                                  */
    double  ms_write;                       /* waiting for the writer thread (a piece, or the last ones)      */
    double  ms_writer_busy;                 /* the writer thread's pwrite time                                */
    double  ms_total;
  } hm_pairs_stats;
int  hm_scan_write_pairs(hm_scan *s, const uint16_t *pixmap, int n_labels, const char *const *paths,
                         hm_pairs_stats *st);
/* the histogram sweep alone, summed over the GPUs: hist (host uint64[2^min(HM_COND_HIST_BITS, 2k)]) = the
 * records of hm_scan_extract's list per key prefix, as hm_k_pairs_hist would count them                       */
int  hm_scan_pairs_hist(hm_scan *s, const uint16_t *pixmap, uint64_t *hist);
/* the plan of the pair files: the fewest passes P such that the prefixes of hist[0..np) cut into P * world
 * windows of near-equal record counts (cut r of W: the prefix boundary nearest to r/W of the total, the lower
 * one on a tie) leave every window within `room` records; cuts (NULL: only *passes) receives the P * world + 1
 * bounds.  HM_ENOMEM when one prefix alone holds more than room.  dist.pair_windows restates it in Python.      */
int  hm_pair_windows(const int64_t *hist, int64_t np, int world, int64_t room, int64_t *passes, int64_t *cuts);
/* ---- device budget and the streamed symmetric scan (DESIGN.md §4c) --------------------------------
 * hm_scan_create computes the bytes the in-core scan would allocate per GPU (table arrays, bucket index,
 * plot, fingerprint, hm_symm_plan(...).bytes).  When they exceed the device budget the scan is STREAMED:
 * nothing is loaded at create time, and every hm_scan_run passes the table through one GPU in run-aligned
 * chunks, keeping only the Bloom filter, the candidate records and the S list (keys with an upper
 * partner) resident.  A streamed scan needs the table strand-symmetric (else HM_EUNSUPPORTED after the
 * pass) and reads the host table again on every run: the hm_host_table given to hm_scan_create (its
 * buffers or descriptors) must stay valid until hm_scan_destroy.  Streamed scans refuse what needs the
 * whole table resident (HM_EUNSUPPORTED): hm_scan_condition, hm_scan_extract, hm_scan_download and
 * hm_scan_run_path(HM_PATH_DIRECT); hm_scan_examine streams (on dev[0]).
 * Several GPUs (n_gpus = G > 1): shard r streams [c_r, c_r+1) through dev[r], c_r = the first run start at
 * or after n*r/G (hm_symm_align_cut's rule; shards may be empty).  Every shard holds the whole-table Bloom
 * filter (its own segment filled by its pass 1, the others all-gathered), its own candidates and S list;
 * pass 2 checks a Bloom hit in the S list of the key's owner through peer memory.  A device id may repeat
 * in dev[] for a streamed scan: those shards share the device and the default budget (an in-core scan
 * refuses repeated ids).  The budget applies to each shard.
 * HETMERS_STREAM=1 streams scans whatever their size (the budget then only sizes the chunks);
 * HETMERS_STREAM_CHUNK=<entries> caps each shard's chunk length below what the budget allows.          */

/* device bytes a scan may hold per GPU; 0 (default) = what cudaMemGetInfo reports free at
 * hm_scan_create (plus the idle part of the memory pool) minus HM_BUDGET_RESERVE.  The executable passes
 * HETMERS_DEVICE_BUDGET=<bytes> here.                                                               */
#define HM_BUDGET_RESERVE (1ll << 30)
void hm_set_device_budget(int64_t bytes);

typedef struct hm_stream_layout            /* what hm_stream_plan chooses for a table under a budget      */
  { int64_t budget;
    int64_t chunk;                          /* entries per chunk buffer (grows if a run is longer)        */
    int64_t fixed_bytes;                    /* stub index, plot, fingerprint, header + Bloom filter        */
    int64_t chunk_bytes;                    /* two chunk buffers, their bucket index, run list, staging    */
    int64_t list_bytes;                     /* left for the resident candidate records and S list          */
    int64_t chunk_list_bytes;               /* list room one chunk may need at most                        */
  } hm_stream_layout;

/* the streamed scan's plan for n entries of k-mer length kmer (ibyte: the table's stub-index bytes);
 * fixed + chunk + list bytes <= budget, chunk is monotone in the budget; HM_ENOMEM if the budget cannot
 * hold one chunk                                                                                     */
int  hm_stream_plan(int64_t n, int kmer, int ibyte, int64_t budget, hm_stream_layout *out);
/* the plan of each of n_shards shards (budget per shard): fixed_bytes holds the whole-table Bloom filter of
 * n_shards segments, chunk and list room are for a share of ceil(n / n_shards) entries (chunks no longer
 * than the share).  n_shards = 1 is hm_stream_plan.                                                    */
int  hm_stream_plan_shards(int64_t n, int kmer, int ibyte, int64_t budget, int n_shards, hm_stream_layout *out);
/* 1 if the scan is streamed, else 0.  *device_bytes: the most device memory the scan held per GPU (in
 * core: what it allocates; streamed: the largest peak of a shard); *chunks: chunks of the last run, summed
 * over the shards (0 in core).  Either pointer may be NULL.                                           */
int  hm_scan_residency(const hm_scan *s, int64_t *device_bytes, int64_t *chunks);

/* ---- lists in host memory (DESIGN.md §4c, *Lists in host memory*) ----
 * A streamed run keeps its candidate records and S list on the device.  With a list host budget set (process-wide,
 * bytes; 0, the default, is off) a run whose lists cannot grow within the device budget moves them to host memory
 * instead of refusing: pass 1 flushes them to host arrays whenever they run out of room (and once more at its end),
 * and pass 2 uploads the candidates a slice at a time, parks every Bloom hit, and answers the round's queries
 * against the S list uploaded a partition at a time.  The device then holds the Bloom filter, one chunk and pass
 * 2's plan (hm_spill_plan); the lists' host bytes must stay within the budget (else HM_ENOMEM naming both sizes).
 * A run whose lists fit is unchanged.  With several shards in one process, one shard spilling makes every shard
 * spill.  The one-process-per-GPU ranks (hm_rank_scan_*) are not affected by it: each has its own list host budget
 * (hm_rank_scan_set_list_host_budget).  HETMERS_LIST_HOST_BUDGET=<bytes> sets it for the executables.          */
void hm_set_list_host_budget(int64_t bytes);

typedef struct hm_spill_stats               /* what the last run of a scan did with its lists                   */
  { int32_t spilled;                        /* 1 if the lists went to host memory                              */
    int32_t pad;
    int64_t flushes;                        /* pass 1 flushes, over the shards                                 */
    int64_t d2h_bytes;                      /* list bytes moved device -> host in pass 1                       */
    int64_t host_peak_bytes;                /* host bytes the lists held at most (every shard's)               */
    int64_t partitions;                     /* S partitions pass 2 walks                                       */
    int64_t rounds;                         /* pass 2 rounds, over the shards                                  */
    int64_t h2d_bytes;                      /* candidate slices and S partitions moved host -> device in pass 2 */
    int64_t slice, part;                    /* candidates per slice, S keys per partition (hm_spill_plan)      */
    int64_t first_key_queries;              /* partitions whose first key was queried, over rounds and shards  */
    double  ms_pass1, ms_flush, ms_pass2;   /* pass 1 (the slowest shard's chunk loop); its flushes (the slowest
                                               shard's); pass 2 (the slowest shard's rounds)                   */
  } hm_spill_stats;
int  hm_scan_spill_stats(const hm_scan *s, hm_spill_stats *out);

typedef struct hm_spill_layout              /* pass 2 of host lists in `room` device bytes                      */
  { int64_t room;
    int64_t slice;                          /* candidates per uploaded slice, and the round's pending slots     */
    int64_t queries;                        /* query slots: 2 per pending slot                                 */
    int64_t part;                           /* S keys per partition                                            */
    int32_t part_bits, pad;                 /* bucket index bits of a partition (hm_pick_bucket_bits(part))    */
    int64_t slice_bytes, part_bytes;        /* device bytes of the slice side and of the partition side        */
  } hm_spill_layout;
/* Pass 2's room arithmetic for n_cand candidates (the most of any shard) and an S list of n_s keys (every shard's).
 * Per slot of a slice: its record (8 KW + 8), a pending slot (8), two queries of 2 (8 KW + 8) + 1 bytes each and
 * their sort scratch (HM_SPILL_SORT_Q per query + HM_SPILL_SORT_FIXED); per partition key 8 KW, plus its uint32
 * bucket index.  Everything at full size if it fits; else the slice side takes at most half the room, the
 * partitions the most the rest holds, and the slice what they leave.  A slice holds at most HM_SPILL_MAX_SLICE
 * candidates (its 2 x that queries are sorted with 32-bit indices) and a partition at most HM_SPILL_MAX_PART keys
 * (its bucket index has 32-bit offsets).  HM_ENOMEM, with the sizes, when the room holds less than
 * min(n, HM_SPILL_MIN) of either.                                                                               */
#define HM_SPILL_MIN        1024
#define HM_SPILL_SORT_Q     32
#define HM_SPILL_SORT_FIXED (64ll << 10)
#define HM_SPILL_MAX_SLICE  0x3FFFFFF0ll
#define HM_SPILL_MAX_PART   0xFFFFFFEFll
int  hm_spill_plan(int64_t n_cand, int64_t n_s, int kmer, int64_t room, hm_spill_layout *out);

/* ---- one rank of a one-process-per-GPU job streaming a strand-symmetric table (DESIGN.md §4c, *Ranks*) ----
 * Rank `rank` of `world` streams its run-aligned share [c_rank, c_rank+1) (the cuts of the in-process shards)
 * through `device` under the device budget; no rank holds the table, and no call reads another rank's memory.
 * The caller runs the collectives between the calls (smudgeplot_b200/dist.py), in this order:
 *   create (seed: the same fingerprint seeds on every rank) -> cuts (the same on every rank)
 *   pass1 -> fingerprint sums summed over the ranks -> prepare(verdict) (an asymmetric table: HM_EUNSUPPORTED)
 *   -> the Bloom segments all-gathered in place (bloom) -> slices(the smallest max_slice of all ranks, capped
 *   by the largest candidate count) -> for every round up to the largest `rounds` of all ranks:
 *   route (counts[q] = queries for rank q) -> the key words all-to-all'ed from send into recv (KW = 1 word per
 *   query, 2 for k > 32) -> answer(keys received) -> the answers all-to-all'ed back from ans_recv into ans_sent
 *   -> settle; then result -> the partial plots summed over the ranks.
 * extract_kmer_pairs' list goes the same way from a prepared pass 1 (after prepare and the Bloom all-gather, or
 * after a finished scan or listing whose status words were clean on every rank; else pass1 ... bloom first):
 *   extract_prepare(pixmap) -> extract_slices(the smallest max_slice of all ranks, capped by the largest
 *   candidate count) -> for every round up to the largest `rounds` of all ranks: extract_route -> the key words
 *   all-to-all'ed as above -> answer -> the answers all-to-all'ed back -> extract_settle; then extract_result ->
 *   the ranks' records gathered on one rank and sorted there with hm_sort_pair_records.
 * Device pointers are returned; they stay valid until the next pass1, slices / extract_slices, extract_result
 * or destroy.
 * Lists in host memory (DESIGN.md §4c, *Lists in host memory*): with set_list_host_budget(bytes > 0) before
 * pass1, a rank whose lists cannot grow within its device budget flushes them to host memory in pass 1 (at most
 * `bytes` there, else HM_ENOMEM naming both sizes).  The caller then agrees one mode for the job: after pass1,
 * spill_stats().spilled on any rank -> host_lists() on every rank that did not spill -> prepare (no S index; its
 * max_slice from hm_rank_spill_plan) -> the Bloom all-gather; the rounds go as above with two differences: each
 * rank's queries include those it owns itself (counts[rank]), so recv holds world * 2 * slice keys and every
 * rank's split, its own included, is exchanged; and answer sorts the keys received, answers them against the
 * rank's S list uploaded a partition at a time, and returns the answers in receive order.  The host lists
 * live until the next pass1 or destroy, so a listing after a scan reuses them.                           */
typedef struct hm_rank_scan hm_rank_scan;
int  hm_rank_scan_create(const hm_host_table *t, int device, int rank, int world, const uint64_t seed[2],
                         hm_rank_scan **out);
/* create from the rank's share alone: `share` holds the entries [cuts[rank], cuts[rank+1]) of a table of n_total
 * entries (its ordinals start at 0, its stub index counts only them), and the caller gives every rank's cuts
 * (int64[world+1], 0 .. n_total, each on a run boundary) and first_keys (uint64[world]: word 0 of entry cuts[r],
 * ~0 when cuts[r] = n_total).  The scan is sized by the whole table, as create sizes it; hm_rank_scan_cuts
 * returns these cuts.                                                                                        */
int  hm_rank_scan_create_share(const hm_host_table *share, int64_t n_total, const int64_t *cuts,
                               const uint64_t *first_keys, int device, int rank, int world, const uint64_t seed[2],
                               hm_rank_scan **out);
void hm_rank_scan_destroy(hm_rank_scan *r);
/* cuts: int64[world+1]; first_keys (optional): uint64[world], word 0 of the first entry of each share */
int  hm_rank_scan_cuts(const hm_rank_scan *r, int64_t *cuts, uint64_t *first_keys);
/* fp: host uint64[4], the fingerprint sums of the entries this rank scanned */
int  hm_rank_scan_pass1(hm_rank_scan *r, uint64_t *fp);
/* world Bloom segments of seg_bytes each; segment q is rank q's */
int  hm_rank_scan_bloom(const hm_rank_scan *r, void **d_segments, int64_t *seg_bytes);
/* max_slice: the most candidates per round the budget leaves room for (HM_ENOMEM below 256) */
int  hm_rank_scan_prepare(hm_rank_scan *r, int symmetric, int64_t *n_cand, int64_t *max_slice);
int  hm_rank_scan_slices(hm_rank_scan *r, int64_t slice, int64_t *rounds, void **d_send, void **d_recv,
                         void **d_ans_recv, void **d_ans_sent);
int  hm_rank_scan_route(hm_rank_scan *r, int64_t round, int64_t *counts);
int  hm_rank_scan_answer(hm_rank_scan *r, int64_t n_received);
int  hm_rank_scan_settle(hm_rank_scan *r);
/* d_plot: device int64[HM_PLOT_CELLS], this rank's partial plot; status: non-zero = do not use the plot */
int  hm_rank_scan_result(hm_rank_scan *r, void **d_plot, uint64_t *status);
/* the most device bytes held since the last pass1 began, that pass's chunks, and the budget */
int  hm_rank_scan_residency(const hm_rank_scan *r, int64_t *device_bytes, int64_t *chunks, int64_t *budget);
/* pixmap: host uint16[HM_PLOT_CELLS], pixel -> smudge label (0 = none).  max_slice: the most candidates per
 * round the budget leaves room for beside the pixmap (HM_ENOMEM below 256, before any launch)             */
int  hm_rank_scan_extract_prepare(hm_rank_scan *r, const uint16_t *pixmap, int64_t *n_cand, int64_t *max_slice);
int  hm_rank_scan_extract_slices(hm_rank_scan *r, int64_t slice, int64_t *rounds, void **d_send, void **d_recv,
                                 void **d_ans_recv, void **d_ans_sent);
int  hm_rank_scan_extract_route(hm_rank_scan *r, int64_t round, int64_t *counts);
int  hm_rank_scan_extract_settle(hm_rank_scan *r);
/* this rank's records (*records malloc'ed, caller frees), sorted as hm_scan_extract sorts; status: non-zero = do
 * not use them.  Pass 1 stays resident for another extract_prepare.                                         */
int  hm_rank_scan_extract_result(hm_rank_scan *r, hm_pair_rec **records, int64_t *n, uint64_t *status);
/* the same records without the sort (the caller orders them, e.g. on the device: hm_k_pairs_sort) */
int  hm_rank_scan_extract_records(hm_rank_scan *r, hm_pair_rec **records, int64_t *n, uint64_t *status);
/* sort n records in place into hm_scan_extract's order: (smudge, key, position, alternative base) */
int  hm_sort_pair_records(hm_pair_rec *records, int64_t n);
/* host bytes this rank's lists may take from the next pass1 on (0, the default: they stay on the device) */
int  hm_rank_scan_set_list_host_budget(hm_rank_scan *r, int64_t bytes);
/* after pass1, when some rank of the job spilled and this one did not: its lists to host memory as well */
int  hm_rank_scan_host_lists(hm_rank_scan *r);
/* this rank's hm_spill_stats: pass 1's flushes since the last pass1, pass 2's rounds, partitions and bytes since
 * the last slices / extract_slices (ms_pass2: the time inside its route, answer and settle calls)          */
int  hm_rank_scan_spill_stats(const hm_rank_scan *r, hm_spill_stats *out);
/* The device plan of a rank's parked routed rounds, for n_cand candidates and an S list of n_s keys (the rank's)
 * in `room` bytes, world ranks, listing or counting.  Per slot of a slice: the slice side -- its record (8 KW +
 * 8), a pending slot (8), two queries (8 KW + 8 each), their send words and slots (8 KW + 4 each) and answers
 * (1 each), and when listing its parked key words (8 KW) and two records (2 x 24) -- and the receive side: world
 * x 2 keys, each received, sorted (8 KW apiece), with two sort permutations (8), its answer before and after the
 * scatter back (2) and its sort scratch (HM_SPILL_SORT_Q, plus HM_SPILL_SORT_FIXED once); HM_RANK_SPILL_FIXED
 * for the counters and allocation rounding.  Per partition key 8 KW plus its uint32 bucket index.  Split as
 * hm_spill_plan splits (slice and receive sides together); a slice holds at most HM_SPILL_MAX_SLICE / world
 * candidates (the world x 2 x slice keys received are sorted with 32-bit indices).  HM_ENOMEM, with the sizes,
 * when the room holds less than min(n, HM_SPILL_MIN) of either.  out->slice_bytes counts both sides.         */
#define HM_RANK_SPILL_FIXED (16ll*HM_MAX_SHARDS + 32*256)
int  hm_rank_spill_plan(int64_t n_cand, int64_t n_s, int kmer, int world, int listing, int64_t room,
                        hm_spill_layout *out);

/* ---- extract_kmer_pairs' pair files across the ranks of a one-process-per-GPU job (csrc/hm_pairs.cu, DESIGN.md
 * §6b; dist.ShardedScan / StreamedShardedScan.write_pairs).  The caller runs the collectives between the calls:
 *   pairs_hist over this rank's records (one uint64 per key prefix: the top min(HM_COND_HIST_BITS, 2k) bits of
 *   key_hi; zeroed by the caller) -> histograms summed over the ranks -> the prefixes cut into windows, window j
 *   going to pass j / world and rank j % world -> per pass, per staged chunk of records: d_dest (int16 per prefix:
 *   the rank owning it in this pass, -1 outside the pass) -> route_count -> route_scatter -> all-to-all -> on the
 *   owner: sort -> label_bounds -> format -> the text written at the offsets the line counts give.
 * d_counts / d_cursor: uint64[world] (world <= 64); route_count adds the records bound for each rank, route_scatter
 * places them from d_cursor[d] (preset to the start of rank d's segment, advanced here; any order inside a
 * segment) and sets *d_flag (zeroed by the caller) when a slot lies at or beyond cap.                        */
int hm_k_pairs_hist(const hm_pair_rec *d_rec, int64_t n, int kmer, uint64_t *d_hist, void *stream);
int hm_k_pairs_route_count(const hm_pair_rec *d_rec, int64_t n, int kmer, const int16_t *d_dest, int world,
                           uint64_t *d_counts, void *stream);
int hm_k_pairs_route_scatter(const hm_pair_rec *d_rec, int64_t n, int kmer, const int16_t *d_dest, int world,
                             uint64_t *d_cursor, hm_pair_rec *d_send, int64_t cap, uint64_t *d_flag, void *stream);
/* n records into hm_sort_pair_records' order through the double buffer (d_rec, d_alt); *in_alt: the result is in
 * d_alt.  Scratch: hm_pairs_sort_scratch_bytes(n) (a size query on the current device; 0 and the error set on
 * failure), HM_ENOMEM if less is given.                                                                       */
int64_t hm_pairs_sort_scratch_bytes(int64_t n);
int hm_k_pairs_sort(hm_pair_rec *d_rec, hm_pair_rec *d_alt, int64_t n, void *d_scratch, int64_t scratch_bytes,
                    int *in_alt, void *stream);
/* sorted records -> d_bounds[2s], d_bounds[2s+1] = first and one-past-last record of smudge s, for s <= n_labels
 * (uint64[2 (n_labels + 1)], zeroed by the caller)                                                            */
int hm_k_pairs_label_bounds(const hm_pair_rec *d_sorted, int64_t n, int n_labels, uint64_t *d_bounds, void *stream);
/* sorted records -> their print_het lines, k + 5 bytes each, at d_text (n (k + 5) bytes)                      */
int hm_k_pairs_format(const hm_pair_rec *d_sorted, int64_t n, int kmer, char *d_text, void *stream);
/* the most device bytes the file phase holds for a window of `records` records (arrays rounded to 512 bytes): the
 * histogram and destination map, 2 MiB of small arrays, and the largest of route (the window's records, a staged
 * chunk of records / 2 and its send buffer), sort (records twice, and 8 bytes per record + 1 MiB allowed for the
 * sort's scratch) and format (the sorted records and their text); -1 on bad arguments                          */
int64_t hm_pairs_bytes(int kmer, int64_t records);

/* ---- conditioning to table files, for tables of any size (csrc/hm_condition.cu, DESIGN.md §4d) ----
 * hm_scan_condition_files writes what hm_scan_condition + hm_scan_download would give -- the source's entries
 * with count >= ethresh (do_trim), plus every kept k-mer's reverse complement with the same count (do_symm),
 * sorted, the original winning where both are present -- as the FastK table `dst` (same kmer, ibyte and parts
 * as the source, parts cut on stub-index buckets).  It reads the table the scan was created from (that
 * hm_host_table must still be valid), in or out of core alike, on dev[0] (on several of the scan's GPUs: see
 * hm_set_condition_gpus), and leaves the scan as it was.  The
 * source passes through the GPU once to histogram the output by key prefix (HM_COND_HIST_BITS bits of the
 * first word), then once per key range of hm_condition_plan: each pass gathers the range's kept originals and
 * reverse complements, sorts the latter, merges (the steps hm_scan_condition takes in place), packs FastK
 * records and hands them to a host thread that
 * writes them while the next range is gathered.  The call's own device bytes stay within what the scan's
 * resident arrays leave of the budget set with hm_set_device_budget, or without one within what is free at the
 * call minus HM_BUDGET_RESERVE.  Refused before any file is
 * written: a scan conditioned in place (HM_EINVAL), a dst one of whose files is one of the source's part files
 * (HM_EINVAL; seen through the part descriptors hm_table_open keeps open -- smudgeplot_b200.hetmers.Scan checks
 * by name for the tables it reads), a budget below one range's smallest working set (HM_ENOMEM).                                                                */
/* GPUs hm_scan_condition_files runs on (process-wide; default 1: dev[0] alone, with one writer thread).  With
 * n > 1 it uses the first min(n, G) devices of the scan, dev[0..]: each histograms a contiguous slice of the source
 * (a streamed scan's through its own loader, an in-core scan's from its resident replica, so nothing crosses PCIe),
 * the plan is made once under the smallest budget of those GPUs, range r runs on GPU r mod G' (from the replica in
 * core, from the host table streamed), and each GPU's writer thread pwrites the range's records at their final
 * offsets (hm_table_write_place / _at) while later ranges are settled.  The files are byte-identical to n = 1's.
 * A device repeated in dev[] (a streamed scan) runs several of these shares, each under its own budget.  A
 * failure on any GPU stops them all; every thread is joined, every allocation freed, every file removed.     */
int  hm_set_condition_gpus(int n);         /* -> the value it replaces */
#define HM_COND_MAX_GPUS  16                /* hm_condition_stats.gpu_peak_bytes entries             */
#define HM_COND_HIST_BITS 20                /* output histogram: 2^min(20, 2k) key prefixes         */
#define HM_COND_MAX_RANGE (1ll << 31)       /* entries one range may hold                           */

typedef struct hm_condition_stats
  { int64_t nels_in, nels_out;
    int32_t ranges, passes;                 /* key ranges; passes over the source (ranges + 1)      */
    int64_t peak_bytes;                     /* most device bytes the call held (on one GPU)          */
    int64_t bytes_read, bytes_written;      /* source bytes sent H2D; table bytes written            */
    double  ms_hist, ms_ranges, ms_write, ms_total;   /* histogram pass; range passes (gather to pack); */
                                            /*   host time writing (overlaps the next range; summed */
                                            /*   over the writer threads); call                     */
    int64_t budget_bytes;                   /* the budget the call planned with: the one set less what */
                                            /*   the scan holds, or free memory less the reserve      */
                                            /*   (several GPUs: the smallest)                         */
    int32_t gpus, pad;                      /* GPUs the call ran on                                  */
    double  ms_write_max;                   /* the busiest writer thread's time                      */
    int64_t gpu_peak_bytes[HM_COND_MAX_GPUS];  /* peak_bytes of each GPU the call ran on             */
  } hm_condition_stats;

typedef struct hm_condition_layout         /* what hm_condition_plan chooses                            */
  { int64_t budget;
    int64_t chunk;                          /* source entries per loaded chunk                           */
    int64_t fixed_bytes;                    /* stub index, bucket counts, histogram, chunk + staging     */
    int64_t range_room;                     /* bytes a range's working set may take: 3/4 of the budget   */
                                            /*   minus the fixed part besides the chunk                  */
    int64_t range_cap;                      /* entries of the largest range                              */
    int64_t range_bytes;                    /* hm_condition_range_bytes(range_cap, ...)                  */
    int32_t n_ranges, hist_bits;
  } hm_condition_layout;

/* device bytes of a range of t output entries at most (kept originals + reverse complements): the region
 * both are gathered into and their FastK records; when symmetrising also the sort buffers (+ a uint32
 * permutation pair for k > 32), the sort scratch, the merged table and the merge's tile counts           */
int64_t hm_condition_range_bytes(int64_t t, int do_symm, int kmer, int ibyte);
/* Cut the 2^hist_bits key prefixes into ranges: cuts[0] = 0 < cuts[1] < ... < cuts[n_ranges] = 2^hist_bits
 * (cuts: room for 2^hist_bits + 1), greedily in key order, no range holding more than the entries whose
 * hm_condition_range_bytes fits range_room.  hist: kept originals + (do_symm) their reverse complements
 * per prefix.  HM_ENOMEM (with the sizes) if the fixed part or one prefix alone does not fit.             */
int hm_condition_plan(int64_t n, int kmer, int ibyte, int64_t budget, int do_symm, const int64_t *hist,
                      int hist_bits, int64_t *cuts, hm_condition_layout *out);
int hm_scan_condition_files(hm_scan *s, int ethresh, int do_trim, int do_symm, const char *dst,
                            hm_condition_stats *st);
/* hm_scan_condition_files into host memory instead of files: the same plan, the same range passes on the same
 * GPUs (hm_set_condition_gpus), and the table writer's memory target (hm_table_write_open_host), so *out holds
 * the records and stub index the files would hold, as one part (free it with hm_host_table_free; hm_scan_create
 * scans it in or out of core).  The buffer is sized by the output histogram, a bound on the records, and checked
 * against host_budget (-1: no cap) before the first range pass: HM_ENOMEM with both sizes when it does not fit,
 * or when it cannot be allocated.  The refusals of hm_scan_condition_files that concern no file stand (a scan
 * conditioned in place: HM_EINVAL; a device budget below one range's working set: HM_ENOMEM); on any failure
 * *out is NULL and nothing stays allocated.  st->bytes_written counts the host bytes (records and index).  The
 * scan is left as it was.                                                                                    */
int hm_scan_condition_host(hm_scan *s, int ethresh, int do_trim, int do_symm, int64_t host_budget,
                           hm_host_table **out, hm_condition_stats *st);

/* ---- conditioning across the ranks of a one-process-per-GPU job (csrc/hm_shard_condition.cu, DESIGN.md §4e) ----
 * Each rank holds a sorted share of the source (m entries; d_keys_lo only for k > 32) and the caller runs the
 * collectives between the calls (smudgeplot_b200/dist.py, ShardedScan.from_ktab(L=...)):
 *   cond_hist (one uint64 per key prefix, HM_COND_HIST_BITS bits of the first word or 2k if fewer; zeroed by the
 *   caller) -> histograms summed over the ranks -> the prefixes cut into one contiguous range per rank -> d_dest
 *   (int16 per prefix: the rank that owns it) -> route_count -> route_scatter -> the send buffer's two regions
 *   all-to-all'ed -> settle (when symmetrising) -> the ranks' shares concatenated in rank order.
 * ethresh: entries with count >= ethresh are kept (0 keeps all); do_symm: add every kept k-mer's reverse
 * complement with its count.  The results are those of hm_scan_condition, the original winning over an equal
 * reverse complement.                                                                                        */
int hm_k_cond_hist(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m, int kmer,
                   int ethresh, int do_symm, uint64_t *d_hist, void *stream);
/* d_counts: uint64[2*world + 2], zeroed by the caller -> [d]: kept originals bound for rank d, [world+d]: reverse
 * complements bound for rank d, [2*world]: all kept originals.  d_tiles: uint64[m/256 + 2] -> the kept
 * originals' offsets per tile of 256 entries, read by route_scatter.                                          */
int hm_k_shard_route_count(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m,
                           int kmer, int ethresh, int do_symm, const int16_t *d_dest, int world, uint64_t *d_counts,
                           uint64_t *d_tiles, void *stream);
/* the send buffer (n_orig + n_rc entries): [0, n_orig) the kept originals in source order (rank d's are the
 * slice after those of ranks below d), then from n_orig the reverse complements, rank d's segment starting at
 * d_cursor[d] (uint64[world], preset by the caller, advanced here; any order inside a segment).  *d_flag
 * (zeroed by the caller) becomes non-zero if an entry found no room.                                          */
int hm_k_shard_route_scatter(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m,
                             int kmer, int ethresh, int do_symm, const int16_t *d_dest, const uint64_t *d_tiles,
                             uint64_t *d_send_key, uint64_t *d_send_lo, uint16_t *d_send_cnt, int64_t n_orig,
                             int64_t n_rc, uint64_t *d_cursor, uint64_t *d_flag, void *stream);
/* received region: [0, n_orig) sorted originals, [n_orig, n_orig + n_rc) reverse complements in any order
 * (both are reordered here) -> d_out_* (room for n_orig + n_rc): the rank's conditioned share, *n_out entries
 * (synchronises the stream).  Scratch: hm_k_shard_settle_bytes(kmer, n_orig + n_rc, n_rc) bytes.  k > 32:
 * HM_EUNSUPPORTED from 2^32 - 16 reverse complements on (the sort carries a 32-bit permutation).           */
int64_t hm_k_shard_settle_bytes(int kmer, int64_t t, int64_t c);
int hm_k_shard_settle(int kmer, uint64_t *d_key, uint64_t *d_lo, uint16_t *d_cnt, int64_t n_orig, int64_t n_rc,
                      void *d_scratch, int64_t scratch_bytes, uint64_t *d_out_key, uint64_t *d_out_lo,
                      uint16_t *d_out_cnt, int64_t *n_out, void *stream);
/* the most device bytes one rank's conditioning holds (its arrays rounded to 512 bytes, plus 1 MiB for small
 * tensors): a share of `share` source entries unpacked (+ its records and the stub index of 2^(8 ibyte)
 * entries), routed into `sent` entries, `received` entries of which rc_received are reverse complements,
 * settled, and the replica of total_out entries gathered beside the rank's conditioned share; -1 on bad
 * arguments                                                                                                */
int64_t hm_shard_condition_bytes(int kmer, int ibyte, int world, int64_t share, int64_t sent, int64_t received,
                                 int64_t rc_received, int64_t total_out, int do_symm);

/* ---- conditioning across the ranks into new table files (dist.condition_ktab, DESIGN.md §4f) ----
 * The steps above in passes: in pass p, rank d owns the p-th sub-range (window) of its range of key prefixes, and
 * d_dest maps the prefixes of this pass's windows to their ranks and every other prefix to -1.  The _window route
 * calls take the arguments of the calls above; an entry (or reverse complement) whose prefix maps to -1 is neither
 * counted nor written, and the tile counts cover the in-window kept originals only.                          */
int hm_k_shard_route_count_window(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m,
                                  int kmer, int ethresh, int do_symm, const int16_t *d_dest, int world,
                                  uint64_t *d_counts, uint64_t *d_tiles, void *stream);
int hm_k_shard_route_scatter_window(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                                    int64_t m, int kmer, int ethresh, int do_symm, const int16_t *d_dest,
                                    const uint64_t *d_tiles, uint64_t *d_send_key, uint64_t *d_send_lo,
                                    uint16_t *d_send_cnt, int64_t n_orig, int64_t n_rc, uint64_t *d_cursor,
                                    uint64_t *d_flag, void *stream);
/* n sorted entries -> FastK records at d_rec (suffix bytes ibyte..kbyte-1, then the little-endian count: stride
 * kbyte - ibyte + 2) and d_bcount[b - b0] = the records in stub bucket b, for the nb buckets [b0, b0 + nb) that
 * must hold every entry (zeroed here).  Synchronises the stream.                                              */
int hm_k_cond_pack(int kmer, int ibyte, const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                   int64_t n, int64_t b0, int64_t nb, uint8_t *d_rec, uint64_t *d_bcount, void *stream);
/* The memory model of one rank: resident for the whole call, its share of `share` source entries unpacked (E =
 * 10 / 18 bytes per entry at k <= 32 / > 32) with its tile counts, the two histograms, the destination map, the
 * route counters, the stub-bucket counts and 1 MiB of small tensors; beside it the larger of the load (the share's
 * records and the stub index) and one pass -- route: `sent` entries; exchange: sent + `received`; settle (do_symm):
 * received twice and hm_k_shard_settle_bytes(kmer, received, rc_received); pack: received + their records.  Arrays
 * are rounded to 512 bytes, as torch's allocator rounds them.  -> the bytes of the pass (monotone in every count),
 * -1 on bad arguments.                                                                                        */
int64_t hm_rank_condition_bytes(int kmer, int ibyte, int world, int64_t share, int64_t sent, int64_t received,
                                int64_t rc_received, int do_symm);
/* Cut one rank's range of np key prefixes (hist: output entries per prefix, summed over the ranks) into
 * sub-ranges, greedily in key order: cuts[0] = 0 < ... < cuts[*n_sub] = np (cuts: room for np + 1; no sub-range
 * when np = 0), each of at
 * most HM_COND_MAX_RANGE entries and of at most the t entries whose pass, counted as sending and receiving t,
 * fits the budget beside the resident part.  HM_ENOMEM with the sizes when the load or one prefix alone does
 * not fit.                                                                                                    */
int hm_rank_condition_cut(int kmer, int ibyte, int world, int64_t share, int do_symm, int64_t budget,
                          const int64_t *hist, int64_t np, int64_t *cuts, int64_t *n_sub);

/* one call: create + run + destroy (what bench.py's e2e leg times) */
int  hm_hetmers_host(const hm_host_table *t, const int *dev, int n_gpus,
                     int64_t *plot, hm_scan_stats *stats);
/* copy device arrays back for tests: any pointer may be NULL */
int  hm_scan_download(hm_scan *s, uint64_t *keys, uint64_t *keys_lo, uint16_t *cnt, uint8_t *deg);

/* ======================= C. FastK table files (host, plain C) ============================ */

typedef struct hm_table hm_table;          /* parsed stub + mapped part payloads            */

/* Open <name>[.ktab] + hidden parts; replaces Open_Kmer_Stream (libfastk.c:786-908).
 * HM_EIO if the stub cannot be opened (the reference's "Cannot open k-mer table").          */
int  hm_table_open(const char *name, hm_table **out);
void hm_table_close(hm_table *t);
const hm_host_table *hm_table_view(const hm_table *t);

/* Incremental table writer: stub int32 kmer, nparts, minval, ibyte + int64 index[1 << 8*ibyte]; parts
 * ".<root>.ktab.<p>" with int32 kmer, int64 n (set on close).  Records (kbyte-ibyte suffix bytes, then a
 * little-endian uint16 count) come in table order; hm_table_write_buckets announces the buckets the next
 * records fill (counts[i] records for bucket b0+i; b0 at or after the last bucket announced, which it
 * continues).  Parts end where fastk.write_ktab(cut_on_buckets=True) ends them for a table of nels_hint
 * entries (byte-identical files when nels_hint is the exact count).  Files are written under temporary
 * names and renamed into place by hm_table_write_close (the stub last); a failure, or
 * hm_table_write_abort, leaves nothing under the final names.  close and abort free the writer.          */
typedef struct hm_table_writer hm_table_writer;
int  hm_table_write_open(const char *name, int kmer, int ibyte, int minval, int nparts, int64_t nels_hint,
                         hm_table_writer **out);
int  hm_table_write_buckets(hm_table_writer *w, int64_t b0, int64_t nb, const int64_t *counts);
int  hm_table_write_append(hm_table_writer *w, const uint8_t *rec, int64_t n);
int  hm_table_write_close(hm_table_writer *w);
void hm_table_write_abort(hm_table_writer *w);
/* Positional mode, instead of write_buckets + append (a writer takes one or the other): ranges of the table are
 * announced in table order with hm_table_write_place (counts[i] records for bucket b0+i, as write_buckets takes
 * them; *first = the range's first ordinal), and their records -- any slice, in any order, from any thread --
 * are written at their final offsets with hm_table_write_at(w, ordinal of rec[0], rec, n), a slice that crosses
 * a part cut going to both parts.  The parts are cut exactly as the append path cuts them, so the files are
 * byte-identical.  A cut is fixed once the bucket holding its ordinal is announced; records of the last bucket
 * announced can still belong to either side of a cut, so hm_table_write_at copies those (at most one bucket's)
 * and the place or hm_table_write_seal (no range follows; close seals too) that settles them writes them.  No
 * call waits for another.  Records not yet placed are an error (HM_EINVAL).                                  */
int  hm_table_write_place(hm_table_writer *w, int64_t b0, int64_t nb, const int64_t *counts, int64_t *first);
int  hm_table_write_at(hm_table_writer *w, int64_t first, const uint8_t *rec, int64_t n);
void hm_table_write_seal(hm_table_writer *w);
/* The same writer with host memory as its target: a one-part table of at most nels_cap records (HM_ENOMEM when
 * that buffer cannot be allocated; announcing more is an error, HM_EINVAL).  write_buckets / append, place / at /
 * seal and abort behave as they do for files; records are copied into one buffer at their final offsets and the
 * stub index is counted in memory.  hm_table_write_close_host closes it (hm_table_write_close refuses a memory
 * writer, and close_host a file writer; both free the writer either way): *out is a one-part table with the
 * given kmer, ibyte and minval whose records are the part files' payloads concatenated and whose index is the
 * stub's, byte for byte, for the same calls.  Free it with hm_host_table_free; on abort or failure nothing stays
 * allocated.                                                                                                  */
int  hm_table_write_open_host(int kmer, int ibyte, int minval, int64_t nels_cap, hm_table_writer **out);
int  hm_table_write_close_host(hm_table_writer *w, hm_host_table **out);
void hm_host_table_free(hm_host_table *t);     /* a table hm_table_write_close_host or hm_scan_condition_host made */

/* .smu writer: "min\t(sum-min)\tcount\n", sum-major, min < FMAX (PloidyPlot.c:1603-1617) */
int  hm_write_smu(const char *path, const int64_t *plot);

#ifdef __cplusplus
}
#endif
#endif

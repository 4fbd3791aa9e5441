/*******************************************************************************************
 * hm_symm.cu -- the strand-symmetric scan: every table entry is read ONCE.
 *
 * The reference insists on a table that holds the reverse complement of each of its k-mers with
 * the same count (examine_table, PloidyPlot.c:1199-1229; it runs `Symmex` otherwise, :1401-1414),
 * but then searches all k positions directly.  On a table that really is symmetric the pairs that
 * differ at a LOW position p < Pr = k/2 are the mirror images (u,v) -> (rc v, rc u) of the pairs
 * that differ at the HIGH position k-1-p, and pairs at high positions sit next to each other in the
 * sorted table: both members share their first Pr bases, i.e. lie in one short *run* of entries.
 * So with N_p(x) = number of partners of x at position p (count sum <= SMAX, PloidyPlot.c:259):
 *
 *     deg(x) = H(x) + U(rc x),   H(x) = sum_{p >= Pr}   N_p(x)     (found inside x's run)
 *                                U(x) = sum_{p >= k-Pr} N_p(x)     (ditto; = H without the middle
 *                                                                   base of an odd k)
 *     deg(rc x) = deg(x), and a pair and its mirror image land in the same plot cell.
 *
 *   symm_fingerprint_kernel   is the table symmetric?  Keyed multiset fingerprints of
 *                             {(x,cnt)} and {(rc x,cnt)} (seeds drawn per process); equal sums
 *                             <=> equal multisets up to a 2^-128 chance.  Tables that fail --
 *                             they may still pass the reference's one-k-mer probe -- take the
 *                             direct search of hm_kernels.cu, so the answer is the reference's
 *                             either way.
 *   runscan_kernel            ("pass 1") tiles of the sorted table are staged into shared memory by
 *                             TMA bulk copies; entries are classified by the adjacency of their
 *                             runs, runs of two are settled by one comparison (H, U, the partner),
 *                             runs of three to RS_RUNCAP entries from the same shared-memory window.
 *                             Entries with U > 0 (the set S) are added to a Bloom filter; pairs
 *                             (x < y) with H(x) = H(y) = 1 become candidate records.
 *   runs_kernel               the runs runscan_kernel only lists (longer than its window can hold)
 *   runscan_dense_kernel      pass 1 for crowded tables (many run mates per entry): all pairs of
 *                             every run, counted with shared-memory atomics
 *   resolve_kernel            ("pass 2") a candidate is an isolated pair iff neither rc x nor rc y
 *                             is in S: Bloom look-up (L2 resident), hits confirmed exactly by
 *                             scanning the run of rc x in the table.  Isolated pairs are counted
 *                             into the plot (shared-memory tile + 64-bit atomics), twice when the
 *                             mirror image is a different pair (PloidyPlot.c:401-415 sees both).
 *
 * Replaces analysis_in_core_1/_2 + the recursion around them (PloidyPlot.c:454-700,:851-1084)
 * for symmetric tables.  Traffic: keys + counts once (TBYTE per entry) + ~2 B per entry of
 * candidate records, instead of 2 x k merge levels in the reference.
 *******************************************************************************************/
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include "hetmers_b200.h"
#include "hm_internal.h"
#include "hm_device.cuh"

#define RS_THREADS 256
#define RS_EPT     8
#define RS_TILE    (RS_THREADS*RS_EPT)        /* entries per CTA tile                            */
#define RS_HALO    64                          /* entries staged on either side of the tile      */
#define RS_WIN     (RS_TILE+2*RS_HALO)
#define RS_SCANCAP RS_HALO                     /* longest run half scanned linearly               */
#define RS_RUNCAP  (RS_HALO+1)                 /* runscan_kernel settles runs of up to this many entries itself:
                                                *   a run whose head lies in the tile is then inside the window  */
#define RS_LONGRUN 32                          /* dense kernel: runs of more entries go to runs_kernel */
#ifndef RS_MINBLOCKS
#define RS_MINBLOCKS 6                         /* resident CTAs per SM the register budget must allow (40 regs, no
                                                *   spills; at k <= 32 six 34 KB windows fit in shared memory).  Each
                                                *   CTA waits on its window and on its step-5 atomic with all its
                                                *   warps, and a sixth CTA covers those waits: runscan_kernel at 2e8
                                                *   entries on one H100 SXM (700 W), 5: 1.027-1.032 ms, 6: 0.977-0.983
                                                *   (DESIGN.md §8)                                                    */
#endif
#ifndef RS_STAGE
#define RS_STAGE   384                         /* candidate records staged per CTA before they leave (a 2048-entry
                                                *   tile of a diploid 1 % table holds 184 +- 14)                    */
#endif

#define SY_STATUS_ASYMMETRIC 1ull              /* a reverse complement was not in the table      */
#define SY_STATUS_OVERFLOW   2ull              /* candidate list full                             */

/* The work area's header holds only counters, which the kernels advance atomically.  Words 0..2 are read by
 * hm_symm_status and tools/time_symm.py as well; hm_k_symm_runscan and hm_symm_stream_begin zero the header. */
#define SY_HDR_CAND   0                        /* candidate records                                */
#define SY_HDR_STATUS 1                        /* SY_STATUS_* bits                                 */
#define SY_HDR_RUNS   2                        /* runs listed for runs_kernel                      */
#define SY_HDR_S      3                        /* streamed scan: S list entries                    */
#define SY_HDR_PEND   4                        /* routed pass 2: parked candidates, then ...       */
#define SY_HDR_QUERY  5                        /*   ... their queries (both reset per round)       */

/* device view of the work area (hm_symm_layout) and of the arrays the streamed and routed scans add to it */
struct SymmView
  { unsigned long long *cand_n;                 /* header word SY_HDR_CAND: the header's first word */
    unsigned long long *status;
    uint32_t *bloom;                            /* n_seg segments of seg_words words               */
    uint32_t  seg_words;
    int       n_seg, self;
    uint64_t  first_key[HM_MAX_SHARDS];         /* word 0 of the first key of segments 1.. (0 unused) */
    uint64_t *cand_key, *cand_lo, *cand_meta;
    unsigned long long cand_cap;
    unsigned long long *runs_n;                 /* heads of runs of three or more entries (table indices) */
    uint64_t *runs;
    unsigned long long runs_cap;
    uint64_t *s_key, *s_lo;                     /* streamed pass 1: the S list (count: header word SY_HDR_S) */
    unsigned long long s_cap;
    const hm_stream_sview *sviews;              /* streamed pass 2, several shards: every shard's S list */
    uint64_t *pend, *pend_key, *pend_lo;        /* routed pass 2: parked candidates (meta; key words for listing) */
    uint64_t *q_key, *q_lo, *q_tag;             /*   and their queries (tag = owner << 32 | pending slot) */
    unsigned long long pend_cap, q_cap;
  };

/* Bloom slot of key (hi,lo).  The 64-bit WORD is chosen by the key's last k/2 bases, the three BITS inside it by
 * the bases before them: rc x and rc y of a candidate pair differ at one base of the front part only, so
 * both of pass 2's look-ups for a pair fall into the same word -- one load (when one shard owns both).  At the
 * filter's ~6 bits per element of S that is 7.1 % false positives per look-up, against 9.1 % for 2 bits in a
 * 32-bit word, with the same one atomic per insert (DESIGN.md §4a, tools/bloom_layout_model.py).            */
template <int KW>
__device__ __forceinline__ void bloom_slot(const SymmView &W, int seg, int kmer, uint64_t hi, uint64_t lo,
                                           uint64_t *&word, uint64_t &mask)
{ const int Pr = kmer >> 1, pup = kmer-Pr;
  uint64_t sfx;                                                /* the last Pr bases, right aligned */
  if (KW == 1)
    sfx = hi >> (64-2*kmer);
  else
    { const int sr = 128-2*kmer;                               /* 0..62 */
      sfx = sr == 0 ? lo : ((lo >> sr) | (hi << (64-sr)));
    }
  if (2*Pr < 64)
    sfx &= (((uint64_t) 1 << (2*Pr)) - 1);
  const uint64_t pfx = hi >> (64-2*pup);                       /* the first pup <= 32 bases */
  uint32_t h = ((uint32_t) sfx ^ (uint32_t) (sfx >> 32) * 0x85EBCA6Bu) * 0x9E3779B1u;     /* 32-bit mixing is plenty here */
  uint32_t g = ((uint32_t) pfx ^ (uint32_t) (pfx >> 32) * 0xC2B2AE35u) * 0x27D4EB2Fu;
  h ^= h >> 15;
  word = (uint64_t *) (W.bloom + (size_t) seg * W.seg_words) + __umulhi(h * 0x2C1B3C6Du,W.seg_words >> 1);
  mask = (1ull << (g >> 26)) | (1ull << ((g >> 20) & 63)) | (1ull << ((g >> 14) & 63));
}

/* L2 residency: the Bloom segments (tens of MB) are what pass 2 hits at random, the candidate records
 * stream through once                                                                             */
__device__ __forceinline__ uint64_t ld_keep(const uint64_t *p)
{ uint64_t v, pol;
  asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}

__device__ __forceinline__ uint64_t ld_stream(const uint64_t *p)
{ uint64_t v, pol;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u64 %0, [%1], %2;" : "=l"(v) : "l"(p), "l"(pol));
  return v;
}

/* *p |= v as a reduction (SASS REDG), which returns nothing to the SM.  atomicOr with its result unused
 * compiled to an ATOMG into RZ in the pass-1 kernels, whose old word L2 still sends back: the Bloom inserts
 * as ATOMGs cost runscan_kernel 0.05 ms at 2e8 entries, as REDGs nothing measurable (DESIGN.md §8)      */
__device__ __forceinline__ void red_or64(uint64_t *p, uint64_t v)
{ asm volatile("red.global.relaxed.gpu.or.b64 [%0], %1;" :: "l"(__cvta_generic_to_global(p)), "l"(v) : "memory"); }

__device__ __forceinline__ int owner_of(const SymmView &W, uint64_t hi)
{ int r = 0;
  for (int s = 1; s < W.n_seg; s++)
    r += (hi >= W.first_key[s]);
  return r;
}

/* all partners of x at positions >= p0, one bucket look-up per candidate (long runs only) */
template <typename IdxT, int KW>
__device__ __noinline__ void neighbours_slow(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                                             const uint16_t *__restrict__ cnt, const IdxT *__restrict__ bucket,
                                             int bshift, int kmer, int p0, int pup,
                                             uint64_t x, uint64_t xl, int cx,
                                             int &H, int &U, int64_t &part, int &ppos)
{ H = 0; U = 0; part = -1; ppos = 0;
  for (int p = p0; p < kmer; p++)
    { int b = base_at<KW>(x,xl,p);
      for (int c = 0; c < 4; c++)
        { if (c == b) continue;
          uint64_t y = x, yl = xl;
          set_base<KW>(y,yl,p,c);
          int64_t j = bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,y,yl);
          if (j >= 0 && cx + (int) __ldg(cnt+j) <= HM_SMAX)
            { H += 1;
              if (p >= pup) U += 1;
              part = j; ppos = p;
            }
        }
    }
}

/* ------------------------------------------------------------------- fingerprint -------- */

__device__ __forceinline__ uint64_t fp_mix(uint64_t hi, uint64_t lo, uint32_t c, uint64_t seed)
{ uint64_t v = (hi ^ seed) * 0xBF58476D1CE4E5B9ull;
  v ^= v >> 32;
  v = (v + lo + ((uint64_t) c << 40) + c) * 0x94D049BB133111EBull;
  v ^= v >> 29;
  v *= (seed | 1);
  v ^= v >> 32;
  return v;
}

template <int KW>
__global__ void __launch_bounds__(256)
symm_fingerprint_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                        const uint16_t *__restrict__ cnt, int64_t i0, int64_t i1, int kmer,
                        uint64_t seed0, uint64_t seed1, unsigned long long *__restrict__ acc)
{ uint64_t a0 = 0, a1 = 0, a2 = 0, a3 = 0;
  const int64_t stride = (int64_t) gridDim.x * blockDim.x;
  for (int64_t i = i0 + (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < i1; i += stride)
    { uint64_t x = keys[i], xl = KW == 2 ? keys_lo[i] : 0, r, rl;
      uint32_t c = cnt[i];
      revcomp_kmer<KW>(x,xl,kmer,r,rl);
      a0 += fp_mix(x,xl,c,seed0);  a1 += fp_mix(x,xl,c,seed1);
      a2 += fp_mix(r,rl,c,seed0);  a3 += fp_mix(r,rl,c,seed1);
    }
  for (int o = 16; o > 0; o >>= 1)
    { a0 += __shfl_xor_sync(0xffffffffu,a0,o); a1 += __shfl_xor_sync(0xffffffffu,a1,o);
      a2 += __shfl_xor_sync(0xffffffffu,a2,o); a3 += __shfl_xor_sync(0xffffffffu,a3,o);
    }
  if ((threadIdx.x & 31) == 0)
    { atomicAdd(acc+0,(unsigned long long) a0); atomicAdd(acc+1,(unsigned long long) a1);
      atomicAdd(acc+2,(unsigned long long) a2); atomicAdd(acc+3,(unsigned long long) a3);
    }
}

extern "C" int hm_k_symm_fingerprint(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                                     int64_t i0, int64_t i1, int kmer, const uint64_t seed[2],
                                     uint64_t *d_acc, void *stream)
{ if (kmer < 1 || kmer > HM_MAX_KMER || (kmer > 32) != (d_keys_lo != NULL) || seed == NULL || d_acc == NULL)
    return hm_set_error(HM_EINVAL,"symm_fingerprint: bad arguments (k=%d)",kmer);
  if (i1 <= i0)
    return HM_OK;
  int64_t want = (i1-i0+255)/256;
  int     grid = (int) (want < 132*16 ? want : 132*16);
  if (kmer <= 32)
    symm_fingerprint_kernel<1><<<grid,256,0,(cudaStream_t) stream>>>
        (d_keys,NULL,d_cnt,i0,i1,kmer,seed[0],seed[1],(unsigned long long *) d_acc);
  else
    symm_fingerprint_kernel<2><<<grid,256,0,(cudaStream_t) stream>>>
        (d_keys,d_keys_lo,d_cnt,i0,i1,kmer,seed[0],seed[1],(unsigned long long *) d_acc);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"symm_fingerprint_kernel");
  return HM_OK;
}

/* per-process seeds of the fingerprint (the table cannot have been chosen against them) */
extern "C" void hm_symm_seeds(uint64_t seed[2])
{ static uint64_t s[2] = {0,0};
  static int have = 0;
  if (!have)
    { FILE *f = fopen("/dev/urandom","rb");
      if (f == NULL || fread(s,sizeof(uint64_t),2,f) != 2)
        { struct timespec ts;
          clock_gettime(CLOCK_REALTIME,&ts);
          s[0] = 0x9E3779B97F4A7C15ull * (uint64_t) ts.tv_nsec ^ (uint64_t) ts.tv_sec;
          s[1] = 0xD1B54A32D192ED03ull * (uint64_t) (uintptr_t) &ts ^ ((uint64_t) ts.tv_nsec << 17);
        }
      if (f != NULL) fclose(f);
      have = 1;
    }
  seed[0] = s[0]; seed[1] = s[1];
}

/* ------------------------------------------------------------------------ layout -------- */

extern "C" int hm_symm_plan(int64_t n, int64_t range, int kmer, int n_seg, hm_symm_layout *out)
{ if (out == NULL || n < 0 || range < 0 || range > n || n_seg < 1 || n_seg > HM_MAX_SHARDS)
    return hm_set_error(HM_EINVAL,"hm_symm_plan: bad arguments");
  int bits = 1;                                  /* Bloom bits per table entry (S is ~1/6 of the table; three bits of one
                                                  *   64-bit word set per element, bloom_slot): 25 MB at 2e8 entries, which the access-policy window
                                                  *   (bloom_window) can keep in the H100's 50 MB L2.  2 bits (50 MB) halve
                                                  *   the exact checks of pass 2 but no longer fit: on one H100 SXM
                                                  *   (400 W) pass 1 took 2.98 ms with 2 bits against 1.53 ms with 1,
                                                  *   pass 2 0.75 against 0.81 ms.  Several GPUs: the segments also cross
                                                  *   NVLink between the kernels, one more reason to keep them small     */
  const char *e = getenv("HETMERS_BLOOM_BITS");
  if (e != NULL && atoi(e) >= 1 && atoi(e) <= 64)
    bits = atoi(e);
  int64_t per = (n+n_seg-1)/n_seg;               /* every segment the same size on every rank: all-gather friendly */
  int64_t segw = (per*bits+31)/32;
  if (segw < 1024) segw = 1024;
  segw = (segw+63) & ~63ll;
  if (segw > 0x7fffffffll)
    return hm_set_error(HM_EUNSUPPORTED,"Bloom segment of %lld words too large",(long long) segw);
  int64_t cap = range/2 + 1024;
  int64_t at = 0;
  memset(out,0,sizeof(*out));
  out->off_header = at;  at += 256;
  out->off_bloom = at;   at += 4*segw*n_seg;
  out->seg_words = segw;
  at = (at+255) & ~255ll;
  out->off_cand_key = at;   at += 8*cap;
  out->off_cand_lo = at;    at += (kmer > 32) ? 8*cap : 0;
  out->off_cand_meta = at;  at += 8*cap;
  out->cand_cap = cap;
  out->off_runs = at;       out->runs_cap = range/3 + 1024;   at += 8*out->runs_cap;
  out->n_seg = n_seg;
  out->range = range;
  out->bytes = (at+255) & ~255ll;
  return HM_OK;
}

/* L2 residency of the Bloom segments for the kernels launched on `st` from here on: an access-policy window
 * marks the filter "persisting" (its read-modify-writes in pass 1 and its look-ups in pass 2 then hit L2
 * although 2 GB of table stream through next to them).  on = 0 lifts the window again.                   */
static void bloom_window(cudaStream_t st, const void *base, size_t bytes, int on)
{ static int limit_set[64] = {0};
  static size_t max_win[64] = {0}, max_persist[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) return;
  if (!limit_set[dev])
    { cudaDeviceProp p;
      limit_set[dev] = 1;
      if (cudaGetDeviceProperties(&p,dev) == cudaSuccess)
        { max_win[dev] = (size_t) p.accessPolicyMaxWindowSize;
          max_persist[dev] = (size_t) p.persistingL2CacheMaxSize;
          if (max_persist[dev] > 0)
            cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize,max_persist[dev]);
        }
      cudaGetLastError();
    }
  if (max_win[dev] == 0 || max_persist[dev] == 0)
    return;
  cudaStreamAttrValue a;
  memset(&a,0,sizeof(a));
  if (on)
    { size_t w = bytes < max_win[dev] ? bytes : max_win[dev];
      a.accessPolicyWindow.base_ptr  = (void *) base;
      a.accessPolicyWindow.num_bytes = w;
      a.accessPolicyWindow.hitRatio  = w <= max_persist[dev] ? 1.0f : (float) max_persist[dev] / (float) w;
      a.accessPolicyWindow.hitProp   = cudaAccessPropertyPersisting;
      a.accessPolicyWindow.missProp  = cudaAccessPropertyStreaming;
    }
  cudaStreamSetAttribute(st,cudaStreamAttributeAccessPolicyWindow,&a);
  cudaGetLastError();
}

static int l2_persist(void)                    /* HETMERS_L2_PERSIST=0 switches the window off */
{ const char *e = getenv("HETMERS_L2_PERSIST");
  return (e == NULL || strcmp(e,"0") != 0);
}

static SymmView make_view(void *d_work, const hm_symm_layout *L, const hm_symm_shards *sh)
{ SymmView W;
  uint8_t *b = (uint8_t *) d_work;
  memset(&W,0,sizeof(W));
  W.cand_n    = (unsigned long long *) (b + L->off_header) + SY_HDR_CAND;
  W.status    = W.cand_n + SY_HDR_STATUS;
  W.bloom     = (uint32_t *) (b + L->off_bloom);
  W.seg_words = (uint32_t) L->seg_words;
  W.n_seg     = L->n_seg;
  W.self      = 0;
  if (sh != NULL && sh->n_seg > 1)
    { W.self = sh->self;
      for (int r = 0; r < sh->n_seg; r++) W.first_key[r] = sh->first_key[r];
    }
  W.cand_key  = (uint64_t *) (b + L->off_cand_key);
  W.cand_lo   = (uint64_t *) (b + L->off_cand_lo);
  W.cand_meta = (uint64_t *) (b + L->off_cand_meta);
  W.cand_cap  = (unsigned long long) L->cand_cap;
  W.runs_n    = W.cand_n + SY_HDR_RUNS;
  W.runs      = (uint64_t *) (b + L->off_runs);
  W.runs_cap  = (unsigned long long) L->runs_cap;
  return W;
}

/* ------------------------------------------------------------------------ pass 1 -------- */

/* shared-memory views of one CTA's window + its staging areas */
template <int KW> struct RsSmem
  { uint64_t *key, *klo;                /* window: RS_WIN slots (+1 spare)                        */
    uint16_t *cnt;
    uint64_t *ckey, *clo, *cmeta;       /* staged candidate records: RS_STAGE                     */
    uint16_t *t1;                       /* per warp: heads of runs of two, then of longer runs (RS_TILE/2 in all) */
    uint16_t *t2r;                      /* CTA: heads of runs left to runs_kernel                  */
  };

__device__ __forceinline__ uint64_t pack_meta(int cx, int cy, int pos, int yb)
{ return (uint64_t) cx | ((uint64_t) cy << 16) | ((uint64_t) pos << 32) | ((uint64_t) yb << 40); }

/* Probe build only: the mode tools/time_runscan_phases.py sets (see the probe block before runscan_kernel).
 * RS_PROBE_IS(m) is a constant false in the default build, so the hooks below compile to nothing there. */
#ifdef RS_PROBE
__device__ int rs_probe_mode;
#define RS_PROBE_IS(m) (rs_probe_mode == (m))
#else
#define RS_PROBE_IS(m) false
#endif

/* candidate records into the CTA's staging area (warp-wide call; `emit` per lane): one shared atomic for
 * all the lanes that emit; lanes that find the staging area full
 * go to the list directly, again with one (global) atomic for all of them                              */
template <int KW>
__device__ __forceinline__ void stage_candidates(const RsSmem<KW> &S, unsigned *s_nc, const SymmView &W,
                                                 bool emit, uint64_t x, uint64_t xl, uint64_t meta,
                                                 int lane, unsigned lt)
{ const unsigned bal = __ballot_sync(0xffffffffu,emit);
  if (bal == 0 || RS_PROBE_IS(4))                      /* probe no-stage: nothing is staged */
    return;
  unsigned base = 0;
  if (lane == 0)
    base = atomicAdd(s_nc,(unsigned) __popc(bal));
  base = __shfl_sync(0xffffffffu,base,0);
  const unsigned at = base + __popc(bal & lt);
  const bool     over = emit && (at >= RS_STAGE);
  if (emit && !over)
    { S.ckey[at] = x;
      if (KW == 2) S.clo[at] = xl;
      S.cmeta[at] = meta;
    }
  if (base + __popc(bal) <= RS_STAGE)                  /* (warp-uniform) nobody overflowed */
    return;
  const unsigned ob = __ballot_sync(0xffffffffu,over);
  unsigned long long g0 = 0;
  if (lane == 0)
    g0 = atomicAdd(W.cand_n,(unsigned long long) __popc(ob));
  g0 = __shfl_sync(0xffffffffu,g0,0) + (unsigned long long) __popc(ob & lt);
  if (over)
    { if (g0 < W.cand_cap)
        { W.cand_key[g0] = x;
          if (KW == 2) W.cand_lo[g0] = xl;
          W.cand_meta[g0] = meta;
        }
      else
        atomicOr(W.status,SY_STATUS_OVERFLOW);
    }
}

/* streamed scan (SL = true): every key that goes into the Bloom filter is also appended to the S list of the
 * view, so that the list is exactly the set the filter over-approximates; one atomic per warp.              */
template <int KW>
__device__ __forceinline__ void s_push(const SymmView &W, uint64_t x, uint64_t xl)
{ const unsigned m = __activemask();
  const int      lane = threadIdx.x & 31, lead = __ffs(m)-1;
  unsigned long long at = 0;
  if (lane == lead)
    at = atomicAdd(W.cand_n + SY_HDR_S,(unsigned long long) __popc(m));
  at = __shfl_sync(m,at,lead) + (unsigned long long) __popc(m & ((1u << lane)-1));
  if (at < W.s_cap)
    { W.s_key[at] = x;
      if (KW == 2) W.s_lo[at] = xl;
    }
  else
    atomicOr(W.status,SY_STATUS_OVERFLOW);
}

template <int KW, bool SL>
__device__ __forceinline__ void bloom_insert(const SymmView &W, int kmer, uint64_t x, uint64_t xl)
{ uint64_t *word, mask;
  bloom_slot<KW>(W,W.self,kmer,x,xl,word,mask);
  if (!RS_PROBE_IS(3) || mask == (uint64_t) (uintptr_t) word)   /* probe no-RED: the slot is computed (the test reads */
    red_or64(word,mask);                                        /*   it and never holds), the RED not issued */
  if (SL)
    s_push<KW>(W,x,xl);
}

/* Step 5 of the pass-1 kernels, after a CTA barrier: the staged records leave with one global atomic per CTA
 * and list (one per record, or per warp, on the one list counter serialises in L2), and every thread moves
 * at most RS_FLUSH of them.  flush_reserve issues thread 0's atomics and, while they are under way, reads
 * the thread's records from shared memory into F; after a second barrier flush_store writes them and the
 * run heads (rare) to the lists.                                                                           */
#define RS_FLUSH ((RS_STAGE+RS_THREADS-1)/RS_THREADS)
struct RsFlush { uint64_t key[RS_FLUSH], lo[RS_FLUSH], meta[RS_FLUSH]; };

template <int KW>
__device__ __forceinline__ void flush_reserve(const RsSmem<KW> &S, unsigned long long *s_cb,
                                              unsigned long long *s_rb, const SymmView &W,
                                              unsigned nc, unsigned nr, RsFlush &F)
{ if (threadIdx.x == 0)
    { if (nc > 0) *s_cb = atomicAdd(W.cand_n,(unsigned long long) nc);
      if (nr > 0) *s_rb = atomicAdd(W.runs_n,(unsigned long long) nr);
    }
#pragma unroll
  for (int j = 0; j < RS_FLUSH; j++)
    { const unsigned i = threadIdx.x + j*RS_THREADS;
      if (i < nc)
        { F.key[j] = S.ckey[i];
          if (KW == 2) F.lo[j] = S.clo[i];
          F.meta[j] = S.cmeta[i];
        }
    }
}

template <int KW>
__device__ __forceinline__ void flush_store(const RsSmem<KW> &S, unsigned long long cb, unsigned long long rb,
                                            const SymmView &W, unsigned nc, unsigned nr, int64_t T0,
                                            const RsFlush &F)
{
#pragma unroll
  for (int j = 0; j < RS_FLUSH; j++)
    { const unsigned i = threadIdx.x + j*RS_THREADS;
      if (i < nc)
        { if (cb+i < W.cand_cap)
            { W.cand_key[cb+i] = F.key[j];
              if (KW == 2) W.cand_lo[cb+i] = F.lo[j];
              W.cand_meta[cb+i] = F.meta[j];
            }
          else
            atomicOr(W.status,SY_STATUS_OVERFLOW);
        }
    }
  for (unsigned i = threadIdx.x; i < nr; i += RS_THREADS)
    if (rb+i < W.runs_cap)
      W.runs[rb+i] = (uint64_t) (T0 + ((int) S.t2r[i] - RS_HALO));
    else
      atomicOr(W.status,SY_STATUS_OVERFLOW);
}

/* Pass 1b: the runs runscan_kernel only lists -- more than RS_RUNCAP entries (or runs that may reach
 * past its window), and on crowded tables the runs runscan_dense_kernel leaves (more than RS_LONGRUN):
 * repeats, low-complexity sequence, tiny k.  The listed count is only known on the device, so the grid
 * is at most one wave and strides over the list.  Each warp takes its lanes' runs one after the other,
 * straight from global memory (the keys of a run are neighbours in the table): one member per lane and
 * trip, with one bucket look-up per candidate partner (neighbours_slow).                              */
template <typename IdxT, int KW, bool SL>
__global__ void __launch_bounds__(256)
runs_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
            const uint16_t *__restrict__ cnt, int64_t n, const IdxT *__restrict__ bucket, int bshift,
            int kmer, int64_t lo, int64_t hi, const SymmView W)
{ const int      Pr = kmer >> 1, pup = kmer-Pr, psh = 64-2*Pr;
  const uint64_t pmask = ~(uint64_t) 0 << psh;
  const unsigned FULL = 0xffffffffu;
  const int      lane = threadIdx.x & 31;
  const unsigned lt   = (1u << lane) - 1;
  unsigned long long nrl = *W.runs_n;
  if (nrl > W.runs_cap) nrl = W.runs_cap;
  const int64_t nr     = (int64_t) nrl;
  const int64_t stride = (int64_t) gridDim.x * blockDim.x;
  for (int64_t r0 = (int64_t) blockIdx.x * blockDim.x + threadIdx.x - lane; r0 < nr; r0 += stride)
    { const int64_t r = r0+lane;
      const bool    valid = (r < nr);
      int64_t  h = 0;
      uint64_t x0 = 0;
      if (valid)
        { h  = (int64_t) W.runs[r];
          x0 = __ldg(keys+h);
        }
      unsigned lb = __ballot_sync(FULL,valid);
      while (lb != 0)
        { const int     src = __ffs(lb)-1;
          lb &= lb-1;
          const int64_t hh = __shfl_sync(FULL,h,src);
          const uint64_t xx = __shfl_sync(FULL,x0,src);
          int64_t end = hh+1;
          while (true)
            { const int64_t t = end+lane;
              const bool same = (t < n) && (((__ldg(keys+t) ^ xx) & pmask) == 0);
              const unsigned sb = __ballot_sync(FULL,same);
              if (sb == FULL) { end += 32; continue; }
              end += __ffs(~sb)-1;
              break;
            }
          for (int64_t g0 = hh; g0 < end; g0 += 32)
            { const int64_t g = g0+lane;
              bool     emit = false;
              uint64_t x = 0, xl = 0, meta = 0;
              if (g < end && g >= lo && g < hi)
                { x = __ldg(keys+g);
                  if (KW == 2) xl = __ldg(keys_lo+g);
                  const int cx = __ldg(cnt+g);
                  int Hn, Un, ppos; int64_t part;
                  neighbours_slow<IdxT,KW>(keys,keys_lo,cnt,bucket,bshift,kmer,Pr,pup,x,xl,cx,Hn,Un,part,ppos);
                  if (Un > 0)
                    bloom_insert<KW,SL>(W,kmer,x,xl);
                  if (Hn == 1 && part > g)
                    { const uint64_t y = __ldg(keys+part), yl = KW == 2 ? __ldg(keys_lo+part) : 0;
                      const int cy = __ldg(cnt+part);
                      int Hy, Uy, py; int64_t party;
                      neighbours_slow<IdxT,KW>(keys,keys_lo,cnt,bucket,bshift,kmer,Pr,pup,y,yl,cy,Hy,Uy,party,py);
                      if (Hy == 1)
                        { emit = true;
                          meta = pack_meta(cx,cy,ppos,base_at<KW>(y,yl,ppos));
                        }
                    }
                }
              const unsigned eb = __ballot_sync(FULL,emit);
              if (eb != 0)
                { unsigned long long base = 0;
                  if (lane == 0)
                    base = atomicAdd(W.cand_n,(unsigned long long) __popc(eb));
                  base = __shfl_sync(FULL,base,0) + (unsigned long long) __popc(eb & lt);
                  if (emit)
                    { if (base < W.cand_cap)
                        { W.cand_key[base] = x;
                          if (KW == 2) W.cand_lo[base] = xl;
                          W.cand_meta[base] = meta;
                        }
                      else
                        atomicOr(W.status,SY_STATUS_OVERFLOW);
                    }
                }
            }
        }
    }
}

/* runscan_kernel's pair test inside a run.  The members of a run share their first Pr = k/2 bases, so two
 * of them differ only in the last k-Pr: 2(k-Pr) <= 32 bits for k <= 32, <= 64 bits for k <= 64.  run_sfx
 * puts those bases left aligned into one word of RunSfx<KW>::T (of x ^ y: the xor of the two suffixes), and
 * one_base_in_run tests that word and gives the same pos as one_base_apart on the whole keys.          */
template <int KW> struct RunSfx    { typedef uint64_t T; };
template <>       struct RunSfx<1> { typedef uint32_t T; };

template <int KW>
__device__ __forceinline__ typename RunSfx<KW>::T run_sfx(uint64_t hi, uint64_t lo, int Pr)
{ if constexpr (KW == 1)
    return (uint32_t) ((hi << 2*Pr) >> 32);                       /* Pr <= 16 */
  else
    return (hi << (2*Pr-32) << 32) | (lo >> (64-2*Pr));            /* 16 <= Pr <= 32 */
}

template <typename T>
__device__ __forceinline__ bool one_base_in_run(T d, int Pr, int &pos)
{ const T u = (d | (d >> 1)) & (T) HM_M5;
  if constexpr (sizeof(T) == 4) pos = Pr + (__clz((int) d) >> 1);
  else                          pos = Pr + (__clzll((long long) d) >> 1);
  return (u & (u-1)) == 0;
}

/* runscan_kernel, step 4 (warp-wide): the lane's member a of the run of L entries at window slots h .. h+L-1,
 * if it has one (in); own = the member is this CTA's to settle.  Its partners in the run give H and U (Bloom
 * insert when U > 0); a candidate record when H(x) = H(partner) = 1 and x is the lower member.  The partner
 * is member `part` of the same run, which lane + part - a holds and has counted in this same pass unless
 * that lane lies past the warp's 32 (only runs straddling two passes): then its H is counted here.
 * LMAX > 0: L <= LMAX, and the run mates are read in one unrolled sweep (slots h .. h+LMAX-1 lie in the
 * window), so their loads overlap instead of forming a chain.                                         -> emit */
template <int KW, bool SL, int LMAX>
__device__ __forceinline__ bool settle_members(const RsSmem<KW> &S, const SymmView &W, int kmer, int Pr, int pup,
                                               int h, int L, int a, bool in, bool own, int lane,
                                               uint64_t &x, uint64_t &xl, uint64_t &meta)
{ int Hx = 0, Ux = 0, part = 0, ppos = 0, cx = 0;
  if (in)
    { x  = S.key[h+a];
      xl = KW == 2 ? S.klo[h+a] : 0;
      cx = S.cnt[h+a];
      auto mate = [&](int b)
        { int pos;
          if (b < L && b != a && one_base_in_run(run_sfx<KW>(x ^ S.key[h+b],KW == 2 ? xl ^ S.klo[h+b] : 0,Pr),Pr,pos) &&
              cx + (int) S.cnt[h+b] <= HM_SMAX)
            { Hx += 1;
              if (pos >= pup) Ux += 1;
              part = b; ppos = pos;
            }
        };
      if constexpr (LMAX > 0)
        {
#pragma unroll
          for (int b = 0; b < LMAX; b++)
            mate(b);
        }
      else
        for (int b = 0; b < L; b++)
          mate(b);
      if (own && Ux > 0)
        bloom_insert<KW,SL>(W,kmer,x,xl);
    }
  const int pl = lane + part - a;                                  /* the partner's lane */
  int       Hy = __shfl_sync(0xffffffffu,Hx,pl & 31);
  if (!in || !own || Hx != 1 || part < a)
    return false;
  const uint64_t y = S.key[h+part], yl = KW == 2 ? S.klo[h+part] : 0;
  const int      cy = S.cnt[h+part];
  if (pl > 31)                                                     /* (part > a, so pl > lane >= 0) */
    { Hy = 0;
      for (int b = 0; b < L; b++)
        { int pos;
          if (b != part && one_base_in_run(run_sfx<KW>(y ^ S.key[h+b],KW == 2 ? yl ^ S.klo[h+b] : 0,Pr),Pr,pos) &&
              cy + (int) S.cnt[h+b] <= HM_SMAX)
            Hy += 1;
        }
    }
  if (Hy != 1)
    return false;
  meta = pack_meta(cx,cy,ppos,base_at<KW>(y,yl,ppos));
  return true;
}

/* Pass 1.  83 % of the entries of a genome-sized table are alone in their run (no other entry shares
 * their first k/2 bases) and 15 % sit in a run of exactly two -- almost always the two alleles of one
 * heterozygous site.  The kernel is limited by instruction issue and by the latency of its few serial
 * phases as much as by bytes (an H100 SXM issues about 100 warp instructions per 32 entries in the time
 * its 3.35 TB/s deliver them), so the common cases are loop-free and, once the tile has landed, every WARP works on its own
 * 256 entries without any CTA barrier:
 *   1. adjacency bits: eq[i] = slots i, i+1 belong to one run (one ballot per 32 slots; a warp computes
 *      the ten words it needs itself and keeps them one per lane)
 *   2. classification of 8 x 32 entries with bit operations, one WORD PER LANE:
 *      head of a two-entry run / head of a longer run / nothing
 *   3. two-entry runs: one comparison settles both members (per-warp task list, every lane busy)
 *   4. longer runs (5 % of the entries, a few per warp) from the same per-warp list, still from shared
 *      memory: a run whose head is in the tile and that has at most RS_RUNCAP = RS_HALO+1 entries lies
 *      inside the window.  Its length is the count of ones from the head on in the adjacency bits of
 *      step 1 (two shuffles, a funnel shift, __ffs; 33 or more: the rest from the keys).  3..8 entries:
 *      a lane per member, the members of all the warp's runs one after the other (a run per lane, every
 *      pair once, costs the warp its longest run's L^2/2 comparisons and a staging call per member:
 *      2.07-2.11 against 1.98-2.01 ms per benchmark step); 9..RS_RUNCAP: the whole warp, one member
 *      per lane.  A member counts its own partners only; the single partner's count is read from the
 *      partner's lane.  Only runs that may reach past the window are listed for runs_kernel (none in
 *      the 2e8-entry benchmark table, whose 3.4e6 runs of three or more took runs_kernel 0.40 ms on one
 *      H100 SXM at 400 W when it settled them all)
 *   Pair tests in steps 3 and 4 look at the bases after the run prefix only, one 32-bit word for k <= 32
 *   and one 64-bit word for k <= 64 (run_sfx, one_base_in_run).
 *   5. candidate records and run heads are staged in shared memory; after a CTA barrier thread 0
 *      reserves their ranges with one global atomic per CTA and list (one per record, or per warp, on
 *      the one list counter serialises in L2) while every thread reads its at most RS_FLUSH records
 *      from shared memory, and after a second barrier every thread stores them (flush_reserve,
 *      flush_store): the CTA ends one atomic round trip and one store after its last warp is done
 * (The alternatives -- every entry scanning its run in place, per-entry classification with predicated
 * list writes, CTA-wide task lists with a barrier per phase -- need more instructions, leave more lanes
 * idle or wait at the barriers.)                                                                      */
#ifdef RS_PROBE
/* Probe build only (make EXTRA=-DRS_PROBE=1, tools/time_runscan_phases.py): the clock64() cycles every warp
 * spends in each phase (0 staging / TMA wait, 1..4 as numbered in the kernel, then step 5 in three: 5 the
 * hand-off between the warps, 6 the global atomics on the list counters until their results are back, 7 the
 * copy of the staged records), summed over all warps with one atomic per warp and phase -- into one of
 * RS_PROBE_SLOTS rows by CTA, as a few hundred thousand atomics on a few addresses would serialise in L2 and
 * time themselves.  Columns RS_PHASES.. hold each CTA's lifetime by thread 0's clock, added once per CTA:
 * 8 start to window landed, 9 landed to every warp done with step 4 (the barrier that opens step 5), 10 from
 * then to thread 0's end (the tail).  And a mode: 0 the full kernel, 1 stage the window and return (load-only bound),
 * 2 every CTA stages tile blockIdx.x % 64, which stays in L2, and does the full work (compute-only bound);
 * each of the next four takes one part out of the full kernel, so its gap to mode 0 is the price of that
 * part: 3 no-RED (bloom_insert computes the slot but issues no atomic), 4 no-stage (stage_candidates and the
 * step-5 flush do nothing), 5 no-long (step 4 is skipped), 6 no-tail (every warp returns after step 4).   */
#define RS_PHASES 8
#define RS_COLS   (RS_PHASES+3)
#define RS_PROBE_SLOTS 1024
__device__ unsigned long long rs_probe_cycles[RS_PROBE_SLOTS*RS_COLS];
#define RS_PROBE_TILE(b)  (rs_probe_mode == 2 ? (b) % 64 : (b))
#define RS_PROBE_START    __shared__ long long rs_t0, rs_t1; \
                          long long rs_t = clock64(); unsigned long long rs_acc[RS_PHASES] = {0, 0, 0, 0, 0, 0, 0, 0}; \
                          if (threadIdx.x == 0) rs_t0 = rs_t;
#define RS_PROBE_MARK(ph) { const long long t_ = clock64(); rs_acc[ph] += (unsigned long long) (t_ - rs_t); rs_t = t_; }
#define RS_PROBE_LANDED() if (threadIdx.x == 0) rs_t1 = clock64();
#define RS_PROBE_ALLDONE  const long long rs_t2 = clock64();
#define RS_PROBE_ROW      (rs_probe_cycles + (blockIdx.x % RS_PROBE_SLOTS)*RS_COLS)
#define RS_PROBE_FLUSH()  { if (lane == 0) _Pragma("unroll") for (int p_ = 0; p_ < RS_PHASES; p_++) \
                              atomicAdd(RS_PROBE_ROW + p_,rs_acc[p_]); }
#define RS_PROBE_LIFE()   { const long long t3_ = clock64(); \
                            if (threadIdx.x == 0) { atomicAdd(RS_PROBE_ROW + RS_PHASES,  (unsigned long long) (rs_t1 - rs_t0)); \
                                             atomicAdd(RS_PROBE_ROW + RS_PHASES+1,(unsigned long long) (rs_t2 - rs_t1)); \
                                             atomicAdd(RS_PROBE_ROW + RS_PHASES+2,(unsigned long long) (t3_ - rs_t2)); } }
#define RS_PROBE_LOADONLY() if (rs_probe_mode == 1) { RS_PROBE_FLUSH(); return; }
#define RS_PROBE_NOTAIL()   if (rs_probe_mode == 6) { RS_PROBE_FLUSH(); return; }

/* cycles != NULL: the sums since the last call into cycles[RS_PHASES+3]; then clear them and set the mode */
extern "C" int hm_probe_runscan(int mode, unsigned long long *cycles)
{ static unsigned long long rows[RS_PROBE_SLOTS*RS_COLS];
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess && cycles != NULL)
    { e = cudaMemcpyFromSymbol(rows,rs_probe_cycles,sizeof(rows));
      for (int p = 0; p < RS_COLS; p++)
        { cycles[p] = 0;
          for (int r = 0; r < RS_PROBE_SLOTS; r++)
            cycles[p] += rows[r*RS_COLS+p];
        }
    }
  memset(rows,0,sizeof(rows));
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbol(rs_probe_cycles,rows,sizeof(rows));
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbol(rs_probe_mode,&mode,sizeof(mode));
  return e == cudaSuccess ? HM_OK : hm_cuda_fail(e,"hm_probe_runscan");
}
#else
#define RS_PROBE_TILE(b)  (b)
#define RS_PROBE_START
#define RS_PROBE_MARK(ph)
#define RS_PROBE_LANDED()
#define RS_PROBE_ALLDONE
#define RS_PROBE_FLUSH()
#define RS_PROBE_LIFE()
#define RS_PROBE_LOADONLY()
#define RS_PROBE_NOTAIL()
#endif

template <typename IdxT, int KW, bool SL>
__global__ void __launch_bounds__(RS_THREADS,RS_MINBLOCKS)
runscan_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
               const uint16_t *__restrict__ cnt, int64_t n, const IdxT *__restrict__ bucket, int bshift,
               int kmer, int64_t lo, int64_t hi, int64_t tile0, int use_tma, const SymmView W)
{ extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ unsigned s_nc, s_nr;
  __shared__ unsigned long long s_base[2];
  RsSmem<KW> S;
  S.key   = (uint64_t *) smem;
  S.klo   = S.key + (KW == 2 ? RS_WIN : 0);
  S.ckey  = S.key + KW*RS_WIN;
  S.clo   = S.ckey + (KW == 2 ? RS_STAGE : 0);
  S.cmeta = S.ckey + KW*RS_STAGE;
  S.cnt   = (uint16_t *) (S.cmeta + RS_STAGE);
  S.t1    = S.cnt + RS_WIN;                          /* per warp: RS_TILE/2/8 heads of two-entry runs        */
  S.t2r   = S.t1 + RS_TILE/2;                        /* CTA: heads of longer runs (at most RS_TILE/3)        */

  const int      Pr   = kmer >> 1;                 /* run = entries sharing their first Pr bases     */
  const int      pup  = kmer - Pr;                 /* positions >= pup have a mirror position < Pr   */
  const int      psh  = 64-2*Pr;
  const uint64_t pmask = ~(uint64_t) 0 << psh;
  const unsigned FULL = 0xffffffffu;
  const int      lane = threadIdx.x & 31;
  const int      warp = threadIdx.x >> 5;
  const unsigned lt   = (1u << lane) - 1;
  RS_PROBE_START

  const int64_t T0 = (tile0 + RS_PROBE_TILE(blockIdx.x)) * RS_TILE;
  const int64_t ws = T0 - RS_HALO;
  const int64_t e0 = ws > 0 ? ws : 0;
  const int64_t e1 = T0+RS_TILE+RS_HALO < n ? T0+RS_TILE+RS_HALO : n;
  const int     v0 = (int) (e0-ws), v1 = (int) (e1-ws);          /* valid window slots [v0,v1)   */

  /* ---- stage the window: TMA bulk copies for the 16-byte multiple, plain loads for the rest ---- */
  const int m   = v1-v0;
  const int mt  = use_tma ? (m & ~7) : 0;
  if (threadIdx.x == 0)
    { s_nc = 0; s_nr = 0;
      if (mt > 0)
        { mbar_init(&s_bar,1);
          fence_proxy_async_smem();
        }
    }
  __syncthreads();
  if (threadIdx.x == 0 && mt > 0)
    { mbar_arrive_expect_tx(&s_bar,(unsigned) (mt*(8*KW+2)));
      bulk_copy_g2s(S.key+v0,keys+e0,(unsigned) (8*mt),&s_bar);
      if (KW == 2)
        bulk_copy_g2s(S.klo+v0,keys_lo+e0,(unsigned) (8*mt),&s_bar);
      bulk_copy_g2s(S.cnt+v0,cnt+e0,(unsigned) (2*mt),&s_bar);
    }
  if (mt < m || v0 > 0 || v1 < RS_WIN)                /* boundary tiles / unaligned tables only (CTA-uniform) */
    { for (int j = mt + threadIdx.x; j < m; j += RS_THREADS)
        { S.key[v0+j] = keys[e0+j];
          if (KW == 2) S.klo[v0+j] = keys_lo[e0+j];
          S.cnt[v0+j] = cnt[e0+j];
        }
      if (mt > 0)
        mbar_wait(&s_bar,0);
      __syncthreads();
      /* slots outside the table: a key no neighbour can share a run with */
      const uint64_t sa = ~S.key[v0], sb = ~S.key[v1-1];
      __syncthreads();
      for (int j = threadIdx.x; j < RS_WIN; j += RS_THREADS)
        if (j < v0)       S.key[j] = sa;
        else if (j >= v1) S.key[j] = sb;
      __syncthreads();
    }
  else
    mbar_wait(&s_bar,0);
  RS_PROBE_MARK(0)
  RS_PROBE_LANDED()
  RS_PROBE_LOADONLY()

  /* ---- 1. adjacency bits of this warp's words wd0-1 .. wd0+RS_EPT, word t in lane t ---- */
  const int wd0 = RS_HALO/32 + warp*RS_EPT;            /* first word (32 slots) of this warp's part of the tile */
  unsigned  eqw = 0;
#pragma unroll
  for (int t = 0; t < RS_EPT+2; t++)
    { const int i = (wd0-1+t)*32 + lane;
      bool eq;
      if (psh >= 32)                                   /* k <= 33: the first Pr bases sit in the upper word */
        { const uint32_t a = (uint32_t) (S.key[i] >> 32);
          uint32_t       b = __shfl_down_sync(FULL,a,1);
          if (lane == 31) b = (uint32_t) (S.key[i+1] >> 32);
          eq = (((a ^ b) >> (psh-32)) == 0);
        }
      else
        eq = (((S.key[i] ^ S.key[i+1]) & pmask) == 0);
      const unsigned bal = __ballot_sync(FULL,eq);
      if (lane == t) eqw = bal;
    }
  RS_PROBE_MARK(1)

  /* ---- 2. classify: lane t in 1..RS_EPT takes word wd0-1+t ---- */
  const int a0 = RS_HALO + (lo > T0 ? (int) (lo-T0 < RS_TILE ? lo-T0 : RS_TILE) : 0);   /* slots this CTA answers for */
  const int a1 = RS_HALO + (hi-T0 < RS_TILE ? (int) (hi-T0) : RS_TILE);
  uint16_t *my1  = S.t1  + warp*(RS_TILE/2/(RS_THREADS/32));
  int n1, n3;
  { const unsigned P = __shfl_up_sync(FULL,eqw,1), N = __shfl_down_sync(FULL,eqw,1);
    unsigned m2 = 0, m3 = 0;
    const int wd = wd0-1+lane;
    if (lane >= 1 && lane <= RS_EPT)
      { const unsigned E = eqw;
        const unsigned em1 = (E << 1) | (P >> 31);                     /* eq[w-1] */
        const unsigned em2 = (E << 2) | (P >> 30);                     /* eq[w-2] */
        const unsigned ep1 = (E >> 1) | (N << 31);                     /* eq[w+1] */
        const int      s0  = wd*32;                                    /* slot of bit 0 */
        unsigned act = 0xffffffffu;
        if (s0 < a0)      act &= (a0-s0 >= 32) ? 0u : (0xffffffffu << (a0-s0));
        if (s0+32 > a1)   act &= (a1-s0 <= 0)  ? 0u : (0xffffffffu >> (s0+32-a1));
        const unsigned more = (em1 & E) | (E & ep1) | (em1 & em2);
        m2 = (E & ~em1 & ~ep1) & act;                                  /* head of a run of exactly two */
        m3 = more & act & ~em1;                                        /* head of a longer run */
      }
    /* per-warp task lists: inclusive scans of the counts over the lanes.  Heads of longer runs follow the
     * heads of runs of two in the same list: two heads are at least two slots apart, so both fit in 128 */
    const int c2 = __popc(m2), c3 = __popc(m3);
    int pre2 = c2, pre3 = c3;
#pragma unroll
    for (int o = 1; o <= RS_EPT; o <<= 1)
      { int v2 = __shfl_up_sync(FULL,pre2,o), v3 = __shfl_up_sync(FULL,pre3,o);
        if (lane >= o) { pre2 += v2; pre3 += v3; }
      }
    n1 = __shfl_sync(FULL,pre2,RS_EPT);
    n3 = __shfl_sync(FULL,pre3,RS_EPT);
    int at = pre2-c2;
    while (m2 != 0)
      { my1[at++] = (uint16_t) (wd*32 + __ffs(m2)-1);
        m2 &= m2-1;
      }
    at = n1 + pre3-c3;
    while (m3 != 0)
      { my1[at++] = (uint16_t) (wd*32 + __ffs(m3)-1);
        m3 &= m3-1;
      }
  }
  __syncwarp();
  if (RS_PROBE_IS(5))                                  /* probe no-long: step 4 is skipped */
    n3 = 0;
  RS_PROBE_MARK(2)

  /* ---- 3. runs of two: one comparison settles both members ---- */
  for (int i0 = 0; i0 < n1; i0 += 32)
    { const int i = i0+lane;
      bool     emit = false;
      uint64_t x = 0, xl = 0, meta = 0;
      if (i < n1)
        { const int w = my1[i];
          x = S.key[w];
          const uint64_t y = S.key[w+1];
          uint64_t yl = 0;
          if (KW == 2) { xl = S.klo[w]; yl = S.klo[w+1]; }
          const int cx = S.cnt[w], cy = S.cnt[w+1];
          int pos;
          if (one_base_in_run(run_sfx<KW>(x ^ y,xl ^ yl,Pr),Pr,pos) && cx+cy <= HM_SMAX)   /* H(x) = H(y) = 1 */
            { emit = true;
              meta = pack_meta(cx,cy,pos,base_at<KW>(y,yl,pos));
              if (pos >= pup)                                              /* U(x) = U(y) = 1: both are in S */
                { bloom_insert<KW,SL>(W,kmer,x,xl);
                  bloom_insert<KW,SL>(W,kmer,y,yl);
                }
            }
        }
      stage_candidates<KW>(S,&s_nc,W,emit,x,xl,meta,lane,lt);
    }
  RS_PROBE_MARK(3)

  /* ---- 4. longer runs, from the window: a run whose head is in the tile and that has at most RS_RUNCAP
   *         entries lies inside it.  Members at or after hi are not ours (slots >= b1) ---- */
  const int b1 = hi-T0 < RS_TILE+RS_HALO ? RS_HALO + (int) (hi-T0) : RS_WIN;
  for (int i0 = 0; i0 < n3; i0 += 32)
    { const int i = i0+lane;
      const int h = i < n3 ? my1[n1+i] : 0;              /* head slot */
      int       L = 0;                                   /* run length; 33: 33 or more */
      { /* the run's extent from the adjacency bits: eq[h], eq[h+1], ... are ones up to its last member.  h lies
         * in word wd0-1+t, t in 1..RS_EPT; lanes t and t+1 hold that word and the next: 32 bits in view */
        const int      t  = (h >> 5) - (wd0-1);
        const unsigned w0 = __shfl_sync(FULL,eqw,t & 31), w1 = __shfl_sync(FULL,eqw,(t+1) & 31);
        const unsigned up = __funnelshift_r(w0,w1,h & 31);                          /* eq[h .. h+31] */
        if (i < n3)
          L = (~up != 0) ? __ffs((int) ~up) : 33;
      }
      /* 3..8 entries: a lane per member, the members of all the lanes' runs one after the other */
      const int Ls = L <= 8 ? L : 0;
      int inc = Ls;                                      /* inclusive scan of the members over the lanes */
#pragma unroll
      for (int o = 1; o < 32; o <<= 1)
        { const int v = __shfl_up_sync(FULL,inc,o);
          if (lane >= o) inc += v;
        }
      const int M = __shfl_sync(FULL,inc,31);
      for (int t0 = 0; t0 < M; t0 += 32)
        { const int t = t0+lane;
          int r = 0;                                     /* member t's run: the first lane whose inc > t */
#pragma unroll
          for (int s = 16; s > 0; s >>= 1)
            if (__shfl_sync(FULL,inc,r+s-1) <= t) r += s;
          const int hr = __shfl_sync(FULL,h,r), Lr = __shfl_sync(FULL,Ls,r);
          const int a  = t - (__shfl_sync(FULL,inc,r) - Lr);
          bool     emit = false;
          uint64_t x = 0, xl = 0, meta = 0;
          emit = settle_members<KW,SL,8>(S,W,kmer,Pr,pup,hr,Lr,a,t < M,hr+a < b1,lane,x,xl,meta);
          stage_candidates<KW>(S,&s_nc,W,emit,x,xl,meta,lane,lt);
        }
      /* 9..RS_RUNCAP entries: the whole warp, one run after the other, a member per lane */
      unsigned lb = __ballot_sync(FULL,L > 8);
      while (lb != 0)
        { const int src = __ffs(lb)-1;
          lb &= lb-1;
          const int hh = __shfl_sync(FULL,h,src);
          int       LL = __shfl_sync(FULL,L,src);
          if (LL > 32)                                   /* (warp-uniform) slots hh .. hh+32 are in the run; the */
            { const uint64_t xh = S.key[hh];             /*   rest of it from the keys, 32 slots at a time       */
              while (LL <= RS_RUNCAP)
                { const int      t = hh+LL+lane;
                  const unsigned sb = __ballot_sync(FULL,t < RS_WIN && ((S.key[t] ^ xh) & pmask) == 0);
                  if (sb != FULL) { LL += __ffs(~sb)-1; break; }
                  LL += 32;
                }
            }
          if (LL > RS_RUNCAP || hh+LL >= RS_WIN)           /* (warp-uniform) may go on past the window: runs_kernel */
            { if (lane == 0)
                S.t2r[atomicAdd(&s_nr,1u)] = (uint16_t) hh;
              continue;
            }
          for (int a0 = 0; a0 < LL; a0 += 32)
            { const int a = a0+lane;
              bool     emit = false;
              uint64_t x = 0, xl = 0, meta = 0;
              emit = settle_members<KW,SL,0>(S,W,kmer,Pr,pup,hh,LL,a,a < LL,hh+a < b1,lane,x,xl,meta);
              stage_candidates<KW>(S,&s_nc,W,emit,x,xl,meta,lane,lt);
            }
        }
    }
  RS_PROBE_MARK(4)
  RS_PROBE_NOTAIL()

  /* ---- 5. every warp moves its share of the staged records out ---- */
  __syncthreads();
  RS_PROBE_MARK(5)
  RS_PROBE_ALLDONE
  if (RS_PROBE_IS(4))                                  /* (probe no-stage: no flush either) */
    { RS_PROBE_FLUSH() return; }
  const unsigned nc = s_nc < RS_STAGE ? s_nc : RS_STAGE, nr = s_nr;
  if (nc == 0 && nr == 0)                              /* (CTA-uniform) */
    { RS_PROBE_MARK(6) RS_PROBE_LIFE() RS_PROBE_FLUSH() return; }
  RsFlush F;
  flush_reserve<KW>(S,&s_base[0],&s_base[1],W,nc,nr,F);
  __syncthreads();
  RS_PROBE_MARK(6)
  flush_store<KW>(S,s_base[0],s_base[1],W,nc,nr,T0,F);
  RS_PROBE_MARK(7)
  RS_PROBE_LIFE()
  RS_PROBE_FLUSH()
}

/* Pass 1, crowded tables.  A run is the set of entries sharing their first k/2 bases, so an entry has
 * n / 4^(k/2) run mates on average whatever the sequence: 0.19 at 2e8 k-mers of k = 31 (where "alone" and
 * "a run of two" are all there is and runscan_kernel's classification pays), but 1.9 at 2e9 and 4.7 at
 * 5e9, where nearly every entry sits in a run of several unrelated k-mers.  Here every window slot
 * compares itself with the slots AFTER it in its run (the run's extent comes from the adjacency bits),
 * a pair found adds to both members' partner counts (byte-packed shared-memory atomics) and records the
 * partner; after a barrier every entry of the tile reads its own counts: Bloom insert if it has an
 * upper partner, candidate record if it and its single partner have one partner each.  All pairs of a
 * run are compared exactly once, the comparisons are spread evenly over the lanes, and the cost grows
 * with the run length instead of falling off a cliff as one thread per run does.  Runs of more than
 * RS_LONGRUN entries are listed for runs_kernel as before.                                            */
template <typename IdxT, int KW, bool SL>
__global__ void __launch_bounds__(RS_THREADS,RS_MINBLOCKS)
runscan_dense_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                     const uint16_t *__restrict__ cnt, int64_t n, int kmer, int64_t lo, int64_t hi,
                     int64_t tile0, int use_tma, const SymmView W)
{ extern __shared__ __align__(128) uint8_t smem[];
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ unsigned s_nc, s_nl;
  __shared__ unsigned long long s_base[2];
  __shared__ unsigned s_eq[RS_WIN/32+1];
  RsSmem<KW> S;
  S.key   = (uint64_t *) smem;
  S.klo   = S.key + (KW == 2 ? RS_WIN : 0);
  S.ckey  = S.key + KW*RS_WIN;
  S.clo   = S.ckey + (KW == 2 ? RS_STAGE : 0);
  S.cmeta = S.ckey + KW*RS_STAGE;
  S.cnt   = (uint16_t *) (S.cmeta + RS_STAGE);
  S.t1    = S.cnt + RS_WIN;                          /* here: a mark per window slot (RS_WIN)                */
  S.t2r   = S.t1 + RS_WIN;                           /* here: heads of runs of more than RS_LONGRUN entries  */
  uint16_t *s_part = S.t2r + RS_TILE/8;               /* partner slot of every window slot (RS_WIN)           */
  unsigned *hu = (unsigned *) (s_part + RS_WIN);      /* partner counts: per slot H (low byte) | U (high byte) */
  uint32_t *rem = hu + RS_WIN/2;                      /* k <= 32: the bases after the run prefix, 32 bits per slot */

  const int      Pr   = kmer >> 1, pup = kmer - Pr, psh = 64-2*Pr;
  const uint64_t pmask = ~(uint64_t) 0 << psh;
  const unsigned FULL = 0xffffffffu;
  const int      lane = threadIdx.x & 31;
  const int      warp = threadIdx.x >> 5;
  const unsigned lt   = (1u << lane) - 1;

  const int64_t T0 = (tile0 + blockIdx.x) * RS_TILE;
  const int64_t ws = T0 - RS_HALO;
  const int64_t e0 = ws > 0 ? ws : 0;
  const int64_t e1 = T0+RS_TILE+RS_HALO < n ? T0+RS_TILE+RS_HALO : n;
  const int     v0 = (int) (e0-ws), v1 = (int) (e1-ws);

  const int m   = v1-v0;
  const int mt  = use_tma ? (m & ~7) : 0;
  if (threadIdx.x == 0)
    { s_nc = 0; s_nl = 0;
      if (mt > 0)
        { mbar_init(&s_bar,1);
          fence_proxy_async_smem();
        }
    }
  for (int j = threadIdx.x; j < RS_WIN/2; j += RS_THREADS)
    hu[j] = 0;
  __syncthreads();
  if (threadIdx.x == 0 && mt > 0)
    { mbar_arrive_expect_tx(&s_bar,(unsigned) (mt*(8*KW+2)));
      bulk_copy_g2s(S.key+v0,keys+e0,(unsigned) (8*mt),&s_bar);
      if (KW == 2)
        bulk_copy_g2s(S.klo+v0,keys_lo+e0,(unsigned) (8*mt),&s_bar);
      bulk_copy_g2s(S.cnt+v0,cnt+e0,(unsigned) (2*mt),&s_bar);
    }
  if (mt < m || v0 > 0 || v1 < RS_WIN)                /* boundary tiles / unaligned tables only (CTA-uniform) */
    { for (int j = mt + threadIdx.x; j < m; j += RS_THREADS)
        { S.key[v0+j] = keys[e0+j];
          if (KW == 2) S.klo[v0+j] = keys_lo[e0+j];
          S.cnt[v0+j] = cnt[e0+j];
        }
      if (mt > 0)
        mbar_wait(&s_bar,0);
      __syncthreads();
      const uint64_t sa = ~S.key[v0], sb = ~S.key[v1-1];
      __syncthreads();
      for (int j = threadIdx.x; j < RS_WIN; j += RS_THREADS)
        if (j < v0)       S.key[j] = sa;
        else if (j >= v1) S.key[j] = sb;
      __syncthreads();
    }
  else
    mbar_wait(&s_bar,0);

  /* ---- adjacency bits of the whole window; k <= 32: the bases after the run prefix as one 32-bit word ---- */
  const bool narrow = (KW == 1) && (kmer-Pr <= 16);      /* CTA-uniform: pair tests in 32-bit arithmetic */
  for (int wd = warp; wd < RS_WIN/32; wd += RS_THREADS/32)
    { const int i = wd*32 + lane;
      bool eq = false;
      const uint64_t ki = S.key[i];
      if (i+1 < RS_WIN)
        eq = (((ki ^ S.key[i+1]) & pmask) == 0);
      if (narrow)
        rem[i] = (uint32_t) ((ki << (2*Pr)) >> 32);
      const unsigned bal = __ballot_sync(FULL,eq);
      if (lane == 0)
        s_eq[wd] = bal;
    }
  if (threadIdx.x == 0)
    s_eq[RS_WIN/32] = 0;
  __syncthreads();

  /* ---- run mates after / before every slot = consecutive ones in the adjacency bits (32 are in view) ---- */
  const int a0 = RS_HALO + (lo > T0 ? (int) (lo-T0 < RS_TILE ? lo-T0 : RS_TILE) : 0);   /* slots this CTA answers for */
  const int a1 = RS_HALO + (hi-T0 < RS_TILE ? (int) (hi-T0) : RS_TILE);
  for (int i = threadIdx.x; i < RS_WIN; i += RS_THREADS)
    { const int      w = i >> 5, b = i & 31;
      const unsigned up = __funnelshift_r(s_eq[w],s_eq[w+1],b);                 /* eq[i], eq[i+1], ... */
      const int      fwd = (~up == 0) ? 32 : __ffs((int) ~up)-1;
      int back = 0;
      if (i > 0)
        { const int      wq = (i-1) >> 5, bq = (i-1) & 31;
          const unsigned dn = __funnelshift_l(wq > 0 ? s_eq[wq-1] : 0u,s_eq[wq],31-bq);   /* eq[i-1], eq[i-2], ... from the top */
          back = (~dn == 0) ? 32 : __clz((int) ~dn);
        }
      uint16_t mark = (uint16_t) fwd;                                            /* 0..31 run mates after this slot */
      if (back+fwd+1 > RS_LONGRUN)
        { mark = 0xffff;                                                         /* member of a long run: not ours */
          if (back == 0 && i >= a0 && i < a1)                                    /* its head, in our range: runs_kernel */
            S.t2r[atomicAdd(&s_nl,1u)] = (uint16_t) i;
        }
      S.t1[i] = mark;
      s_part[i] = (uint16_t) i;
    }
  __syncthreads();

  /* ---- every slot against the slots after it in its run ---- */
  for (int i = threadIdx.x; i < RS_WIN; i += RS_THREADS)
    { const int fwd = S.t1[i];
      if (fwd == 0 || fwd == 0xffff)
        continue;
      const int cx = S.cnt[i];
      if (narrow)
        { const uint32_t rx = rem[i];
          for (int j = i+1; j <= i+fwd; j++)
            { const uint32_t d = rx ^ rem[j];
              const uint32_t u = (d | (d>>1)) & 0x55555555u;
              if ((u & (u-1)) == 0 && cx + (int) S.cnt[j] <= HM_SMAX)
                { const int      pos = Pr + (__clz((int) d) >> 1);
                  const unsigned inc = 1u | (pos >= pup ? 0x100u : 0u);
                  atomicAdd(hu + (i>>1), inc << (16*(i&1)));
                  atomicAdd(hu + (j>>1), inc << (16*(j&1)));
                  s_part[i] = (uint16_t) j;                /* any partner: only read when there is exactly one */
                  s_part[j] = (uint16_t) i;
                }
            }
        }
      else
        { const uint64_t x = S.key[i], xl = KW == 2 ? S.klo[i] : 0;
          for (int j = i+1; j <= i+fwd; j++)
            { int pos;
              if (one_base_apart<KW>(x,xl,S.key[j],KW == 2 ? S.klo[j] : 0,pos) && cx + (int) S.cnt[j] <= HM_SMAX)
                { const unsigned inc = 1u | (pos >= pup ? 0x100u : 0u);
                  atomicAdd(hu + (i>>1), inc << (16*(i&1)));
                  atomicAdd(hu + (j>>1), inc << (16*(j&1)));
                  s_part[i] = (uint16_t) j;
                  s_part[j] = (uint16_t) i;
                }
            }
        }
    }
  __syncthreads();

  /* ---- every entry of the tile: its counts -> Bloom insert, candidate record ---- */
  for (int i0 = RS_HALO + (threadIdx.x & ~31); i0 < RS_HALO+RS_TILE; i0 += RS_THREADS)
    { const int i = i0+lane;
      bool     emit = false;
      uint64_t x = 0, xl = 0, meta = 0;
      if (i >= a0 && i < a1 && S.t1[i] != 0xffff)
        { const unsigned c = (hu[i>>1] >> (16*(i&1))) & 0xffffu;
          const int H = (int) (c & 0xff), U = (int) (c >> 8);
          if (H > 0)
            { x = S.key[i];
              if (KW == 2) xl = S.klo[i];
              if (U > 0)
                bloom_insert<KW,SL>(W,kmer,x,xl);
              const int j = s_part[i];
              if (H == 1 && j > i && ((hu[j>>1] >> (16*(j&1))) & 0xffu) == 1)
                { const uint64_t y = S.key[j], yl = KW == 2 ? S.klo[j] : 0;
                  int pos;
                  one_base_apart<KW>(x,xl,y,yl,pos);
                  emit = true;
                  meta = pack_meta(S.cnt[i],S.cnt[j],pos,base_at<KW>(y,yl,pos));
                }
            }
        }
      stage_candidates<KW>(S,&s_nc,W,emit,x,xl,meta,lane,lt);
    }

  /* ---- every warp moves its share of the staged records and the long-run heads out ---- */
  __syncthreads();
  const unsigned nc = s_nc < RS_STAGE ? s_nc : RS_STAGE, nr = s_nl;
  if (nc == 0 && nr == 0)                              /* (CTA-uniform) */
    return;
  RsFlush F;
  flush_reserve<KW>(S,&s_base[0],&s_base[1],W,nc,nr,F);
  __syncthreads();
  flush_store<KW>(S,s_base[0],s_base[1],W,nc,nr,T0,F);
}

/* f(Inst<IdxT,KW>()) for the instantiation that serves (kmer, idx64): KW key words, IdxT bucket offsets */
template <typename I, int K> struct Inst { typedef I IdxT; static constexpr int KW = K; };

template <class F>
static cudaError_t dispatch(int kmer, int idx64, F f)
{ if (kmer <= 32)
    return idx64 ? f(Inst<uint64_t,1>()) : f(Inst<uint32_t,1>());
  return idx64 ? f(Inst<uint64_t,2>()) : f(Inst<uint32_t,2>());
}

template <typename IdxT, int KW, bool SL = false>
static cudaError_t launch_runscan(const uint64_t *keys, const uint64_t *keys_lo, const uint16_t *cnt, int64_t n,
                                  const void *bucket, int bits, int kmer, int64_t lo, int64_t hi,
                                  const SymmView &W, cudaStream_t st)
{ static int configured[64] = {0};                            /* per instantiation */
  int dev = 0;
  cudaGetDevice(&dev);
  int64_t tile0 = lo/RS_TILE, tile1 = (hi+RS_TILE-1)/RS_TILE;
  int     tma   = ((((uintptr_t) keys) | ((uintptr_t) cnt) | ((uintptr_t) (keys_lo ? keys_lo : keys))) & 15) == 0;
  /* mean number of run mates of an entry = n / 4^(k/2): sparse tables take the classifying kernel, crowded
   * ones the all-pairs-in-the-run kernel (HETMERS_RUNSCAN=sparse|dense forces one)                       */
  const int   Pr  = kmer >> 1;
  double      lam = (2*Pr >= 62) ? 0.0 : (double) n / (double) ((uint64_t) 1 << (2*Pr));
  bool        dense = (lam > 0.6);
  const char *force = getenv("HETMERS_RUNSCAN");
  if (force != NULL && strcmp(force,"dense") == 0)  dense = true;
  if (force != NULL && strcmp(force,"sparse") == 0) dense = false;
  cudaError_t e;
  if (dense)
    { size_t smem = (size_t) RS_WIN*(8*KW+2) + (size_t) RS_STAGE*8*(KW+1) +
                    2*(size_t) (RS_WIN+RS_TILE/8+RS_WIN) + 4*(size_t) (RS_WIN/2+RS_WIN);   /* 52 KB (k <= 32) / 74 KB */
      if (smem > 48*1024 && (dev >= 64 || !(configured[dev] & 2)))
        { e = cudaFuncSetAttribute(runscan_dense_kernel<IdxT,KW,SL>,cudaFuncAttributeMaxDynamicSharedMemorySize,(int) smem);
          if (e != cudaSuccess) return e;
          if (dev < 64) configured[dev] |= 2;
        }
      runscan_dense_kernel<IdxT,KW,SL><<<(unsigned) (tile1-tile0),RS_THREADS,smem,st>>>
          (keys,keys_lo,cnt,n,kmer,lo,hi,tile0,tma,W);
    }
  else
    { size_t smem = (size_t) RS_WIN*(8*KW+2) + (size_t) RS_STAGE*8*(KW+1) +
                    2*(size_t) (RS_TILE/2+RS_TILE/2);                                /* 34 KB (k <= 32) / 55 KB */
      if (smem > 48*1024 && (dev >= 64 || !(configured[dev] & 1)))
        { e = cudaFuncSetAttribute(runscan_kernel<IdxT,KW,SL>,cudaFuncAttributeMaxDynamicSharedMemorySize,(int) smem);
          if (e != cudaSuccess) return e;
          if (dev < 64) configured[dev] |= 1;
        }
      runscan_kernel<IdxT,KW,SL><<<(unsigned) (tile1-tile0),RS_THREADS,smem,st>>>
          (keys,keys_lo,cnt,n,(const IdxT *) bucket,64-bits,kmer,lo,hi,tile0,tma,W);
    }
  return cudaGetLastError();
}

template <typename IdxT, int KW, bool SL = false>
static cudaError_t launch_runs(const uint64_t *keys, const uint64_t *keys_lo, const uint16_t *cnt, int64_t n,
                               const void *bucket, int bits, int kmer, int64_t lo, int64_t hi,
                               const SymmView &W, cudaStream_t st)
{ /* (the Bloom filter is filled inside runscan_kernel: a kernel of its own would read the records once more) */
  /* the count of listed runs is only known on the device, and on sparse tables it is ~0 (runscan_kernel settles
   * runs of up to RS_RUNCAP entries itself): at most one wave of CTAs, striding over the list               */
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  int64_t want = ((hi-lo)/64+255)/256;                        /* a thread per run if every 60th entry headed one */
  int     grid = (int) (want < sms*8 ? (want > 0 ? want : 1) : sms*8);
  runs_kernel<IdxT,KW,SL><<<grid,256,0,st>>>(keys,keys_lo,cnt,n,(const IdxT *) bucket,64-bits,kmer,lo,hi,W);
  return cudaGetLastError();
}

extern "C" int hm_k_symm_runscan(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                                 const void *d_bucket, int bits, int idx64, int kmer, int64_t lo, int64_t hi,
                                 void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards,
                                 void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER)
    return hm_set_error(HM_EUNSUPPORTED,"symmetric scan needs %d <= k <= %d (k=%d)",HM_SYMM_MIN_KMER,HM_MAX_KMER,kmer);
  if (lo < 0 || hi > n || lo > hi || bits < 1 || bits > 30 || d_work == NULL || layout == NULL)
    return hm_set_error(HM_EINVAL,"symm_runscan: bad range [%lld,%lld) of %lld or bits %d",
                        (long long) lo,(long long) hi,(long long) n,bits);
  if ((kmer > 32) != (d_keys_lo != NULL))
    return hm_set_error(HM_EINVAL,"symm_runscan: second key word array %s for k=%d",
                        d_keys_lo ? "given" : "missing",kmer);
  if ((shards != NULL && shards->n_seg > 1) != (layout->n_seg > 1) ||
      (shards != NULL && shards->n_seg > 1 && (shards->n_seg != layout->n_seg || shards->self < 0 ||
                                               shards->self >= shards->n_seg)))
    return hm_set_error(HM_EINVAL,"symm_runscan: shard table does not match the work-area layout");
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = make_view(d_work,layout,shards);
  HM_CUDA(cudaMemsetAsync(W.cand_n,0,256,st));
  HM_CUDA(cudaMemsetAsync(W.bloom + (size_t) W.self*W.seg_words,0,sizeof(uint32_t)*(size_t) W.seg_words,st));
  if (l2_persist())
    bloom_window(st,W.bloom,sizeof(uint32_t)*(size_t) W.seg_words*(size_t) W.n_seg,1);
  if (hi == lo)
    return HM_OK;
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { return launch_runscan<typename decltype(I)::IdxT,decltype(I)::KW>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,
                                                                       lo,hi,W,st); });
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"runscan_kernel");
  return HM_OK;
}

/* the runs runscan listed (three or more entries on sparse tables, more than RS_LONGRUN on crowded ones):
 * second half of "pass 1", a launch of its own so that callers can time the dominant kernel alone      */
extern "C" int hm_k_symm_runs(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                              const void *d_bucket, int bits, int idx64, int kmer, int64_t lo, int64_t hi,
                              void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards,
                              void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || d_work == NULL || layout == NULL ||
      (kmer > 32) != (d_keys_lo != NULL) || lo < 0 || hi > n || lo > hi)
    return hm_set_error(HM_EINVAL,"symm_runs: bad arguments");
  if (hi == lo)
    return HM_OK;
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = make_view(d_work,layout,shards);
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { return launch_runs<typename decltype(I)::IdxT,decltype(I)::KW>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,
                                                                    lo,hi,W,st); });
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"runs_kernel");
  return HM_OK;
}

/* ------------------------------------------------------------------------ pass 2 -------- */

#define RV_TS   192     /* shared-memory plot tile: sums < 192, mins < 96 */
#define RV_TM   96
#define RV_TROW 97      /* its row stride: odd, so that cells of one min in different rows are in different banks */
#define RV_THREADS 1024
#ifndef RV_ILP
#define RV_ILP 2                   /* candidates per thread and trip (4 spills at 64 registers: slower) */
#endif
#define RV_QCAP  (32*(RV_ILP+1))   /* queued Bloom hits per warp: fewer than 32 left over + a trip's */
#define RV_PROBE 4                 /* keys of a bucket the exact check loads at once */
#define RV_HA    (1ull << 48)      /* a queued record's meta: the Bloom bits of rc x / rc y were set */
#define RV_HB    (1ull << 49)

#ifdef RESOLVE_PROBE
/* Probe build only (make EXTRA=-DRESOLVE_PROBE=1, tools/time_resolve_phases.py).  A mode: 0 the full kernel, 1 the
 * candidate records only (loaded and dropped: the bound the record stream sets), 2 records and Bloom look-ups with
 * every hit taken as not isolated (no exact check), 3 the full kernel counting what it sees; and the counts of mode
 * 3: candidates, Bloom hits on rc x only / rc y only / both, exact checks that take the general path
 * (has_upper_partner), and the sizes of the buckets the exact checks scan (0 .. RVP_BINS-2 keys, then more).    */
#define RVP_BINS 50
#define RVP_CAND 0
#define RVP_HA   1
#define RVP_HB   2
#define RVP_HAB  3
#define RVP_GEN  4
#define RVP_HIST 5
#define RVP_NCTR (RVP_HIST+RVP_BINS)
__device__ unsigned long long rvp_ctr[RVP_NCTR];
__device__ int rvp_mode;
#define RVP_MODE rvp_mode
#define RVP_COUNT(i,v) { if (rvp_mode == 3) atomicAdd(rvp_ctr+(i),(unsigned long long) (v)); }
#define RVP_BUCKET(sz) RVP_COUNT(RVP_HIST + ((sz) < RVP_BINS-1 ? (int) (sz) : RVP_BINS-1),1)

/* ctr != NULL: the counts since the last call into ctr[RVP_NCTR]; then clear them and set the mode */
extern "C" int hm_probe_resolve(int mode, unsigned long long *ctr)
{ static unsigned long long rows[RVP_NCTR];
  cudaError_t e = cudaDeviceSynchronize();
  if (e == cudaSuccess && ctr != NULL)
    { e = cudaMemcpyFromSymbol(rows,rvp_ctr,sizeof(rows));
      memcpy(ctr,rows,sizeof(rows));
    }
  memset(rows,0,sizeof(rows));
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbol(rvp_ctr,rows,sizeof(rows));
  if (e == cudaSuccess)
    e = cudaMemcpyToSymbol(rvp_mode,&mode,sizeof(mode));
  return e == cudaSuccess ? HM_OK : hm_cuda_fail(e,"hm_probe_resolve");
}
#else
#define RVP_MODE 0
#define RVP_COUNT(i,v)
#define RVP_BUCKET(sz)
#endif

/* q's bucket [l,r) holds q's whole run (the bucket prefix is no longer than the run prefix): is q there
 * (found), and has it a partner at a position >= pup with a count sum <= HM_SMAX?  RV_PROBE keys (first
 * words) are loaded at once.  The check reads sectors at random from the table, and it is bound by how many
 * it reads, not by latency: so the second key word is read only for a key in q's run, and a count only for
 * an actual partner of q (on the bench table that takes the counts' sector -- a quarter of what the check
 * read -- out of nearly every check).                                                                  */
template <int KW>
__device__ __forceinline__ bool bucket_upper_partner(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                                                     const uint16_t *__restrict__ cnt, int64_t l, int64_t r,
                                                     int psh, int pup, uint64_t q, uint64_t ql, int cq, bool &found)
{ bool hit = false;
  found = false;
  for (int64_t i0 = l; i0 < r; i0 += RV_PROBE)
    { uint64_t z[RV_PROBE];
#pragma unroll
      for (int u = 0; u < RV_PROBE; u++)
        z[u] = (i0+u < r) ? __ldg(keys+i0+u) : ~q;             /* ~q: another run */
#pragma unroll
      for (int u = 0; u < RV_PROBE; u++)
        { if (((z[u] ^ q) >> psh) != 0)                        /* another run: neither q nor a partner */
            continue;
          const uint64_t zl = KW == 2 ? __ldg(keys_lo+i0+u) : 0;
          int pos;
          if (z[u] == q && (KW == 1 || zl == ql))
            found = true;
          else if (one_base_apart<KW>(q,ql,z[u],zl,pos) && pos >= pup && cq + (int) __ldg(cnt+i0+u) <= HM_SMAX)
            hit = true;
        }
    }
  return hit;
}

/* The general case of the exact check (a bucket prefix longer than the run prefix -- tiny tables -- or a
 * bucket of more than 48 keys): does table entry q (count cq: the table is symmetric, so it is the count
 * of the candidate member whose reverse complement q is) have a partner at a position >= pup?  Exact.  */
template <typename IdxT, int KW>
__device__ __noinline__ bool has_upper_partner(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                                               const uint16_t *__restrict__ cnt, int64_t n,
                                               const IdxT *__restrict__ bucket, int bshift, int kmer,
                                               uint64_t q, uint64_t ql, int cq, unsigned long long *status)
{ const int Pr = kmer >> 1, pup = kmer-Pr, psh = 64-2*Pr;
  if (bshift >= psh)                                            /* bucket prefix no longer than the run prefix */
    { const uint64_t bk = q >> bshift;
      const int64_t  l = (int64_t) bucket[bk], r = (int64_t) bucket[bk+1];
      if (r-l <= 48)
        { bool found = false, hit = false;
          for (int64_t i = l; i < r; i++)
            { const uint64_t z = __ldg(keys+i), zl = KW == 2 ? __ldg(keys_lo+i) : 0;
              if (z == q && (KW == 1 || zl == ql))
                { found = true; continue; }
              if (((z ^ q) >> psh) != 0)
                continue;
              int pos;
              if (one_base_apart<KW>(q,ql,z,zl,pos) && pos >= pup && cq + (int) __ldg(cnt+i) <= HM_SMAX)
                hit = true;
            }
          if (!found)
            atomicOr(status,SY_STATUS_ASYMMETRIC);
          return hit;
        }
    }
  int64_t j = bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,q,ql);
  if (j < 0)
    { atomicOr(status,SY_STATUS_ASYMMETRIC);
      return true;
    }
  bool capped = false;
  for (int dir = -1; dir <= 1; dir += 2)
    { int steps = 0;
      for (int64_t i = j+dir; i >= 0 && i < n; i += dir)
        { uint64_t z = __ldg(keys+i);
          if (((z ^ q) >> psh) != 0) break;
          if (++steps > RS_SCANCAP) { capped = true; break; }
          int pos;
          if (one_base_apart<KW>(q,ql,z,KW == 2 ? __ldg(keys_lo+i) : 0,pos) && pos >= pup &&
              cq + (int) __ldg(cnt+i) <= HM_SMAX)
            return true;
        }
    }
  if (!capped)
    return false;
  int H, U, ppos; int64_t part;
  neighbours_slow<IdxT,KW>(keys,keys_lo,cnt,bucket,bshift,kmer,pup,pup,q,ql,cq,H,U,part,ppos);
  return (U > 0);
}

/* where pass 2 checks a Bloom hit exactly (isolated_after_all) */
enum Lookup
  { LK_TABLE,        /* in core: is there an upper partner of the key in its run of the table                     */
    LK_SLIST,        /* streamed: is the key in the sorted S list (several shards: the owner's, through W.sviews) */
    LK_ROUTED,       /* one rank of a one-process-per-GPU job: keys it owns in its own S list; a candidate left
                      *   with a hit on a key owned elsewhere is parked (route_push) and settled once the owners
                      *   have answered                                                                         */
    LK_PARK          /* streamed, S list in host memory: no look-up at all; every candidate with a hit is parked
                      *   (route_push; each query tagged with its key's owner when the view has several shards,
                      *   which the one-process rounds ignore and a rank's routes by) and settled once the S
                      *   partitions have answered its queries                                                 */
  };

/* Routed pass 2 (DESIGN.md §4c, *Ranks*): a parked candidate goes to the view's pending list -- its meta, and its
 * key words as well when the sink lists pairs (KEY) -- and each of its keys owned by another rank becomes a query
 * to the owner, tagged owner << 32 | pending slot.  Two atomics per parked candidate: not a hot path.          */
template <int KW, bool KEY>
__device__ __forceinline__ void route_push(const SymmView &W, uint64_t x, uint64_t xl, uint64_t meta,
                                           bool fa, int oa, uint64_t rx, uint64_t rxl,
                                           bool fb, int ob, uint64_t ry, uint64_t ryl)
{ const unsigned long long nq = (fa ? 1ull : 0ull) + (fb ? 1ull : 0ull);
  const unsigned long long slot = atomicAdd(W.cand_n+SY_HDR_PEND,1ull), q = atomicAdd(W.cand_n+SY_HDR_QUERY,nq);
  if (slot >= W.pend_cap || q+nq > W.q_cap)
    { atomicOr(W.status,SY_STATUS_OVERFLOW); return; }
  W.pend[slot] = meta & ~(RV_HA | RV_HB);
  if (KEY)
    { W.pend_key[slot] = x;
      if (KW == 2) W.pend_lo[slot] = xl;
    }
  unsigned long long at = q;
  if (fa)
    { W.q_key[at] = rx; if (KW == 2) W.q_lo[at] = rxl;
      W.q_tag[at] = ((uint64_t) oa << 32) | slot; at++;
    }
  if (fb)
    { W.q_key[at] = ry; if (KW == 2) W.q_lo[at] = ryl;
      W.q_tag[at] = ((uint64_t) ob << 32) | slot;
    }
}

/* one candidate whose Bloom bits were set for rc x (RV_HA in its meta) and/or rc y (RV_HB): is it isolated
 * after all?  Exact.  LK_TABLE looks for an upper partner in the table: when the bucket prefix is no longer than
 * the run prefix (every table of more than a few entries) both buckets' offsets are loaded at once and then
 * RV_PROBE keys and counts of a bucket at once, two dependent accesses instead of one per key.  LK_SLIST and
 * LK_ROUTED look the key up in an S list (keys / bucket: the sorted list and its index); a candidate LK_ROUTED
 * parks is not isolated here, and it is parked with its key words when the sink lists pairs.                 */
template <typename IdxT, int KW, Lookup LK, class Sink>
__device__ __forceinline__ bool isolated_after_all(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                                                   const uint16_t *__restrict__ cnt, int64_t n,
                                                   const IdxT *__restrict__ bucket, int bshift, int kmer,
                                                   const SymmView &W, uint64_t x, uint64_t xl, uint64_t meta)
{ const int  cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff);
  const int  p  = (int) ((meta >> 32) & 0xff), yb = (int) ((meta >> 40) & 3);
  const bool ha = (meta & RV_HA) != 0, hb = (meta & RV_HB) != 0;
  uint64_t rx, rxl, ry, ryl;
  revcomp_kmer<KW>(x,xl,kmer,rx,rxl);
  ry = rx; ryl = rxl;
  set_base<KW>(ry,ryl,kmer-1-p,3-yb);                      /* rc y = rc x with the mirrored base swapped */
  if (LK == LK_PARK)
    { const int oa = (ha && W.n_seg > 1) ? owner_of(W,rx) : W.self, ob = (hb && W.n_seg > 1) ? owner_of(W,ry) : W.self;
      route_push<KW,Sink::NEEDS_KEY>(W,x,xl,meta,ha,oa,rx,rxl,hb,ob,ry,ryl);
      return false;
    }
  if (LK == LK_ROUTED)
    { const int  oa = (ha && W.n_seg > 1) ? owner_of(W,rx) : W.self, ob = (hb && W.n_seg > 1) ? owner_of(W,ry) : W.self;
      if ((ha && oa == W.self && bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,rx,rxl) >= 0) ||
          (hb && ob == W.self && bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,ry,ryl) >= 0))
        return false;
      const bool fa = ha && oa != W.self, fb = hb && ob != W.self;
      if (!fa && !fb)
        return true;
      route_push<KW,Sink::NEEDS_KEY>(W,x,xl,meta,fa,oa,rx,rxl,fb,ob,ry,ryl);
      return false;
    }
  if (LK == LK_SLIST && W.n_seg > 1)                       /* several shards: the S list of the key's owner */
    { if (ha)
        { const hm_stream_sview &a = W.sviews[owner_of(W,rx)];
          if (bucket_find<IdxT,KW>(a.s_key,a.s_lo,(const IdxT *) a.s_bucket,64-a.bits,rx,rxl) >= 0)
            return false;
        }
      if (hb)
        { const hm_stream_sview &b = W.sviews[owner_of(W,ry)];
          if (bucket_find<IdxT,KW>(b.s_key,b.s_lo,(const IdxT *) b.s_bucket,64-b.bits,ry,ryl) >= 0)
            return false;
        }
      return true;
    }
  if (LK == LK_SLIST)
    return !((ha && bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,rx,rxl) >= 0) ||
             (hb && bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,ry,ryl) >= 0));
  const int Pr = kmer >> 1, pup = kmer-Pr, psh = 64-2*Pr;
  if (bshift >= psh)
    { int64_t la = 0, ra = 0, lb = 0, rb = 0;
      if (ha) { const uint64_t bk = rx >> bshift; la = (int64_t) bucket[bk]; ra = (int64_t) bucket[bk+1]; }
      if (hb) { const uint64_t bk = ry >> bshift; lb = (int64_t) bucket[bk]; rb = (int64_t) bucket[bk+1]; }
      if (ha) RVP_BUCKET(ra-la);
      if (hb) RVP_BUCKET(rb-lb);
      if (ra-la <= 48 && rb-lb <= 48)
        { bool found;
          if (ha)
            { const bool up = bucket_upper_partner<KW>(keys,keys_lo,cnt,la,ra,psh,pup,rx,rxl,cx,found);
              if (!found)
                atomicOr(W.status,SY_STATUS_ASYMMETRIC);
              if (up)
                return false;
            }
          if (hb)
            { const bool up = bucket_upper_partner<KW>(keys,keys_lo,cnt,lb,rb,psh,pup,ry,ryl,cy,found);
              if (!found)
                atomicOr(W.status,SY_STATUS_ASYMMETRIC);
              if (up)
                return false;
            }
          return true;
        }
    }
  RVP_COUNT(RVP_GEN,1)
  if (ha && has_upper_partner<IdxT,KW>(keys,keys_lo,cnt,n,bucket,bshift,kmer,rx,rxl,cx,W.status))
    return false;
  if (hb && has_upper_partner<IdxT,KW>(keys,keys_lo,cnt,n,bucket,bshift,kmer,ry,ryl,cy,W.status))
    return false;
  return true;
}

__device__ __forceinline__ void count_pair(uint32_t *tile, unsigned long long *__restrict__ plot,
                                           uint64_t meta, int kmer)
{ const int cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff);
  const int p  = (int) ((meta >> 32) & 0xff);
  const unsigned wgt = (2*p == kmer-1) ? 1u : 2u;          /* middle base: the mirror pair is found itself */
  const int s = cx+cy;
  const int m = cx < cy ? cx : cy;
  if (s < RV_TS && m < RV_TM)
    atomicAdd(tile + s*RV_TROW + m, wgt);
  else
    atomicAdd(plot + s*HM_PLOT_W + m, (unsigned long long) wgt);
}

/* extract_kmer_pairs' records of isolated candidates (warp-wide call; lab = the candidate's pixel label, 0 for
 * lanes that list nothing).  A candidate (x < y, differing at p, bases bx < by, counts cx, cy) stands for the
 * pair itself and, unless 2p = k-1, its mirror image (u, v) = (rc y, rc x) at p' = k-1-p with cu = cy, cv = cx
 * -- a pair of its own that the direct passes find from u.  Each is listed as pass2_extract_kernel lists it: the
 * member with the higher count (the lower one on a tie), the other member's base at the varying position.
 * One atomic per warp on the counter, which counts every record, also those beyond cap.                    */
/* list_pairs' records one at a time, for PrefixSink: how many a candidate lists, and the candidate's own record
 * (mirror = false) or its mirror image's (mirror = true).  list_pairs keeps its own inline copy, so that the
 * listing kernels compile as they did; the pair-file tests compare the two byte for byte.                      */
template <int KW>
__device__ __forceinline__ int pair_records(uint64_t meta, unsigned lab, int kmer)
{ const int p = (int) ((meta >> 32) & 0xff);
  return lab == 0 ? 0 : (2*p == kmer-1 ? 1 : 2);
}

template <int KW>
__device__ __forceinline__ hm_pair_rec pair_record(uint64_t x, uint64_t xl, uint64_t meta, unsigned lab, int kmer,
                                                   bool mirror)
{ const int cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff);
  const int p  = (int) ((meta >> 32) & 0xff), by = (int) ((meta >> 40) & 3);
  const int bx = base_at<KW>(x,xl,p);
  hm_pair_rec r;
  r.smudge = lab; r.pad = 0;
  if (!mirror)
    { r.pos = (uint8_t) p;
      if (cx < cy)                                         /* y, alt bx */
        { uint64_t y = x, yl = xl;
          set_base<KW>(y,yl,p,by);
          r.key_hi = y; r.key_lo = yl; r.alt = (uint8_t) bx;
        }
      else                                                 /* x, alt by */
        { r.key_hi = x; r.key_lo = xl; r.alt = (uint8_t) by; }
      return r;
    }
  const int q = kmer-1-p;
  uint64_t  rx, rxl;
  revcomp_kmer<KW>(x,xl,kmer,rx,rxl);
  r.pos = (uint8_t) q;
  if (cy < cx)                                             /* v = rc x, alt = u's base 3-by */
    { r.key_hi = rx; r.key_lo = rxl; r.alt = (uint8_t) (3-by); }
  else                                                     /* u = rc y, alt = v's base 3-bx */
    { set_base<KW>(rx,rxl,q,3-by);
      r.key_hi = rx; r.key_lo = rxl; r.alt = (uint8_t) (3-bx);
    }
  return r;
}

template <int KW>
__device__ __forceinline__ void list_pairs(uint64_t x, uint64_t xl, uint64_t meta, unsigned lab, int kmer,
                                           hm_pair_rec *__restrict__ out, unsigned long long cap,
                                           unsigned long long *__restrict__ count, int lane, unsigned lt)
{ const int      cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff);
  const int      p  = (int) ((meta >> 32) & 0xff), by = (int) ((meta >> 40) & 3);
  const int      nr = lab == 0 ? 0 : (2*p == kmer-1 ? 1 : 2);
  const unsigned b1 = __ballot_sync(0xffffffffu,nr >= 1), b2 = __ballot_sync(0xffffffffu,nr == 2);
  if (b1 == 0)
    return;
  unsigned long long at = 0;
  if (lane == 0)
    at = atomicAdd(count,(unsigned long long) (__popc(b1)+__popc(b2)));
  at = __shfl_sync(0xffffffffu,at,0) + (unsigned long long) (__popc(b1 & lt)+__popc(b2 & lt));
  if (nr == 0)
    return;
  const int bx = base_at<KW>(x,xl,p);
  hm_pair_rec r;
  r.smudge = lab; r.pad = 0;
  r.pos = (uint8_t) p;
  if (cx < cy)                                             /* y, alt bx */
    { uint64_t y = x, yl = xl;
      set_base<KW>(y,yl,p,by);
      r.key_hi = y; r.key_lo = yl; r.alt = (uint8_t) bx;
    }
  else                                                     /* x, alt by */
    { r.key_hi = x; r.key_lo = xl; r.alt = (uint8_t) by; }
  if (at < cap)
    out[at] = r;
  if (nr == 2)
    { const int q = kmer-1-p;
      uint64_t  rx, rxl;
      revcomp_kmer<KW>(x,xl,kmer,rx,rxl);
      r.pos = (uint8_t) q;
      if (cy < cx)                                         /* v = rc x, alt = u's base 3-by */
        { r.key_hi = rx; r.key_lo = rxl; r.alt = (uint8_t) (3-by); }
      else                                                 /* u = rc y, alt = v's base 3-bx */
        { set_base<KW>(rx,rxl,q,3-by);
          r.key_hi = rx; r.key_lo = rxl; r.alt = (uint8_t) (3-bx);
        }
      if (at+1 < cap)
        out[at+1] = r;
    }
}

extern __shared__ __align__(16) uint64_t rv_smem[];     /* pass 2's dynamic shared memory (resolve / extract_kernel) */

/* What pass 2 does with a candidate once it is known whether it is isolated.  take() is called by every lane of
 * a warp at once, with iso = false where a lane has nothing to give; begin() and end() by every thread of the
 * CTA before and after its sweep.  NEEDS_KEY: take() uses the candidate's key words, so the routed pass parks
 * them with the candidate.  QUEUES: where the warps' queues start in rv_smem.                                */
struct CountSink                                 /* the plot: resolve_kernel */
  { uint32_t *tile;                              /* the CTA's shared-memory plot tile: RV_TS x RV_TROW counters */
    unsigned long long *plot;
    int kmer;
    static constexpr bool NEEDS_KEY = false;
    static constexpr int  QUEUES = RV_TS*RV_TROW/2;     /* after the tile */
    __device__ __forceinline__ void begin() const
    { for (int t = threadIdx.x; t < RV_TS*RV_TROW; t += blockDim.x)
        tile[t] = 0;
      __syncthreads();
    }
    __device__ __forceinline__ void take(bool iso, uint64_t, uint64_t, uint64_t meta) const
    { if (iso)
        count_pair(tile,plot,meta,kmer);
    }
    __device__ __forceinline__ void end() const
    { __syncthreads();
      for (int t = threadIdx.x; t < RV_TS*RV_TROW; t += blockDim.x)
        { uint32_t v = tile[t];
          if (v != 0)                                    /* (column RV_TM is padding: always 0) */
            atomicAdd(plot + (t/RV_TROW)*HM_PLOT_W + (t%RV_TROW), (unsigned long long) v);
        }
    }
  };

template <int KW>
struct ListSink                                  /* extract_kmer_pairs' records: extract_kernel */
  { const uint16_t *pixmap;
    hm_pair_rec *out;
    unsigned long long cap, *count;
    int kmer;
    static constexpr bool NEEDS_KEY = true;
    static constexpr int  QUEUES = 0;
    __device__ __forceinline__ void begin() const {}
    __device__ __forceinline__ void end() const {}
    __device__ __forceinline__ void take(bool iso, uint64_t x, uint64_t xl, uint64_t meta) const
    { const int lane = threadIdx.x & 31;
      unsigned  lab = 0;
      if (iso)
        { const int cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff);
          lab = __ldg(pixmap + (cx+cy)*HM_PLOT_W + (cx < cy ? cx : cy));
        }
      list_pairs<KW>(x,xl,meta,lab,kmer,out,cap,count,lane,(1u << lane) - 1);
    }
  };

/* The records ListSink would list, by key prefix (the top hb bits of key_hi, as pairs_hist_kernel bins them):
 * HIST = true adds each to hist[prefix] (one atomic per distinct prefix of a warp); HIST = false stores only
 * those with p0 <= prefix < p1 into out, one atomic per warp on the counter, which counts past cap          */
template <int KW, bool HIST>
struct PrefixSink
  { const uint16_t *pixmap;
    unsigned long long *hist;
    hm_pair_rec *out;
    unsigned long long cap, *count;
    uint64_t p0, p1;
    int kmer, hb;
    static constexpr bool NEEDS_KEY = true;
    static constexpr int  QUEUES = 0;
    __device__ __forceinline__ void begin() const {}
    __device__ __forceinline__ void end() const {}
    __device__ __forceinline__ void take(bool iso, uint64_t x, uint64_t xl, uint64_t meta) const
    { const int lane = threadIdx.x & 31;
      unsigned  lab = 0;
      if (iso)
        { const int cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff);
          lab = __ldg(pixmap + (cx+cy)*HM_PLOT_W + (cx < cy ? cx : cy));
        }
      const int   nr = pair_records<KW>(meta,lab,kmer);
      hm_pair_rec r0, r1;
      uint64_t    f0 = 0, f1 = 0;
      if (nr >= 1) { r0 = pair_record<KW>(x,xl,meta,lab,kmer,false); f0 = r0.key_hi >> (64-hb); }
      if (nr == 2) { r1 = pair_record<KW>(x,xl,meta,lab,kmer,true);  f1 = r1.key_hi >> (64-hb); }
      if (HIST)
        { warp_count(hist,nr >= 1,f0);
          warp_count(hist,nr == 2,f1);
          return;
        }
      const bool     in0 = nr >= 1 && f0 >= p0 && f0 < p1, in1 = nr == 2 && f1 >= p0 && f1 < p1;
      const unsigned b0 = __ballot_sync(0xffffffffu,in0), b1 = __ballot_sync(0xffffffffu,in1);
      if ((b0 | b1) == 0)
        return;
      const unsigned lt = (1u << lane) - 1;
      unsigned long long at = 0;
      if (lane == 0)
        at = atomicAdd(count,(unsigned long long) (__popc(b0)+__popc(b1)));
      at = __shfl_sync(0xffffffffu,at,0) + (unsigned long long) (__popc(b0 & lt)+__popc(b1 & lt));
      if (in0 && at < cap)
        out[at] = r0;
      at += in0;
      if (in1 && at < cap)
        out[at] = r1;
    }
  };

/* Pass 2 over the view's candidates.  Candidates whose Bloom look-up misses (~95 %) go to the sink at once.
 * The others need the exact answer, and a warp in which one lane does that stalls all 32: they are parked in
 * the warp's queue in shared memory (RV_QCAP records of KW+1 words) -- the whole record, with the two Bloom
 * answers in its meta -- and settled 32 at a time, every lane busy, without reading the record or the filter
 * again.  RV_ILP candidates per thread and trip keep that many record / Bloom loads in flight (the sweep is
 * bound by latency: record -> Bloom word, and for the hits bucket offsets -> keys, not by bytes or
 * instructions).                                                                                            */
template <typename IdxT, int KW, Lookup LK, class Sink>
__device__ __forceinline__ void sweep(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                                      const uint16_t *__restrict__ cnt, int64_t n, const IdxT *__restrict__ bucket,
                                      int bshift, int kmer, const SymmView &W, const Sink &sink)
{ const unsigned FULL = 0xffffffffu;
  const int      lane = threadIdx.x & 31;
  const unsigned lt   = (1u << lane) - 1;
  uint64_t *qk = rv_smem + Sink::QUEUES + (threadIdx.x >> 5)*RV_QCAP*(KW+1);   /* this warp's queue */
  uint64_t *ql = qk + (KW == 2 ? RV_QCAP : 0);
  uint64_t *qm = qk + KW*RV_QCAP;
  int       qn = 0;
  sink.begin();
  unsigned long long ncl = *W.cand_n;
  if (ncl > W.cand_cap) ncl = W.cand_cap;
  const int64_t nc     = (int64_t) ncl;
  const int64_t stride = (int64_t) gridDim.x * blockDim.x;
  const int64_t first  = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  for (uint32_t it = 0; first-lane + (int64_t) it*RV_ILP*stride < nc; it++)
    { uint64_t x[RV_ILP], xl[RV_ILP], meta[RV_ILP];
      uint64_t *wa[RV_ILP], *wb[RV_ILP], ba[RV_ILP], bb[RV_ILP], va[RV_ILP], vb[RV_ILP];
      bool     ok[RV_ILP];
#pragma unroll
      for (int u = 0; u < RV_ILP; u++)
        { const int64_t i = first + ((int64_t) it*RV_ILP+u)*stride;
          ok[u] = (i < nc);
          x[u] = 0; xl[u] = 0; meta[u] = 0;
          if (ok[u])
            { x[u] = ld_stream(W.cand_key+i);
              if (KW == 2) xl[u] = ld_stream(W.cand_lo+i);
              meta[u] = ld_stream(W.cand_meta+i);
            }
        }
#ifdef RESOLVE_PROBE
      if (RVP_MODE == 1)
        { uint64_t d = 0;
          for (int u = 0; u < RV_ILP; u++) d ^= x[u] ^ xl[u] ^ meta[u];
          if (d == 0x5eedull) atomicOr(W.status,0ull);            /* keeps the loads */
          continue;
        }
#endif
#pragma unroll
      for (int u = 0; u < RV_ILP; u++)
        { const int p  = (int) ((meta[u] >> 32) & 0xff), yb = (int) ((meta[u] >> 40) & 3);
          uint64_t rx, rxl, ry, ryl;
          revcomp_kmer<KW>(x[u],xl[u],kmer,rx,rxl);
          ry = rx; ryl = rxl;
          set_base<KW>(ry,ryl,kmer-1-p,3-yb);
          bloom_slot<KW>(W,W.n_seg > 1 ? owner_of(W,rx) : 0,kmer,rx,rxl,wa[u],ba[u]);
          bloom_slot<KW>(W,W.n_seg > 1 ? owner_of(W,ry) : 0,kmer,ry,ryl,wb[u],bb[u]);
        }
#pragma unroll
      for (int u = 0; u < RV_ILP; u++)
        { va[u] = 0; vb[u] = 0;
          if (ok[u])
            { va[u] = ld_keep(wa[u]);
              vb[u] = (wb[u] == wa[u]) ? va[u] : ld_keep(wb[u]);   /* one shard owns both: the same word */
            }
        }
#pragma unroll
      for (int u = 0; u < RV_ILP; u++)
        { const bool ha = (va[u] & ba[u]) == ba[u], hb = (vb[u] & bb[u]) == bb[u];
          bool hit = ok[u] && (ha || hb);
          RVP_COUNT(RVP_CAND,ok[u]) RVP_COUNT(RVP_HA,hit && !hb) RVP_COUNT(RVP_HB,hit && !ha) RVP_COUNT(RVP_HAB,hit && ha && hb)
          sink.take(ok[u] && !hit,x[u],xl[u],meta[u]);
          if (RVP_MODE == 2) hit = false;                        /* not isolated, not checked */
          const unsigned bal = __ballot_sync(FULL,hit);
          if (hit)
            { const int at = qn + __popc(bal & lt);
              qk[at] = x[u];
              if (KW == 2) ql[at] = xl[u];
              qm[at] = meta[u] | (ha ? RV_HA : 0) | (hb ? RV_HB : 0);
            }
          qn += __popc(bal);
        }
      __syncwarp();
      while (qn >= 32)
        { qn -= 32;
          uint64_t       xx = qk[qn+lane], xxl = KW == 2 ? ql[qn+lane] : 0;
          const uint64_t mm = qm[qn+lane];
          if (!Sink::NEEDS_KEY)                    /* the next trip refills the slots once every lane has read them */
            __syncwarp();
          const bool iso = isolated_after_all<IdxT,KW,LK,Sink>(keys,keys_lo,cnt,n,bucket,bshift,kmer,W,xx,xxl,mm);
          if (Sink::NEEDS_KEY)                     /* the key words again: not live across the exact check */
            { xx = qk[qn+lane]; xxl = KW == 2 ? ql[qn+lane] : 0; }
          sink.take(iso,xx,xxl,mm);
          if (Sink::NEEDS_KEY)
            __syncwarp();
        }
    }
  uint64_t xx = 0, xxl = 0, mm = 0;
  bool     iso = false;
  if (lane < qn)
    { xx = qk[lane]; xxl = KW == 2 ? ql[lane] : 0; mm = qm[lane];
      iso = isolated_after_all<IdxT,KW,LK,Sink>(keys,keys_lo,cnt,n,bucket,bshift,kmer,W,xx,xxl,mm);
    }
  sink.take(iso,xx,xxl,mm);
  sink.end();
}

/* pass 2's grid: `want` CTAs, at most `most`; HETMERS_PASS2_CTAS=g caps it at g (each CTA then strides over more
 * candidates: tests) */
static int rv_grid(int64_t want, int64_t most)
{ const char *e = getenv("HETMERS_PASS2_CTAS");
  if (e != NULL && atoi(e) >= 1 && atoi(e) < most)
    most = atoi(e);
  return (int) (want < most ? (want > 0 ? want : 1) : most);
}

/* Pass 2 of the plot: sweep with the count sink.  One CTA of 1024 threads per SM: one plot tile per SM, the rest of
 * shared memory holds the queues.                                                                             */
template <typename IdxT, int KW, Lookup LK>
__global__ void __launch_bounds__(RV_THREADS,1)
resolve_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
               const uint16_t *__restrict__ cnt, int64_t n, const IdxT *__restrict__ bucket, int bshift,
               int kmer, const SymmView W, unsigned long long *__restrict__ plot)
{ const CountSink sink = { (uint32_t *) rv_smem, plot, kmer };
  sweep<IdxT,KW,LK>(keys,keys_lo,cnt,n,bucket,bshift,kmer,W,sink);
}

template <typename IdxT, int KW, Lookup LK = LK_TABLE>
static cudaError_t launch_resolve(const uint64_t *keys, const uint64_t *keys_lo, const uint16_t *cnt, int64_t n,
                                  const void *bucket, int bits, int kmer, const SymmView &W,
                                  unsigned long long *plot, int64_t range, cudaStream_t st)
{ static int configured[64] = {0};                            /* per instantiation */
  size_t smem = (size_t) RV_TS*RV_TROW*sizeof(uint32_t) + (size_t) (RV_THREADS/32)*RV_QCAP*8*(KW+1);   /* 121 KB / 145 KB */
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  if (dev >= 64 || !configured[dev])
    { cudaError_t e = cudaFuncSetAttribute(resolve_kernel<IdxT,KW,LK>,cudaFuncAttributeMaxDynamicSharedMemorySize,(int) smem);
      if (e != cudaSuccess) return e;
      if (dev < 64) configured[dev] = 1;
    }
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  int64_t want = (range/8+RV_THREADS-1)/RV_THREADS;            /* ~1 candidate per 10 entries */
  int     grid = rv_grid(want,sms);
  resolve_kernel<IdxT,KW,LK><<<grid,RV_THREADS,smem,st>>>(keys,keys_lo,cnt,n,(const IdxT *) bucket,64-bits,kmer,W,plot);
  return cudaGetLastError();
}

extern "C" int hm_k_symm_resolve(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                                 const void *d_bucket, int bits, int idx64, int kmer,
                                 void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards,
                                 unsigned long long *d_plot, void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || d_work == NULL || layout == NULL || d_plot == NULL)
    return hm_set_error(HM_EINVAL,"symm_resolve: bad arguments");
  if ((kmer > 32) != (d_keys_lo != NULL))
    return hm_set_error(HM_EINVAL,"symm_resolve: second key word array %s for k=%d",
                        d_keys_lo ? "given" : "missing",kmer);
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = make_view(d_work,layout,shards);
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { return launch_resolve<typename decltype(I)::IdxT,decltype(I)::KW>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,W,
                                                                       d_plot,layout->range,st); });
  if (l2_persist())
    bloom_window(st,NULL,0,0);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"resolve_kernel");
  return HM_OK;
}

/* ------------------------------------------------------------------ pair listing -------- */

#define EX_THREADS 512              /* k <= 32: 2 CTAs per SM (64 registers); k > 32 spilled at 64 registers: 1 CTA,
                                     * and so did the routed listing at k <= 32: 1 CTA                              */

/* extract_kmer_pairs on the symmetric scan's work area: sweep with the list sink over the view's candidates (a
 * slice of them: slice_view), so an isolated candidate whose pixel carries a label is listed instead of counted.
 * No plot tile: shared memory holds only the queues.
 * LK_ROUTED: the routed listing of one rank (DESIGN.md §4c, *Ranks*), with its sorted S list and S index as keys /
 * bucket; route_list_kernel lists the candidates it parks once the owners have answered.                     */
template <typename IdxT, int KW, Lookup LK>
__global__ void __launch_bounds__(EX_THREADS,KW == 1 && LK == LK_TABLE ? 2 : 1)
extract_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
               const uint16_t *__restrict__ cnt, int64_t n, const IdxT *__restrict__ bucket, int bshift,
               int kmer, const SymmView W, const uint16_t *__restrict__ pixmap,
               hm_pair_rec *__restrict__ out, unsigned long long cap, unsigned long long *__restrict__ count)
{ const ListSink<KW> sink = { pixmap, out, cap, count, kmer };
  sweep<IdxT,KW,LK>(keys,keys_lo,cnt,n,bucket,bshift,kmer,W,sink);
}

template <typename IdxT, int KW, Lookup LK = LK_TABLE>
static cudaError_t launch_extract(const uint64_t *keys, const uint64_t *keys_lo, const uint16_t *cnt, int64_t n,
                                  const void *bucket, int bits, int kmer, const SymmView &W,
                                  const uint16_t *pixmap, hm_pair_rec *out, int64_t cap, unsigned long long *count,
                                  cudaStream_t st)
{ static int per_sm[64] = {0};                                /* per instantiation */
  size_t smem = (size_t) (EX_THREADS/32)*RV_QCAP*8*(KW+1);       /* 24 KB / 36 KB */
  int dev = 0, sms = 132, occ = 1;
  cudaGetDevice(&dev);
  if (dev >= 64 || per_sm[dev] == 0)                           /* one wave of resident CTAs */
    { cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ,extract_kernel<IdxT,KW,LK>,EX_THREADS,smem);
      if (e != cudaSuccess) return e;
      if (occ < 1) occ = 1;
      if (dev < 64) per_sm[dev] = occ;
    }
  else
    occ = per_sm[dev];
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  int64_t want = ((int64_t) W.cand_cap+EX_THREADS*RV_ILP-1)/(EX_THREADS*RV_ILP);
  int     grid = rv_grid(want,(int64_t) sms*occ);
  extract_kernel<IdxT,KW,LK><<<grid,EX_THREADS,smem,st>>>(keys,keys_lo,cnt,n,(const IdxT *) bucket,64-bits,kmer,W,
                                                          pixmap,out,(unsigned long long) cap,count);
  return cudaGetLastError();
}

/* the candidates [c0, c1) of a view as its whole list: pass 2 reads min(header count, cand_cap) records from
 * cand_key, so the header's count (of all candidates) must reach c1 unless c0 = 0                          */
static SymmView slice_view(SymmView W, int64_t c0, int64_t c1)
{ W.cand_key += c0; W.cand_meta += c0;
  if (W.cand_lo != NULL) W.cand_lo += c0;
  W.cand_cap = (unsigned long long) (c1-c0);
  return W;
}

extern "C" int hm_k_symm_extract(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                                 const void *d_bucket, int bits, int idx64, int kmer,
                                 void *d_work, const hm_symm_layout *layout, const hm_symm_shards *shards,
                                 const uint16_t *d_pixmap, int64_t c0, int64_t c1, hm_pair_rec *d_out, int64_t cap,
                                 unsigned long long *d_count, void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || d_work == NULL || layout == NULL || d_pixmap == NULL ||
      d_count == NULL || c0 < 0 || c1 < c0 || cap < 0 || (cap > 0 && d_out == NULL))
    return hm_set_error(HM_EINVAL,"symm_extract: bad arguments");
  if ((kmer > 32) != (d_keys_lo != NULL))
    return hm_set_error(HM_EINVAL,"symm_extract: second key word array %s for k=%d",
                        d_keys_lo ? "given" : "missing",kmer);
  if (c1 > layout->cand_cap)
    c1 = layout->cand_cap;
  if (c1 <= c0)
    return HM_OK;
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = slice_view(make_view(d_work,layout,shards),c0,c1);
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { return launch_extract<typename decltype(I)::IdxT,decltype(I)::KW>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,W,
                                                                       d_pixmap,d_out,cap,d_count,st); });
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"extract_kernel");
  return HM_OK;
}

/* extract_kernel's sweep with a PrefixSink: the pair files' histogram (HIST) and window sweeps (DESIGN.md §6c).
 * The window sweep at k <= 32 spills at 64 registers (2 CTAs per SM): it runs 1 CTA per SM, as k > 32 does.  */
template <typename IdxT, int KW, bool HIST>
__global__ void __launch_bounds__(EX_THREADS,KW == 1 && HIST ? 2 : 1)
pairs_sweep_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                   const uint16_t *__restrict__ cnt, int64_t n, const IdxT *__restrict__ bucket, int bshift,
                   int kmer, const SymmView W, const PrefixSink<KW,HIST> sink)
{ sweep<IdxT,KW,LK_TABLE>(keys,keys_lo,cnt,n,bucket,bshift,kmer,W,sink); }

template <typename IdxT, int KW, bool HIST>
static cudaError_t launch_pairs_sweep(const uint64_t *keys, const uint64_t *keys_lo, const uint16_t *cnt, int64_t n,
                                      const void *bucket, int bits, int kmer, const SymmView &W,
                                      const PrefixSink<KW,HIST> &sink, cudaStream_t st)
{ static int per_sm[64] = {0};                                /* per instantiation */
  size_t smem = (size_t) (EX_THREADS/32)*RV_QCAP*8*(KW+1);
  int dev = 0, sms = 132, occ = 1;
  cudaGetDevice(&dev);
  if (dev >= 64 || per_sm[dev] == 0)
    { cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ,pairs_sweep_kernel<IdxT,KW,HIST>,EX_THREADS,smem);
      if (e != cudaSuccess) return e;
      if (occ < 1) occ = 1;
      if (dev < 64) per_sm[dev] = occ;
    }
  else
    occ = per_sm[dev];
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  int64_t want = ((int64_t) W.cand_cap+EX_THREADS*RV_ILP-1)/(EX_THREADS*RV_ILP);
  int     grid = rv_grid(want,(int64_t) sms*occ);
  pairs_sweep_kernel<IdxT,KW,HIST><<<grid,EX_THREADS,smem,st>>>(keys,keys_lo,cnt,n,(const IdxT *) bucket,64-bits,kmer,
                                                                W,sink);
  return cudaGetLastError();
}

int hm_symm_pairs_sweep(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                        const void *d_bucket, int bits, int idx64, int kmer, void *d_work,
                        const hm_symm_layout *layout, const hm_symm_shards *shards,
                        const uint16_t *d_pixmap, int hb, unsigned long long *d_hist, uint64_t p0,
                        uint64_t p1, hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count,
                        void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || d_work == NULL || layout == NULL || d_pixmap == NULL ||
      hb < 1 || hb > 2*kmer || hb > 32 || cap < 0 || (d_hist == NULL && (d_count == NULL || (cap > 0 && d_out == NULL))))
    return hm_set_error(HM_EINVAL,"symm_pairs_sweep: bad arguments");
  if ((kmer > 32) != (d_keys_lo != NULL))
    return hm_set_error(HM_EINVAL,"symm_pairs_sweep: second key word array %s for k=%d",
                        d_keys_lo ? "given" : "missing",kmer);
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = make_view(d_work,layout,shards);
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { using IdxT = typename decltype(I)::IdxT;
      constexpr int KW = decltype(I)::KW;
      if (d_hist != NULL)
        { const PrefixSink<KW,true> sink = { d_pixmap, d_hist, NULL, 0, NULL, 0, 0, kmer, hb };
          return launch_pairs_sweep<IdxT,KW,true>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,W,sink,st);
        }
      const PrefixSink<KW,false> sink = { d_pixmap, NULL, d_out, (unsigned long long) cap, d_count, p0, p1, kmer, hb };
      return launch_pairs_sweep<IdxT,KW,false>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,W,sink,st); });
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"pairs_sweep_kernel");
  return HM_OK;
}

/* candidate count + status word of the last runscan/resolve on this work area (synchronises) */
extern "C" int hm_symm_status(const void *d_work, const hm_symm_layout *layout, uint64_t *n_cand,
                              uint64_t *status, void *stream)
{ uint64_t h[2] = {0,0};
  HM_CUDA(cudaMemcpyAsync(h,(const uint8_t *) d_work + layout->off_header,sizeof(h),cudaMemcpyDeviceToHost,
                          (cudaStream_t) stream));
  HM_CUDA(cudaStreamSynchronize((cudaStream_t) stream));
  if (n_cand != NULL) *n_cand = h[SY_HDR_CAND];
  if (status != NULL) *status = h[SY_HDR_STATUS];
  return HM_OK;
}

/* Move a proposed shard cut to the next run boundary at or after it (a run = entries sharing their
 * first k/2 bases): pairs found by the run scan then never straddle two shards.                 */
extern "C" int hm_symm_align_cut(const uint64_t *d_keys, int64_t n, int kmer, int64_t cut, int64_t *out)
{ if (d_keys == NULL || out == NULL || cut < 0 || cut > n || kmer < HM_SYMM_MIN_KMER)
    return hm_set_error(HM_EINVAL,"hm_symm_align_cut: bad arguments");
  const int psh = 64-2*(kmer>>1);
  if (cut == 0 || cut == n)
    { *out = cut; return HM_OK; }
  uint64_t prev, buf[4096];
  HM_CUDA(cudaMemcpy(&prev,d_keys+cut-1,sizeof(uint64_t),cudaMemcpyDeviceToHost));
  while (cut < n)
    { int64_t m = n-cut < 4096 ? n-cut : 4096;
      HM_CUDA(cudaMemcpy(buf,d_keys+cut,sizeof(uint64_t)*(size_t) m,cudaMemcpyDeviceToHost));
      for (int64_t i = 0; i < m; i++)
        if (((buf[i] ^ prev) >> psh) != 0)
          { *out = cut+i; return HM_OK; }
      cut += m;
    }
  *out = n;
  return HM_OK;
}

/* ------------------------------------------------------------------ streamed scan -------- */
/* The table passes through the GPU chunk by chunk (hm_scan.cu drives it, DESIGN.md §4c).  The work area of
 * hm_symm_plan(n, 0, kmer, 1) supplies the header and the whole-table Bloom filter (only they are used); the
 * run list of one chunk, the candidate records and the S list are arrays of the caller's, the last two
 * resident and grown between chunks.  Several shards: hm_symm_plan(n, 0, kmer, G) -- shard r fills segment r,
 * the caller all-gathers the segments before pass 2; n_seg of the view is the shards' descriptor's (the
 * shards up to the last non-empty one), so that no key is owned by an empty shard at the end.           */
static SymmView stream_view(void *d_work, const hm_symm_layout *L, const hm_stream_lists *R, const hm_symm_shards *sh)
{ SymmView W = make_view(d_work,L,NULL);
  W.n_seg = 1;
  if (sh != NULL && sh->n_seg > 1)
    { W.n_seg = sh->n_seg; W.self = sh->self;
      for (int r = 0; r < sh->n_seg; r++) W.first_key[r] = sh->first_key[r];
    }
  else if (sh != NULL)
    W.self = sh->self;
  W.cand_key = R->cand_key; W.cand_lo = R->cand_lo; W.cand_meta = R->cand_meta;
  W.cand_cap = (unsigned long long) R->cand_cap;
  W.runs = R->runs; W.runs_cap = (unsigned long long) R->runs_cap;
  W.s_key = R->s_key; W.s_lo = R->s_lo; W.s_cap = (unsigned long long) R->s_cap;
  return W;
}

int hm_symm_stream_begin(void *d_work, const hm_symm_layout *L, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  SymmView W = make_view(d_work,L,NULL);
  size_t bloom_bytes = sizeof(uint32_t)*(size_t) W.seg_words*(size_t) L->n_seg;   /* every segment */
  HM_CUDA(cudaMemsetAsync(W.cand_n,0,256,st));
  HM_CUDA(cudaMemsetAsync(W.bloom,0,bloom_bytes,st));
  if (l2_persist())
    bloom_window(st,W.bloom,bloom_bytes,1);
  return HM_OK;
}

int hm_symm_stream_chunk(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                                    int64_t n, const void *d_bucket, int bits, int kmer, int64_t hi,
                                    void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                                    const hm_symm_shards *shards, void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || hi < 0 || hi > n || bits < 1 || bits > 30 ||
      (kmer > 32) != (d_keys_lo != NULL) || (shards != NULL && (shards->self < 0 || shards->self >= L->n_seg ||
                                                                shards->n_seg > L->n_seg)))
    return hm_set_error(HM_EINVAL,"symm_stream_chunk: bad arguments (k=%d, %lld of %lld entries)",
                        kmer,(long long) hi,(long long) n);
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = stream_view(d_work,L,R,shards);
  HM_CUDA(cudaMemsetAsync(W.runs_n,0,sizeof(uint64_t),st));                 /* the run list is per chunk */
  if (hi == 0)
    return HM_OK;
  cudaError_t e;
  if (kmer <= 32)
    { e = launch_runscan<uint32_t,1,true>(d_keys,NULL,d_cnt,n,d_bucket,bits,kmer,0,hi,W,st);
      if (e == cudaSuccess) e = launch_runs<uint32_t,1,true>(d_keys,NULL,d_cnt,n,d_bucket,bits,kmer,0,hi,W,st);
    }
  else
    { e = launch_runscan<uint32_t,2,true>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,0,hi,W,st);
      if (e == cudaSuccess) e = launch_runs<uint32_t,2,true>(d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,kmer,0,hi,W,st);
    }
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"runscan_kernel / runs_kernel (streamed)");
  return HM_OK;
}

/* header words: candidates so far, status bits, S entries so far (synchronises) */
int hm_symm_stream_counts(const void *d_work, const hm_symm_layout *L, uint64_t *n_cand,
                                     uint64_t *status, uint64_t *n_s, void *stream)
{ uint64_t h[SY_HDR_S+1];
  HM_CUDA(cudaMemcpyAsync(h,(const uint8_t *) d_work + L->off_header,sizeof(h),cudaMemcpyDeviceToHost,
                          (cudaStream_t) stream));
  HM_CUDA(cudaStreamSynchronize((cudaStream_t) stream));
  *n_cand = h[SY_HDR_CAND]; *status = h[SY_HDR_STATUS]; *n_s = h[SY_HDR_S];
  return HM_OK;
}

/* the candidate and S counts back to 0 once their entries have been copied out (status and Bloom filter stay) */
int hm_symm_stream_reset_lists(void *d_work, const hm_symm_layout *L, void *stream)
{ unsigned long long *h = (unsigned long long *) ((uint8_t *) d_work + L->off_header);
  HM_CUDA(cudaMemsetAsync(h+SY_HDR_CAND,0,sizeof(uint64_t),(cudaStream_t) stream));
  HM_CUDA(cudaMemsetAsync(h+SY_HDR_S,0,sizeof(uint64_t),(cudaStream_t) stream));
  return HM_OK;
}

/* pass 2 of the streamed scan: the exact check of a Bloom hit is a look-up in the sorted S list (several shards:
 * the S list of the key's owner, reached through the view's d_views)                                          */
int hm_symm_stream_resolve(const uint64_t *d_s_key, const uint64_t *d_s_lo, int64_t n_s,
                                      const void *d_s_bucket, int bits, int idx64, int kmer, int64_t range,
                                      void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                                      const hm_symm_shards *shards, const hm_stream_sview *d_views,
                                      unsigned long long *d_plot, void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || (kmer > 32) != (d_s_lo != NULL) || d_plot == NULL ||
      (shards != NULL && shards->n_seg > 1 && d_views == NULL))
    return hm_set_error(HM_EINVAL,"symm_stream_resolve: bad arguments");
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = stream_view(d_work,L,R,shards);
  W.sviews = d_views;
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { return launch_resolve<typename decltype(I)::IdxT,decltype(I)::KW,LK_SLIST>(d_s_key,d_s_lo,NULL,n_s,d_s_bucket,bits,
                                                                                kmer,W,d_plot,range,st); });
  if (l2_persist())
    bloom_window(st,NULL,0,0);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"resolve_kernel (streamed)");
  return HM_OK;
}

/* ------------------------------------------------------------------ routed pass 2 --------- */
/* One rank of a one-process-per-GPU job streams its own share (hm_scan.cu hm_rank_scan_*, DESIGN.md §4c): nobody
 * can read another rank's S list, so pass 2 goes in rounds over slices [c0, c1) of the rank's candidates.
 * resolve_kernel<..., LK_ROUTED> settles what the rank's own S list decides and parks the rest (route_push);
 * route_count / route_scatter group the queries by owner (a one-digit radix sort: not a hot path); the caller
 * sends the key words to their owners, route_answer_kernel answers the keys that arrive, the answers come back
 * in the order they were sent, and route_mark / route_settle count every parked candidate none of whose
 * queried keys was found.                                                                                     */
static SymmView route_view(void *d_work, const hm_symm_layout *L, const hm_stream_lists *R, const hm_symm_shards *sh,
                           const hm_route_bufs *B, int64_t c0, int64_t c1)
{ SymmView W = slice_view(stream_view(d_work,L,R,sh),c0,c1);    /* (the header counts all candidates: >= c1) */
  W.pend = B->pend; W.pend_key = B->pend_key; W.pend_lo = B->pend_lo;
  W.q_key = B->q_key; W.q_lo = B->q_lo; W.q_tag = B->q_tag;
  W.pend_cap = (unsigned long long) B->pend_cap; W.q_cap = (unsigned long long) B->q_cap;
  return W;
}

/* the arguments hm_symm_route_resolve and hm_symm_route_extract share: a slice the buffers can take */
static bool route_args_ok(int kmer, const uint64_t *d_s_lo, const hm_stream_lists *R, const hm_route_bufs *B,
                          int64_t c0, int64_t c1)
{ return kmer >= HM_SYMM_MIN_KMER && kmer <= HM_MAX_KMER && (kmer > 32) == (d_s_lo != NULL) && B != NULL &&
         c0 >= 0 && c1 >= c0 && c1 <= R->cand_cap && c1-c0 <= B->pend_cap && 2*(c1-c0) <= B->q_cap;
}

int hm_symm_route_resolve(const uint64_t *d_s_key, const uint64_t *d_s_lo, int64_t n_s,
                          const void *d_s_bucket, int bits, int idx64, int kmer, int64_t c0, int64_t c1,
                          void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                          const hm_symm_shards *shards, const hm_route_bufs *B, unsigned long long *d_plot, void *stream)
{ if (d_plot == NULL || !route_args_ok(kmer,d_s_lo,R,B,c0,c1))
    return hm_set_error(HM_EINVAL,"symm_route_resolve: bad arguments");
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = route_view(d_work,L,R,shards,B,c0,c1);
  HM_CUDA(cudaMemsetAsync(W.cand_n+SY_HDR_PEND,0,2*sizeof(uint64_t),st));   /* the round's pending and query counts */
  if (c1 == c0)
    return HM_OK;
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { return launch_resolve<typename decltype(I)::IdxT,decltype(I)::KW,LK_ROUTED>(d_s_key,d_s_lo,NULL,n_s,d_s_bucket,bits,
                                                                                 kmer,W,d_plot,8*(c1-c0),st); });
  if (l2_persist())
    bloom_window(st,NULL,0,0);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"resolve_kernel (routed)");
  return HM_OK;
}

__global__ void route_count_kernel(const uint64_t *__restrict__ tag, int64_t nq, unsigned long long *__restrict__ counts)
{ for (int64_t j = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; j < nq; j += (int64_t) gridDim.x*blockDim.x)
    atomicAdd(counts + (tag[j] >> 32),1ull);
}

template <int KW>
__global__ void route_scatter_kernel(const uint64_t *__restrict__ qk, const uint64_t *__restrict__ ql,
                                     const uint64_t *__restrict__ tag, int64_t nq, unsigned long long *__restrict__ cursor,
                                     uint64_t *__restrict__ send, uint32_t *__restrict__ send_slot)
{ for (int64_t j = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; j < nq; j += (int64_t) gridDim.x*blockDim.x)
    { const uint64_t t = tag[j];
      const unsigned long long at = atomicAdd(cursor + (t >> 32),1ull);
      send[KW*at] = qk[j];
      if (KW == 2) send[KW*at+1] = ql[j];
      send_slot[at] = (uint32_t) t;
    }
}

static int route_grid(int64_t n)
{ int64_t g = (n+255)/256;
  return (int) (g < 1 ? 1 : (g > 4096 ? 4096 : g));
}

/* the last round's queries grouped by owner into B->send (KW words each) and B->send_slot; counts[r] = queries
 * for rank r (r < world), *n_pend = parked candidates, *status = the header's status word (synchronises)     */
int hm_symm_route_group(int kmer, int world, void *d_work, const hm_symm_layout *L, const hm_route_bufs *B,
                        int64_t *counts, int64_t *n_sent, int64_t *n_pend, uint64_t *status, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  uint64_t h[SY_HDR_QUERY+1];
  HM_CUDA(cudaMemcpyAsync(h,(const uint8_t *) d_work + L->off_header,sizeof(h),cudaMemcpyDeviceToHost,st));
  HM_CUDA(cudaMemsetAsync(B->counts,0,2*HM_MAX_SHARDS*sizeof(unsigned long long),st));
  HM_CUDA(cudaStreamSynchronize(st));
  int64_t nq = (int64_t) h[SY_HDR_QUERY];
  *status = h[SY_HDR_STATUS];
  *n_pend = (int64_t) h[SY_HDR_PEND] < B->pend_cap ? (int64_t) h[SY_HDR_PEND] : B->pend_cap;
  if (nq > B->q_cap) nq = B->q_cap;                       /* (an overflow is in the status word) */
  *n_sent = nq;
  for (int r = 0; r < world; r++) counts[r] = 0;
  if (nq == 0)
    return HM_OK;
  route_count_kernel<<<route_grid(nq),256,0,st>>>(B->q_tag,nq,B->counts);
  unsigned long long c[HM_MAX_SHARDS], cur[HM_MAX_SHARDS], acc = 0;
  HM_CUDA(cudaMemcpyAsync(c,B->counts,sizeof(c),cudaMemcpyDeviceToHost,st));
  HM_CUDA(cudaStreamSynchronize(st));
  for (int r = 0; r < HM_MAX_SHARDS; r++)
    { cur[r] = acc; acc += c[r];
      if (r < world) counts[r] = (int64_t) c[r];
    }
  HM_CUDA(cudaMemcpyAsync(B->counts+HM_MAX_SHARDS,cur,sizeof(cur),cudaMemcpyHostToDevice,st));
  if (kmer > 32)
    route_scatter_kernel<2><<<route_grid(nq),256,0,st>>>(B->q_key,B->q_lo,B->q_tag,nq,B->counts+HM_MAX_SHARDS,B->send,B->send_slot);
  else
    route_scatter_kernel<1><<<route_grid(nq),256,0,st>>>(B->q_key,B->q_lo,B->q_tag,nq,B->counts+HM_MAX_SHARDS,B->send,B->send_slot);
  HM_CUDA(cudaGetLastError());
  HM_CUDA(cudaStreamSynchronize(st));
  return HM_OK;
}

/* one thread per key that arrived (KW words each): is it in this rank's S list?  One byte back per key */
template <typename IdxT, int KW>
__global__ void route_answer_kernel(const uint64_t *__restrict__ s_key, const uint64_t *__restrict__ s_lo,
                                    const IdxT *__restrict__ s_bucket, int bshift, const uint64_t *__restrict__ recv,
                                    int64_t n, uint8_t *__restrict__ ans)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    { const uint64_t q = recv[KW*i], ql = KW == 2 ? recv[KW*i+1] : 0;
      ans[i] = bucket_find<IdxT,KW>(s_key,s_lo,s_bucket,bshift,q,ql) >= 0 ? 1 : 0;
    }
}

int hm_symm_route_answer(const uint64_t *d_s_key, const uint64_t *d_s_lo, const void *d_s_bucket, int bits,
                         int idx64, int kmer, const uint64_t *d_recv, int64_t n, uint8_t *d_ans, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n > 0)
    { const int g = route_grid(n), sh = 64-bits;
      HM_CUDA(dispatch(kmer,idx64,[&](auto I)
        { typedef typename decltype(I)::IdxT IdxT;
          route_answer_kernel<IdxT,decltype(I)::KW><<<g,256,0,st>>>(d_s_key,d_s_lo,(const IdxT *) d_s_bucket,sh,d_recv,n,d_ans);
          return cudaGetLastError(); }));
    }
  HM_CUDA(cudaStreamSynchronize(st));
  return HM_OK;
}

#define ROUTE_FOUND (1ull << 63)                           /* a parked candidate's meta: some queried key is in S */

__global__ void route_mark_kernel(const uint8_t *__restrict__ ans, const uint32_t *__restrict__ send_slot, int64_t n,
                                  unsigned long long *__restrict__ pend)
{ for (int64_t j = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; j < n; j += (int64_t) gridDim.x*blockDim.x)
    if (ans[j])
      atomicOr(pend + send_slot[j],ROUTE_FOUND);
}

/* count_pair's weight rule, straight into the plot (few candidates) */
__global__ void route_settle_kernel(const uint64_t *__restrict__ pend, int64_t n, int kmer,
                                    unsigned long long *__restrict__ plot)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    { const uint64_t meta = pend[i];
      if (meta & ROUTE_FOUND)
        continue;
      const int cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff), p = (int) ((meta >> 32) & 0xff);
      const int s = cx+cy, m = cx < cy ? cx : cy;
      atomicAdd(plot + s*HM_PLOT_W + m,(unsigned long long) ((2*p == kmer-1) ? 1 : 2));
    }
}

/* d_ans: the answers to the round's n_sent queries, in the order they were sent (synchronises) */
int hm_symm_route_settle(int kmer, const hm_route_bufs *B, const uint8_t *d_ans, int64_t n_sent, int64_t n_pend,
                         unsigned long long *d_plot, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n_sent > 0)
    route_mark_kernel<<<route_grid(n_sent),256,0,st>>>(d_ans,B->send_slot,n_sent,(unsigned long long *) B->pend);
  if (n_pend > 0)
    route_settle_kernel<<<route_grid(n_pend),256,0,st>>>(B->pend,n_pend,kmer,d_plot);
  HM_CUDA(cudaGetLastError());
  HM_CUDA(cudaStreamSynchronize(st));
  return HM_OK;
}

/* ------------------------------------------------------------------ lists in host memory ---- */
/* The streamed scan whose candidate records and S list went to host memory in pass 1 (hm_scan.cu, DESIGN.md §4c,
 * *Lists in host memory*).  A round sweeps candidate slices with resolve_kernel<..., LK_PARK>: a Bloom miss is
 * counted at once, a hit parked with a query per key that hit (q_tag = pending slot).  The round's queries are
 * then sorted by key into B->send (KW words each) and B->send_slot, so that the queries falling in one S partition
 * are one contiguous range; route_answer_kernel answers each range against its uploaded partition, and
 * hm_symm_route_settle counts the parked candidates none of whose queries was found.                          */

/* one slice of n candidates (R's cand_key / cand_lo / cand_meta) swept into the round's pending list and queries;
 * reset: the slice opens a round (its pending and query counts start at 0)                                     */
int hm_symm_park_resolve(int kmer, int64_t n, int reset, void *d_work, const hm_symm_layout *L,
                         const hm_stream_lists *R, const hm_symm_shards *shards, const hm_route_bufs *B,
                         unsigned long long *d_plot, void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || d_plot == NULL || B == NULL || n < 0 || n > R->cand_cap ||
      (kmer > 32) != (R->cand_lo != NULL))
    return hm_set_error(HM_EINVAL,"symm_park_resolve: bad arguments");
  cudaStream_t st = (cudaStream_t) stream;
  hm_stream_lists S = *R;
  S.cand_cap = n;
  SymmView W = route_view(d_work,L,&S,shards,B,0,n);
  if (reset)
    HM_CUDA(cudaMemsetAsync(W.cand_n+SY_HDR_PEND,0,2*sizeof(uint64_t),st));
  HM_CUDA(cudaMemsetAsync(W.cand_n,0xff,sizeof(uint64_t),st));      /* the sweep reads min(header, cand_cap) = n */
  if (n == 0)
    return HM_OK;
  cudaError_t e = kmer > 32
    ? launch_resolve<uint32_t,2,LK_PARK>(NULL,NULL,NULL,0,NULL,2,kmer,W,d_plot,8*n,st)
    : launch_resolve<uint32_t,1,LK_PARK>(NULL,NULL,NULL,0,NULL,2,kmer,W,d_plot,8*n,st);
  if (l2_persist())
    bloom_window(st,NULL,0,0);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"resolve_kernel (parked)");
  return HM_OK;
}

/* the round's parked candidates and queries so far, and the status word (synchronises) */
int hm_symm_park_counts(const void *d_work, const hm_symm_layout *L, int64_t *n_pend, int64_t *n_q, uint64_t *status,
                        void *stream)
{ uint64_t h[SY_HDR_QUERY+1];
  HM_CUDA(cudaMemcpyAsync(h,(const uint8_t *) d_work + L->off_header,sizeof(h),cudaMemcpyDeviceToHost,
                          (cudaStream_t) stream));
  HM_CUDA(cudaStreamSynchronize((cudaStream_t) stream));
  *n_pend = (int64_t) h[SY_HDR_PEND]; *n_q = (int64_t) h[SY_HDR_QUERY]; *status = h[SY_HDR_STATUS];
  return HM_OK;
}

__global__ void park_iota_kernel(uint32_t *__restrict__ v, int64_t n)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    v[i] = (uint32_t) i;
}

__global__ void park_gather_kernel(const uint64_t *__restrict__ src, const uint32_t *__restrict__ perm, int64_t n,
                                   uint64_t *__restrict__ dst)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    dst[i] = src[perm[i]];
}

/* the queries in key order: KW words each into send, their pending slots into slot */
template <int KW>
__global__ void park_pack_kernel(const uint64_t *__restrict__ qk, const uint64_t *__restrict__ ql,
                                 const uint64_t *__restrict__ tag, const uint32_t *__restrict__ perm, int64_t n,
                                 uint64_t *__restrict__ send, uint32_t *__restrict__ slot)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    { const uint32_t j = perm[i];
      send[KW*i] = qk[j];
      if (KW == 2) send[KW*i+1] = ql[j];
      slot[i] = (uint32_t) tag[j];
    }
}

/* Sort the n_q queries of the round by key: a radix sort of key -> query index (k > 32: by the second word, then
 * stably by the first), the queries gathered in that order into B->send and their slots into one of perm_a /
 * perm_b, which B->send_slot is set to.  perm_a / perm_b: uint32[q_cap]; B->send holds 2 q_cap words at k > 32
 * (the second half is scratch there).  tmp: hm_sort_perm_bytes(q_cap) bytes.                                 */
int hm_symm_park_sort(int kmer, hm_route_bufs *B, int64_t n_q, uint32_t *perm_a, uint32_t *perm_b,
                      void *tmp, int64_t tmp_bytes, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n_q <= 0)
    return HM_OK;
  if (n_q > B->q_cap)
    return hm_set_error(HM_EINVAL,"symm_park_sort: %lld queries for %lld slots",(long long) n_q,(long long) B->q_cap);
  const int g = route_grid(n_q);
  int rc;
  park_iota_kernel<<<g,256,0,st>>>(perm_a,n_q);
  if (kmer <= 32)
    { if ((rc = hm_sort_perm(B->q_key,B->send,perm_a,perm_b,n_q,tmp,tmp_bytes,st)) != HM_OK) return rc;
      park_pack_kernel<1><<<g,256,0,st>>>(B->q_key,NULL,B->q_tag,perm_b,n_q,B->send,perm_a);
      B->send_slot = perm_a;
    }
  else
    { uint64_t *hi = B->send + B->q_cap;
      if ((rc = hm_sort_perm(B->q_lo,B->send,perm_a,perm_b,n_q,tmp,tmp_bytes,st)) != HM_OK) return rc;
      park_gather_kernel<<<g,256,0,st>>>(B->q_key,perm_b,n_q,hi);
      if ((rc = hm_sort_perm(hi,B->send,perm_b,perm_a,n_q,tmp,tmp_bytes,st)) != HM_OK) return rc;
      park_pack_kernel<2><<<g,256,0,st>>>(B->q_key,B->q_lo,B->q_tag,perm_a,n_q,B->send,perm_b);
      B->send_slot = perm_b;
    }
  HM_CUDA(cudaGetLastError());
  return HM_OK;
}

/* ------------------------------------------------------------------ parked routed rounds ---- */
/* One rank of a one-process-per-GPU job whose lists went to host memory (hm_scan.cu hm_rank_scan_*, DESIGN.md §4c,
 * *Lists in host memory*, *Ranks*).  A round sweeps one uploaded slice with resolve_kernel or extract_kernel
 * <..., LK_PARK>: every Bloom hit is parked, each hit key a query tagged owner << 32 | pending slot, the owner
 * possibly this rank; route_group sends them.  The owner sorts the keys it receives (hm_symm_recv_sort), answers
 * them against its S list a partition at a time (route_answer_kernel over each contiguous range) and puts the
 * answers back in receive order (hm_symm_recv_unsort), so that they return in the order they were sent.      */

/* the listing's sweep of one slice of n candidates: misses with a labelled pixel listed at once, hits parked with
 * their key words (a new round: the pending and query counts, and the record counter, start at 0)             */
int hm_symm_park_extract(int kmer, int64_t n, void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                         const hm_symm_shards *shards, const hm_route_bufs *B, const uint16_t *d_pixmap,
                         hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count, void *stream)
{ if (kmer < HM_SYMM_MIN_KMER || kmer > HM_MAX_KMER || B == NULL || n < 0 || n > R->cand_cap || d_pixmap == NULL ||
      d_count == NULL || d_out == NULL || cap < 2*n || (kmer > 32) != (R->cand_lo != NULL) || B->pend_key == NULL ||
      (kmer > 32 && B->pend_lo == NULL))
    return hm_set_error(HM_EINVAL,"symm_park_extract: bad arguments");
  cudaStream_t st = (cudaStream_t) stream;
  hm_stream_lists S = *R;
  S.cand_cap = n;
  SymmView W = route_view(d_work,L,&S,shards,B,0,n);
  HM_CUDA(cudaMemsetAsync(W.cand_n+SY_HDR_PEND,0,2*sizeof(uint64_t),st));
  HM_CUDA(cudaMemsetAsync(W.cand_n,0xff,sizeof(uint64_t),st));      /* the sweep reads min(header, cand_cap) = n */
  HM_CUDA(cudaMemsetAsync(d_count,0,sizeof(unsigned long long),st));
  if (n == 0)
    return HM_OK;
  cudaError_t e = kmer > 32
    ? launch_extract<uint32_t,2,LK_PARK>(NULL,NULL,NULL,0,NULL,2,kmer,W,d_pixmap,d_out,cap,d_count,st)
    : launch_extract<uint32_t,1,LK_PARK>(NULL,NULL,NULL,0,NULL,2,kmer,W,d_pixmap,d_out,cap,d_count,st);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"extract_kernel (parked)");
  return HM_OK;
}

/* word `w` of each received key (kw words apiece), in the order perm gives (NULL: as received) */
__global__ void recv_word_kernel(const uint64_t *__restrict__ recv, int kw, int w, const uint32_t *__restrict__ perm,
                                 int64_t n, uint64_t *__restrict__ dst)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    dst[i] = recv[(int64_t) kw*(perm != NULL ? (int64_t) perm[i] : i) + w];
}

/* the received keys in key order: both words of key perm[i] to sorted[2i], sorted[2i+1] */
__global__ void recv_pack_kernel(const uint64_t *__restrict__ recv, const uint32_t *__restrict__ perm, int64_t n,
                                 uint64_t *__restrict__ sorted)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    { const int64_t j = perm[i];
      sorted[2*i] = recv[2*j]; sorted[2*i+1] = recv[2*j+1];
    }
}

/* Sort the n keys received (KW words each, in recv) by key into sorted (KW words each; 2n words at k > 32, also the
 * scratch there): a radix sort of key -> receive index (k > 32: by the second word, then stably by the first).
 * *perm: perm_a or perm_b, whichever holds each sorted key's receive index.  perm_a / perm_b: uint32[n];
 * tmp: hm_sort_perm_bytes(n) bytes.                                                                         */
int hm_symm_recv_sort(int kmer, const uint64_t *recv, int64_t n, uint64_t *sorted, uint32_t *perm_a, uint32_t *perm_b,
                      void *tmp, int64_t tmp_bytes, uint32_t **perm, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  *perm = perm_a;
  if (n <= 0)
    return HM_OK;
  const int g = route_grid(n);
  int rc;
  park_iota_kernel<<<g,256,0,st>>>(perm_a,n);
  if (kmer <= 32)
    { if ((rc = hm_sort_perm(recv,sorted,perm_a,perm_b,n,tmp,tmp_bytes,st)) != HM_OK) return rc;
      *perm = perm_b;
    }
  else
    { uint64_t *a = sorted, *b = sorted + n;
      recv_word_kernel<<<g,256,0,st>>>(recv,2,1,NULL,n,a);
      if ((rc = hm_sort_perm(a,b,perm_a,perm_b,n,tmp,tmp_bytes,st)) != HM_OK) return rc;
      recv_word_kernel<<<g,256,0,st>>>(recv,2,0,perm_b,n,a);
      if ((rc = hm_sort_perm(a,b,perm_b,perm_a,n,tmp,tmp_bytes,st)) != HM_OK) return rc;
      recv_pack_kernel<<<g,256,0,st>>>(recv,perm_a,n,sorted);
      *perm = perm_a;
    }
  HM_CUDA(cudaGetLastError());
  return HM_OK;
}

__global__ void recv_unsort_kernel(const uint8_t *__restrict__ ans_sorted, const uint32_t *__restrict__ perm, int64_t n,
                                   uint8_t *__restrict__ ans)
{ for (int64_t i = (int64_t) blockIdx.x*blockDim.x + threadIdx.x; i < n; i += (int64_t) gridDim.x*blockDim.x)
    ans[perm[i]] = ans_sorted[i];
}

/* the answers to the sorted keys back in receive order: ans[perm[i]] = ans_sorted[i] (synchronises) */
int hm_symm_recv_unsort(const uint8_t *d_ans_sorted, const uint32_t *d_perm, int64_t n, uint8_t *d_ans, void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n > 0)
    recv_unsort_kernel<<<route_grid(n),256,0,st>>>(d_ans_sorted,d_perm,n,d_ans);
  HM_CUDA(cudaGetLastError());
  HM_CUDA(cudaStreamSynchronize(st));
  return HM_OK;
}

/* ------------------------------------------------------------------ routed pair listing ---- */
/* extract_kmer_pairs on one rank (hm_rank_scan_extract_*, DESIGN.md §4c): the rounds of routed pass 2, with
 * extract_kernel<..., LK_ROUTED> in place of resolve_kernel and route_list_kernel in place of route_settle_kernel.
 * A round's records (at most two per candidate of its slice) go to out through one counter, which counts every
 * record, also those beyond cap.                                                                          */
int hm_symm_route_extract(const uint64_t *d_s_key, const uint64_t *d_s_lo, int64_t n_s,
                          const void *d_s_bucket, int bits, int idx64, int kmer, int64_t c0, int64_t c1,
                          void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                          const hm_symm_shards *shards, const hm_route_bufs *B, const uint16_t *d_pixmap,
                          hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count, void *stream)
{ if (d_pixmap == NULL || d_count == NULL || d_out == NULL || !route_args_ok(kmer,d_s_lo,R,B,c0,c1) ||
      B->pend_key == NULL || (kmer > 32 && B->pend_lo == NULL) || cap < 2*(c1-c0))
    return hm_set_error(HM_EINVAL,"symm_route_extract: bad arguments");
  cudaStream_t st = (cudaStream_t) stream;
  SymmView W = route_view(d_work,L,R,shards,B,c0,c1);
  HM_CUDA(cudaMemsetAsync(W.cand_n+SY_HDR_PEND,0,2*sizeof(uint64_t),st));   /* the round's pending and query counts */
  HM_CUDA(cudaMemsetAsync(d_count,0,sizeof(unsigned long long),st));
  if (c1 == c0)
    return HM_OK;
  cudaError_t e = dispatch(kmer,idx64,[&](auto I)
    { return launch_extract<typename decltype(I)::IdxT,decltype(I)::KW,LK_ROUTED>(d_s_key,d_s_lo,NULL,n_s,d_s_bucket,bits,
                                                                                 kmer,W,d_pixmap,d_out,cap,d_count,st); });
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"extract_kernel (routed)");
  return HM_OK;
}

/* every parked candidate none of whose queried keys was found (no ROUTE_FOUND) is isolated: listed if its pixel
 * has a label.  list_pairs is warp-wide, so every lane of a warp stays in the loop (one atomic per warp).      */
template <int KW>
__global__ void route_list_kernel(const uint64_t *__restrict__ pend, const uint64_t *__restrict__ pkey,
                                  const uint64_t *__restrict__ plo, int64_t n, int kmer,
                                  const uint16_t *__restrict__ pixmap, hm_pair_rec *__restrict__ out,
                                  unsigned long long cap, unsigned long long *__restrict__ count)
{ const int      lane = threadIdx.x & 31;
  const unsigned lt   = (1u << lane) - 1;
  const int64_t  stride = (int64_t) gridDim.x*blockDim.x;
  for (int64_t w = (int64_t) blockIdx.x*blockDim.x + (threadIdx.x & ~31); w < n; w += stride)
    { const int64_t i = w + lane;
      uint64_t meta = 0, x = 0, xl = 0;
      unsigned lab = 0;
      if (i < n)
        { meta = pend[i];
          if (!(meta & ROUTE_FOUND))
            { const int cx = (int) (meta & 0xffff), cy = (int) ((meta >> 16) & 0xffff);
              x = pkey[i];
              if (KW == 2) xl = plo[i];
              lab = pixmap[(cx+cy)*HM_PLOT_W + (cx < cy ? cx : cy)];
            }
        }
      list_pairs<KW>(x,xl,meta,lab,kmer,out,cap,count,lane,lt);
    }
}

/* d_ans: the answers to the round's n_sent queries, in send order; lists the round's parked candidates that are
 * isolated after all into d_out (synchronises)                                                            */
int hm_symm_route_list(int kmer, const hm_route_bufs *B, const uint8_t *d_ans, int64_t n_sent, int64_t n_pend,
                       const uint16_t *d_pixmap, hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count,
                       void *stream)
{ cudaStream_t st = (cudaStream_t) stream;
  if (n_sent > 0)
    route_mark_kernel<<<route_grid(n_sent),256,0,st>>>(d_ans,B->send_slot,n_sent,(unsigned long long *) B->pend);
  if (n_pend > 0)
    { if (kmer > 32)
        route_list_kernel<2><<<route_grid(n_pend),256,0,st>>>(B->pend,B->pend_key,B->pend_lo,n_pend,kmer,d_pixmap,
                                                              d_out,(unsigned long long) cap,d_count);
      else
        route_list_kernel<1><<<route_grid(n_pend),256,0,st>>>(B->pend,B->pend_key,NULL,n_pend,kmer,d_pixmap,
                                                              d_out,(unsigned long long) cap,d_count);
    }
  HM_CUDA(cudaGetLastError());
  HM_CUDA(cudaStreamSynchronize(st));
  return HM_OK;
}

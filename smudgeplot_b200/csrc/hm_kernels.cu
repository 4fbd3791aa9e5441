/*******************************************************************************************
 * hm_kernels.cu -- CUDA kernels (sm_90a) + layer-A entry points of include/hetmers_b200.h.
 *
 * One-substitution neighbour search over a sorted, device-resident k-mer table.
 * Integer / memory-bound work: no tensor cores (see DESIGN.md §5 for the roofline).
 *
 * What replaces what (reference file:line under smudgeplot's src/lib):
 *   unpack_records_{tma_,}kernel  Next_Kmer_Entry + Current_Entry   libfastk.c:1159-1176,:1230-1269
 *   bucket_index_kernel     stub index + GoTo_Kmer_Entry       libfastk.c:1320-1409
 *   filter_build_kernel     (none: the merge's "no head has this suffix", PloidyPlot.c:618-643)
 *   pass1_filter_kernel     analysis_in_core_1 / _thread_1     PloidyPlot.c:454-568,:168-301
 *   pass2_plot_kernel       analysis_in_core_2 / _thread_2     PloidyPlot.c:570-700,:303-452
 *   pass2_extract_kernel    the same in extract_kmer_pairs      PloidyList.c:425-450,:680-705
 *   min_count_kernel        examine_table (trim half)          PloidyPlot.c:1171-1197
 *   find_keys_kernel        GoTo_Kmer_Entry exact-hit use      PloidyPlot.c:1213
 *******************************************************************************************/
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "hetmers_b200.h"
#include "hm_internal.h"
#include "hm_device.cuh"

/* ------------------------------------------------------------------ error plumbing ------ */

static thread_local char g_err[1024] = "";

extern "C" const char *hm_last_error(void) { return g_err; }
extern "C" int hm_abi_version(void) { return 1; }

extern "C" int hm_set_error(int code, const char *fmt, ...)
{ va_list ap;
  va_start(ap,fmt);
  vsnprintf(g_err,sizeof(g_err),fmt,ap);
  va_end(ap);
  return code;
}

int hm_cuda_fail(cudaError_t e, const char *what)
{ return hm_set_error(HM_ECUDA,"%s: %s",what,cudaGetErrorString(e)); }

extern "C" int hm_device_count(void)
{ int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess)
    { cudaGetLastError(); return 0; }
  return n;
}

extern "C" int hm_device_info(int dev, char *name, int name_len, int *sm_count, int64_t *total_mem)
{ cudaDeviceProp p;
  cudaError_t e = cudaGetDeviceProperties(&p,dev);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"cudaGetDeviceProperties");
  if (name != NULL && name_len > 0)
    { strncpy(name,p.name,name_len-1); name[name_len-1] = 0; }
  if (sm_count != NULL) *sm_count = p.multiProcessorCount;
  if (total_mem != NULL) *total_mem = (int64_t) p.totalGlobalMem;
  return HM_OK;
}

extern "C" int hm_pick_bucket_bits(int64_t n)
{ int lg = 0;
  while (lg < 62 && ((int64_t) 1 << (lg+1)) <= n)
    lg += 1;                                  /* floor(log2 n) */
  int bits = lg-1;                            /* ~2-4 entries per bucket */
  if (bits > 30) bits = 30;
  if (bits < 2)  bits = 2;
  return bits;
}

/* ------------------------------------------------------------------ device helpers ------ */

/* Filter words are streamed (each probed column walks the bitmap once, no reuse), everything else
 * pass 1 touches (keys, bucket offsets, counts) is re-read by neighbouring probes: ask L2 to drop
 * the former first.  P1_FILTER_LD=0 plain __ldg, 1 L2::evict_first, 2 + L1::no_allocate.        */
#ifndef P1_FILTER_LD
#define P1_FILTER_LD 0
#endif
__device__ __forceinline__ uint64_t make_evict_first_policy(void)
{ uint64_t pol = 0;
#if P1_FILTER_LD >= 1
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol));
#endif
  return pol;
}

__device__ __forceinline__ uint32_t ld_filter(const uint32_t *p, uint64_t pol)
{
#if P1_FILTER_LD == 1
  uint32_t v;
  asm volatile("ld.global.nc.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
#elif P1_FILTER_LD == 2
  uint32_t v;
  asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.u32 %0, [%1], %2;" : "=r"(v) : "l"(p), "l"(pol));
  return v;
#else
  (void) pol;
  return __ldg(p);
#endif
}

/* ------------------------------------------------------------------------- unpack ------- */

__device__ __forceinline__ int upper_bound_index(const int64_t *__restrict__ index,
                                                 int l, int r, int64_t o)
{ /* first b in [l,r] with index[b] > o  (r is a valid answer bound) */
  while (l < r)
    { int m = (l+r)>>1;
      if (__ldg(index+m) > o) r = m; else l = m+1;
    }
  return l;
}

__global__ void __launch_bounds__(256)
unpack_records_kernel(const uint8_t *__restrict__ rec, int64_t n, int64_t first,
                      const int64_t *__restrict__ index, int ixlen, int ibyte, int hbyte,
                      uint64_t *__restrict__ keys, uint64_t *__restrict__ keys_lo,
                      uint16_t *__restrict__ cnt)
{ __shared__ int s_blo, s_bhi;
  int64_t t0 = (int64_t) blockIdx.x * blockDim.x;
  if (threadIdx.x == 0)
    { int64_t o0 = first+t0;
      int64_t o1 = first + (t0+blockDim.x < n ? t0+blockDim.x : n) - 1;
      s_blo = upper_bound_index(index,0,ixlen-1,o0);
      s_bhi = upper_bound_index(index,s_blo,ixlen-1,o1);
    }
  __syncthreads();
  int64_t i = t0+threadIdx.x;
  if (i >= n)
    return;
  int pbyte = hbyte+2;
  uint64_t b = (uint64_t) upper_bound_index(index,s_blo,s_bhi,first+i);
  const uint8_t *r = rec + i*pbyte;
  uint64_t key = b << (64-8*ibyte), klo = 0;
  for (int j = 0; j < hbyte; j++)                     /* suffix byte j is key byte ibyte+j */
    { int pos = ibyte+j;
      if (pos < 8) key |= (uint64_t) r[j] << (56-8*pos);
      else         klo |= (uint64_t) r[j] << (56-8*(pos-8));
    }
  keys[i] = key;
  if (keys_lo != NULL)
    keys_lo[i] = klo;
  cnt[i]  = (uint16_t) (r[hbyte] | (r[hbyte+1]<<8));
}

/* ---- TMA-staged variant ---------------------------------------------------------------
 * FastK records are 5..9 bytes at an odd stride, so a thread-per-record global read is a string
 * of byte loads.  Here one elected thread asks the TMA engine for the CTA's whole tile of
 * UNP_TILE records (cp.async.bulk global -> shared, completion on an mbarrier; SASS: UBLKCP),
 * the CTA narrows the stub-index range while the bytes are in flight, and the unaligned record
 * fields are then picked out of shared memory; keys/counts leave as coalesced 8- / 2-byte stores.
 * Needs a 16-byte aligned source (tile size UNP_TILE*pbyte is a multiple of 16 by construction). */
#define UNP_TILE 1024

/* upper_bound_index by a whole warp: 32 probes per round instead of one (the stub index has 2^24 entries:
 * 5 dependent rounds instead of 24; one thread bisecting twice per tile was what bounded the kernel) */
__device__ __forceinline__ int warp_upper_bound_index(const int64_t *__restrict__ index, int l, int r, int64_t o)
{ const int lane = threadIdx.x & 31;
  while (r-l >= 32)
    { const int      width = (r-l) >> 5;
      const int      p   = l + (lane+1)*width - 1;                         /* < r */
      const unsigned gt  = __ballot_sync(0xffffffffu,__ldg(index+p) > o);
      if (gt == 0)
        l += 32*width;
      else
        { const int f = __ffs((int) gt)-1;
          r = l + (f+1)*width - 1;
          l = l + f*width;
        }
    }
  const int      p  = l+lane;
  const unsigned gt = __ballot_sync(0xffffffffu,p <= r && __ldg(index + (p <= r ? p : r)) > o);
  return gt != 0 ? l + __ffs((int) gt)-1 : r;
}

#define UNP_MAXSPAN 16384          /* stub-index buckets a tile may span before records bisect on their own */

/* The prefix of a record is the stub-index bucket its ordinal falls into.  Records and buckets are both in
 * order, so a tile resolves its prefixes together: every NON-EMPTY bucket that starts inside the tile marks
 * its first record (the tile spans ~90 buckets at 2e8 k-mers: one coalesced pass over that slice of the
 * index), and a max-scan over the 1024 marks hands every record the last bucket that started at or before
 * it.  (One global-memory bisection per record would cost ~7 dependent loads each.)                        */
__global__ void __launch_bounds__(256)
unpack_records_tma_kernel(const uint8_t *__restrict__ rec, int64_t first,
                          const int64_t *__restrict__ index, int ixlen, int ibyte, int hbyte,
                          uint64_t *__restrict__ keys, uint64_t *__restrict__ keys_lo,
                          uint16_t *__restrict__ cnt)
{ extern __shared__ __align__(128) uint8_t s_rec[];
  __shared__ __align__(8) uint64_t s_bar;
  __shared__ int s_blo, s_bhi;
  __shared__ int s_mark[UNP_TILE];
  __shared__ int s_wmax[8];
  const int      pbyte = hbyte+2;
  const unsigned bytes = (unsigned) (UNP_TILE*pbyte);
  const int64_t  t0    = (int64_t) blockIdx.x * UNP_TILE;
  const int64_t  base  = first+t0;                       /* table ordinal of the tile's first record */

  if (threadIdx.x == 0)
    { mbar_init(&s_bar,1);
      fence_proxy_async_smem();
    }
  for (int r = threadIdx.x; r < UNP_TILE; r += 256)
    s_mark[r] = 0;
  __syncthreads();
  if (threadIdx.x == 0)
    { mbar_arrive_expect_tx(&s_bar,bytes);
      bulk_copy_g2s(s_rec,rec + t0*pbyte,bytes,&s_bar);
    }
  if (threadIdx.x < 32)                                                 /* overlaps the copy */
    { const int lo_b = warp_upper_bound_index(index,0,ixlen-1,base);
      const int hi_b = warp_upper_bound_index(index,lo_b,ixlen-1,base+UNP_TILE-1);
      if (threadIdx.x == 0) { s_blo = lo_b; s_bhi = hi_b; }
    }
  __syncthreads();
  const int  blo = s_blo, bhi = s_bhi;
  const bool together = (bhi-blo <= UNP_MAXSPAN);        /* CTA-uniform */
  int pre[UNP_TILE/256];
  if (together)
    { /* bucket b covers ordinals [index[b-1], index[b]); blo holds the tile's first record */
      for (int b = blo+1+threadIdx.x; b <= bhi; b += 256)
        { const int64_t s0 = __ldg(index+b-1), s1 = __ldg(index+b);
          if (s1 > s0)                                   /* non-empty: starts inside the tile (blo < b <= bhi) */
            s_mark[(int) (s0-base)] = b;
        }
      __syncthreads();
      /* inclusive max-scan of the marks: 4 consecutive records per thread, then warps, then the CTA */
      const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
      int m = blo;
#pragma unroll
      for (int k = 0; k < UNP_TILE/256; k++)
        { const int v = s_mark[threadIdx.x*(UNP_TILE/256)+k];
          if (v > m) m = v;
          pre[k] = m;
        }
      int run = m;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1)
        { const int v = __shfl_up_sync(0xffffffffu,run,o);
          if (lane >= o && v > run) run = v;
        }
      if (lane == 31) s_wmax[warp] = run;
      __syncthreads();
      int before = blo;                                   /* max of everything in earlier threads */
      for (int w = 0; w < warp; w++)
        if (s_wmax[w] > before) before = s_wmax[w];
      const int prev = __shfl_up_sync(0xffffffffu,run,1);
      if (lane > 0 && prev > before) before = prev;
      __syncthreads();                                     /* everybody has read the marks: reuse them for the result */
#pragma unroll
      for (int k = 0; k < UNP_TILE/256; k++)
        s_mark[threadIdx.x*(UNP_TILE/256)+k] = before > pre[k] ? before : pre[k];
      __syncthreads();
    }
  mbar_wait(&s_bar,0);

#pragma unroll
  for (int k = 0; k < UNP_TILE/256; k++)
    { const int      r = threadIdx.x + 256*k;              /* consecutive lanes, consecutive records: coalesced stores */
      const int64_t  i = t0+r;
      const uint8_t *q = s_rec + r*pbyte;
      uint64_t b = together ? (uint64_t) s_mark[r] : (uint64_t) upper_bound_index(index,blo,bhi,first+i);
      uint64_t key = b << (64-8*ibyte), klo = 0;
      for (int j = 0; j < hbyte; j++)
        { int pos = ibyte+j;
          if (pos < 8) key |= (uint64_t) q[j] << (56-8*pos);
          else         klo |= (uint64_t) q[j] << (56-8*(pos-8));
        }
      keys[i] = key;
      if (keys_lo != NULL)
        keys_lo[i] = klo;
      cnt[i]  = (uint16_t) (q[hbyte] | (q[hbyte+1]<<8));
    }
}

extern "C" int hm_k_unpack_records(const uint8_t *d_rec, int64_t n, int64_t first,
                                   const int64_t *d_stub_index, int ibyte, int kmer,
                                   uint64_t *d_keys, uint64_t *d_keys_lo, uint16_t *d_cnt, void *stream)
{ if (kmer < 1 || kmer > HM_MAX_KMER)
    return hm_set_error(HM_EUNSUPPORTED,"k-mer length %d not supported (1..%d)",kmer,HM_MAX_KMER);
  int kbyte = (kmer+3)>>2;
  if (ibyte < 1 || ibyte > 3 || ibyte > kbyte)
    return hm_set_error(HM_EFORMAT,"prefix bytes ibyte=%d invalid for k=%d",ibyte,kmer);
  if ((kmer > 32) != (d_keys_lo != NULL))
    return hm_set_error(HM_EINVAL,"unpack: second key word array %s for k=%d",
                        d_keys_lo ? "given" : "missing",kmer);
  if (n <= 0)
    return HM_OK;
  int     hbyte = kbyte-ibyte, pbyte = hbyte+2;
  int64_t done  = 0;
  if ((((uintptr_t) d_rec) & 15) == 0 && n >= UNP_TILE)         /* full tiles through the TMA path */
    { int64_t ntiles = n/UNP_TILE;
      unpack_records_tma_kernel<<<(unsigned) ntiles,256,(size_t) UNP_TILE*pbyte,(cudaStream_t) stream>>>
          (d_rec,first,d_stub_index,1<<(8*ibyte),ibyte,hbyte,d_keys,d_keys_lo,d_cnt);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess)
        return hm_cuda_fail(e,"unpack_records_tma_kernel");
      done = ntiles*UNP_TILE;
    }
  if (done < n)                                                   /* tail / unaligned source */
    { int64_t m = n-done;
      int64_t nblk = (m+255)/256;
      unpack_records_kernel<<<(unsigned) nblk,256,0,(cudaStream_t) stream>>>
          (d_rec + done*pbyte,m,first+done,d_stub_index,1<<(8*ibyte),ibyte,hbyte,d_keys+done,
           d_keys_lo ? d_keys_lo+done : NULL,d_cnt+done);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess)
        return hm_cuda_fail(e,"unpack_records_kernel");
    }
  return HM_OK;
}

/* ------------------------------------------------------------------- bucket index ------- */

/* bucket[b] = first i with (keys[i] >> bshift) >= b, for b in [0, 2^bits]; thread i fills the
 * (normally 0 or 1) buckets that start at entry i.                                           */
template <typename IdxT>
__global__ void __launch_bounds__(256)
bucket_index_kernel(const uint64_t *__restrict__ keys, int64_t n, int bshift, int64_t nbuckets,
                    IdxT *__restrict__ bucket, int64_t i0, int64_t i1)
{ int64_t i = i0 + (int64_t) blockIdx.x * blockDim.x + threadIdx.x;     /* entries [i0,i1]; i == n is the end mark */
  if (i > i1 || i > n)
    return;
  int64_t cur  = (i < n) ? (int64_t) (keys[i] >> bshift) : nbuckets;
  int64_t prev = (i > 0) ? (int64_t) (keys[i-1] >> bshift) : -1;
  for (int64_t b = prev+1; b <= cur; b++)
    bucket[b] = (IdxT) i;
}

/* entries [i0,i1) of a table whose entries [0,i1) are in place (+ the end mark when i1 == n): lets
 * the loader index every chunk right behind its unpack instead of in a pass of its own         */
int hm_build_bucket_index_range(const uint64_t *d_keys, int64_t n, int bits, void *d_bucket,
                                int idx64, int64_t i0, int64_t i1, void *stream)
{ if (bits < 1 || bits > 30)
    return hm_set_error(HM_EINVAL,"bucket bits %d out of range 1..30",bits);
  if (!idx64 && n >= 0xFFFFFFFFll)
    return hm_set_error(HM_EINVAL,"32-bit offsets need n < 2^32-1");
  int64_t last = (i1 >= n) ? n : i1-1;
  if (last < i0)
    return HM_OK;
  int64_t nblk = (last-i0+1+255)/256;
  if (idx64)
    bucket_index_kernel<uint64_t><<<(unsigned) nblk,256,0,(cudaStream_t) stream>>>
        (d_keys,n,64-bits,(int64_t) 1<<bits,(uint64_t *) d_bucket,i0,last);
  else
    bucket_index_kernel<uint32_t><<<(unsigned) nblk,256,0,(cudaStream_t) stream>>>
        (d_keys,n,64-bits,(int64_t) 1<<bits,(uint32_t *) d_bucket,i0,last);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"bucket_index_kernel");
  return HM_OK;
}

extern "C" int hm_k_build_bucket_index(const uint64_t *d_keys, int64_t n, int bits,
                                       void *d_bucket, int idx64, void *stream)
{ return hm_build_bucket_index_range(d_keys,n,bits,d_bucket,idx64,0,n,stream); }

/* ------------------------------------------------------------------ prefix filter ------- */

/* Presence bitmap over the first F bits of every key: bit f set iff some table entry starts
 * with f.  64..128 bits per entry (DESIGN.md §4): a probe for a k-mer that is NOT in
 * the table -- 99 % of all probes -- is answered by one 4-byte load that neighbouring lanes
 * share, instead of a bucket lookup + bisection.                                              */
__global__ void __launch_bounds__(256)
filter_build_kernel(const uint64_t *__restrict__ keys, int64_t i0, int64_t n, int fshift,
                    uint32_t *__restrict__ filter)
{ int64_t i = i0 + (int64_t) blockIdx.x * blockDim.x + threadIdx.x;     /* entries [i0,n) */
  if (i >= n)
    return;
  uint64_t pf = keys[i] >> fshift;
  /* sorted keys: equal prefixes are adjacent, so only the first of a run needs to set the bit */
  if (i > 0 && (keys[i-1] >> fshift) == pf)
    return;
  atomicOr(filter + (pf>>5), 1u << (pf & 31));
}

int hm_build_filter_range(const uint64_t *d_keys, int filter_bits, uint32_t *d_filter,
                          int64_t i0, int64_t i1, void *stream);

extern "C" int hm_pick_filter_bits(int64_t n)
{ /* 23..45 filter bits per entry: fewer let more candidates survive to the bucket look-up, more cost
   * filter traffic (= #probed (position, base) pairs x filter size: every probe column streams the
   * whole bitmap once).  Pass 1 at 2e8 entries on one H100 SXM (400 W): 2^33 bits (43 per entry)
   * 14.6 ms, 2^34 17.4 ms, 2^35 26.3 ms                                                          */
  int lg = 0;                                  /* round(log2 n) */
  while (lg < 62 && ((int64_t) 1 << (lg+1)) <= n)
    lg += 1;
  if (lg < 61 && (double) n > 1.41421356 * (double) ((int64_t) 1 << lg))
    lg += 1;
  int fb = lg+5;
  if (fb < HM_FILTER_MIN_BITS) fb = HM_FILTER_MIN_BITS;
  if (fb > HM_FILTER_MAX_BITS) fb = HM_FILTER_MAX_BITS;
  return fb;
}

extern "C" int64_t hm_filter_words(int filter_bits)
{ return ((int64_t) 1 << filter_bits) >> 5; }

extern "C" int hm_k_build_filter(const uint64_t *d_keys, int64_t n, int filter_bits,
                                 uint32_t *d_filter, void *stream)
{ if (filter_bits < HM_FILTER_MIN_BITS || filter_bits > HM_FILTER_MAX_BITS)
    return hm_set_error(HM_EINVAL,"filter bits %d out of range %d..%d",filter_bits,
                        HM_FILTER_MIN_BITS,HM_FILTER_MAX_BITS);
  HM_CUDA(cudaMemsetAsync(d_filter,0,sizeof(uint32_t)*(size_t) hm_filter_words(filter_bits),
                          (cudaStream_t) stream));
  return hm_build_filter_range(d_keys,filter_bits,d_filter,0,n,stream);
}

/* set the bits of entries [i0,i1) (entries [0,i1) in place, filter zeroed by the caller) */
int hm_build_filter_range(const uint64_t *d_keys, int filter_bits, uint32_t *d_filter,
                          int64_t i0, int64_t i1, void *stream)
{ if (i1 <= i0)
    return HM_OK;
  int64_t nblk = (i1-i0+255)/256;
  filter_build_kernel<<<(unsigned) nblk,256,0,(cudaStream_t) stream>>>(d_keys,i0,i1,64-filter_bits,d_filter);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"filter_build_kernel");
  return HM_OK;
}

/* -------------------------------------------------------------------------- pass 1 ------ */

#ifndef P1_WARPS
#define P1_WARPS   8            /* warps per CTA                                     */
#endif
#ifndef P1_GRID_PER_SM
#define P1_GRID_PER_SM 1024      /* CTAs launched per SM, started in table order, each striding over a few
                                  * groups of 8 chunks.  Few persistent CTAs drift apart and lose the L2
                                  * reuse of filter sectors between neighbours: pass 1 at 2e8 entries on
                                  * one H100 SXM (400 W) 25.9 ms at 32/SM, 21.4 at 256/SM, 17.4 at 1024/SM */
#endif
#ifndef P1_MINBLOCKS
#define P1_MINBLOCKS 6          /* resident CTAs per SM the register budget must allow (40 regs, no spills) */
#endif
#define P1_QCAP    64           /* per-warp candidate queue: < 32 left + <= 32 pushed */
#define P1_RUNCAP  12           /* forward scan bound for the high positions          */

/* Where the incidence bytes live.  One GPU / dense mode: everything in `self`.  Sharded mode
 * (DESIGN.md §6): every GPU has a full-length array but only the slice of the entries it OWNS is
 * meaningful; bytes of foreign entries are reached through the owner's array, mapped here over
 * NVLink (peer access in one process, CUDA IPC between processes).  Pass 1's increments to a
 * foreign partner are remote atomics, pass 2's look-ups of a foreign partner are remote loads:
 * the exchange step is fused into the two kernels, no collective moves the array.             */
struct DegView
  { uint32_t *self;
    int64_t   lo, hi;                          /* entries owned by this GPU                      */
    int       n;                               /* shards (0 = everything is local)               */
    int64_t   off[HM_MAX_SHARDS+1];
    uint32_t *peer[HM_MAX_SHARDS];
    uint32_t *defer_cnt;                       /* pass 2: per-CTA counts of deferred foreign look-ups */
    void     *defer_ent;                       /*         their (entry, partner) index pairs          */
    int64_t   defer_cap;                       /*         entries per CTA (0 = look up inline)        */
  };

static DegView make_deg_view(uint8_t *d_deg, int64_t lo, int64_t hi, const hm_shards *sh)
{ DegView v;
  memset(&v,0,sizeof(v));
  v.self = (uint32_t *) d_deg;
  if (sh == NULL || sh->n_shards <= 1)
    { v.lo = INT64_MIN; v.hi = INT64_MAX; v.n = 0; }
  else
    { v.lo = lo; v.hi = hi; v.n = sh->n_shards;
      for (int r = 0; r <= sh->n_shards; r++) v.off[r] = sh->off[r];
      for (int r = 0; r < sh->n_shards; r++)  v.peer[r] = (uint32_t *) sh->deg[r];
    }
  return v;
}

#define P2_DEFER_HEADER 4096                   /* bytes reserved for the per-CTA counters */

__device__ __forceinline__ uint32_t *deg_words(const DegView &v, int64_t j)
{ if (j >= v.lo && j < v.hi)
    return v.self;
  int r = 0;
  while (r+1 < v.n && j >= v.off[r+1])
    r += 1;
  return v.peer[r];
}

/* book one qualifying pair (oi < j): both incidence bytes, and the upper partner of oi.  The bytes are
 * packed four to a word and added to with word-wide atomics: no carry into the neighbouring byte as long
 * as a degree stays below 256, i.e. 3k < 256 (the reference's uint8 Pair wraps instead, PloidyPlot.c:163) */
static_assert(3*HM_MAX_KMER < 256,"byte-packed incidence counters would carry into their neighbours");
template <typename IdxT>
__device__ __forceinline__ void book_pair(const uint16_t *__restrict__ cnt, int64_t oi, int64_t j,
                                          int64_t lo, const DegView &dv, IdxT *__restrict__ up)
{ if ((int) __ldg(cnt+oi) + (int) __ldg(cnt+j) <= HM_SMAX)         /* PloidyPlot.c:259 */
    { atomicAdd(dv.self + (oi>>2), 1u << (8*(oi&3)));
      atomicAdd(deg_words(dv,j) + (j>>2), 1u << (8*(j&3)));
      up[oi-lo] = (IdxT) j;
    }
}

/* A warp owns 32 consecutive table entries at a time (lane = entry).  For entry x only
 * neighbours y > x are sought (the lower member books the pair), and a neighbour differing at
 * base p shares x's first p bases with x AND with every entry between them, so p is bounded by
 * lcp(x, successor(x)).
 *
 *   low positions  p < PH = ceil(F/2): y's F-bit prefix is tested against the presence filter -- one
 *        predicated 4-byte load per (p, alt), fully unrolled, no divergence; survivors are only
 *        remembered as bits of a per-lane mask.
 *   high positions p >= PH: y shares x's filter prefix, so it sits in the short run of entries
 *        that follow x with the same PH-base prefix: scan that run and test x^z for a
 *        single-base difference (long runs fall back to per-position candidates).
 *   survivors are expanded into a per-warp shared-memory queue and resolved 32 at a time by a
 *        bucket lookup + bisection with every lane busy (the expensive, divergent part of the
 *        search runs at full SIMT efficiency and only for ~1 candidate per entry).            */
template <typename IdxT, int F, int KW>
__global__ void __launch_bounds__(P1_WARPS*32,P1_MINBLOCKS)
pass1_filter_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                    const uint16_t *__restrict__ cnt,
                    int64_t n, const IdxT *__restrict__ bucket, int bshift,
                    const uint32_t *__restrict__ filter, int kmer,
                    int64_t lo, int64_t hi, const DegView dv, IdxT *__restrict__ up)
{ __shared__ uint64_t s_qy[P1_WARPS][P1_QCAP];
  __shared__ uint64_t s_ql[KW == 2 ? P1_WARPS : 1][KW == 2 ? P1_QCAP : 1];
  __shared__ IdxT     s_qi[P1_WARPS][P1_QCAP];

  constexpr int PH  = (F+1)/2;                              /* positions with a bit in the prefix */
  constexpr int NA  = PH < 9 ? PH : 9;
  constexpr int SFT = F > 32 ? F-32 : 0;                    /* filter bits taken from the low word */
  constexpr int MW  = KW == 2 ? 3 : 1;                      /* words of the long-run fallback mask */
  const unsigned FULL = 0xffffffffu;
  const int      lane = threadIdx.x & 31;
  const int      warp = threadIdx.x >> 5;
  const unsigned lt   = (1u << lane) - 1;
  uint64_t *qy = s_qy[warp];
  uint64_t *ql = s_ql[KW == 2 ? warp : 0];
  IdxT     *qi = s_qi[warp];
  int       qn = 0;                                      /* warp-uniform queue fill */
  const uint64_t pol = make_evict_first_policy();

  const int64_t nchunks = (hi-lo+31) >> 5;
  for (int64_t c = (int64_t) blockIdx.x * P1_WARPS + warp; c < nchunks;
       c += (int64_t) gridDim.x * P1_WARPS)
    { const int64_t i = lo + (c<<5) + lane;
      const bool    valid = (i < hi);
      uint64_t x = 0, nxt = 0, xw = 0, nxtw = 0;         /* xw / nxtw: second key word (KW == 2) */
      int      pmax = -1;
      if (valid)
        { x = keys[i];
          if (KW == 2) xw = keys_lo[i];
          if (i+1 < n)
            { nxt = keys[i+1];
              if (KW == 2) nxtw = keys_lo[i+1];
              if (KW == 1 || x != nxt)
                pmax = __clzll((long long) (x ^ nxt)) >> 1;
              else
                pmax = 32 + (__clzll((long long) (xw ^ nxtw)) >> 1);
              if (pmax > kmer-1) pmax = kmer-1;
            }
        }
      /* ---- low positions: filter probes, branch-free ----
       * candidate = x with base p replaced by c in {1,2,3}; it is wanted iff it is > x (c above
       * the current base).  Survivor bits are shifted into two 32-bit masks in probe order:
       * ma holds positions [0,NA), mb positions [NA,PH).                                       */
      const uint32_t xh = (uint32_t) (x >> 32), xl = (uint32_t) x;
      uint32_t ma = 0, mb = 0;
      /* the filter bit is  w >> (pf & 31)  with pf = the candidate's F-bit prefix.  Replacing base p
       * leaves the low five prefix bits alone unless p is one of the last ~3 covered positions, so
       * the shift that brings the bit to the TOP of the word (31 - (pf & 31)) is computed once per
       * entry; a funnel shift then appends that top bit to the survivor mask in one instruction.  */
      constexpr int LOWBITS = F <= 32 ? 37-F : 5-SFT;       /* bits of yh below the word index */
      const uint32_t pf_own = F <= 32 ? (xh >> (32-F)) : ((xh << SFT) | (xl >> (32-SFT)));
      const uint32_t sl_own = 31 - (pf_own & 31);
#pragma unroll
      for (int p = 0; p < PH; p++)
        { const bool pa = (p <= pmax);
#pragma unroll
          for (int c = 1; c <= 3; c++)
            { bool     act;
              uint32_t widx, sl;
              if (p < 16)                                    /* base p lives in the high half */
                { const int      s  = 30-2*p;
                  const uint32_t yh = (xh & ~(3u << s)) | ((uint32_t) c << s);
                  act  = pa && (yh > xh);
                  widx = yh >> LOWBITS;
                  if (s >= LOWBITS)                          /* low prefix bits untouched */
                    sl = sl_own;
                  else if (F <= 32)
                    sl = 31 - ((yh >> (32-F)) & 31);
                  else
                    sl = 31 - (((yh << SFT) | (xl >> (32-SFT))) & 31);
                }
              else                                           /* F > 32: base p in the low half */
                { const int      s  = 62-2*p;
                  const uint32_t yl = (xl & ~(3u << s)) | ((uint32_t) c << s);
                  act  = pa && (yl > xl);
                  widx = xh >> (5-SFT);
                  sl   = 31 - (((xh << SFT) | (yl >> (32-SFT))) & 31);
                }
              uint32_t w = 0;
              if (act)
                w = ld_filter(filter + widx,pol);
              const uint32_t top = w << sl;                  /* the filter bit, at bit 31 */
              if (p < NA) ma = __funnelshift_l(top,ma,1);    /* (ma << 1) | bit */
              else        mb = __funnelshift_l(top,mb,1);
            }
        }

      /* ---- high positions: the run of entries sharing x's PH-base prefix ---- */
      uint64_t mhi[MW];
#pragma unroll
      for (int w = 0; w < MW; w++)
        mhi[w] = 0;
      if (pmax >= PH)
        { bool longrun = (i+P1_RUNCAP < n) &&
                         (((x ^ __ldg(keys+i+P1_RUNCAP)) >> (64-2*PH)) == 0);
          if (longrun)
            { for (int p = PH; p <= pmax; p++)
                { int b = (int) (((p < 32 ? x : xw) >> (62-2*(p&31))) & 3);
                  for (int cc = b+1; cc <= 3; cc++)
                    { int t = 3*(p-PH)+cc-1;
#pragma unroll
                      for (int w = 0; w < MW; w++)
                        if ((t>>6) == w)
                          mhi[w] |= (uint64_t) 1 << (t&63);
                    }
                }
            }
          else
            { int64_t  j = i+1;
              uint64_t z = nxt, zw = nxtw;
              while (true)
                { uint64_t dd = x ^ z;
                  if ((dd >> (64-2*PH)) != 0)
                    break;
                  uint64_t t = (dd | (dd>>1)) & 0x5555555555555555ull;
                  bool one = ((t & (t-1)) == 0);           /* at most one base of word 0 differs */
                  if (KW == 2)
                    { uint64_t dw = xw ^ zw;
                      uint64_t u  = (dw | (dw>>1)) & 0x5555555555555555ull;
                      one = one && ((u & (u-1)) == 0) && ((t == 0) != (u == 0));
                    }
                  if (one)                                  /* exactly one base differs */
                    book_pair<IdxT>(cnt,i,j,lo,dv,up);
                  j += 1;
                  if (j >= n)
                    break;
                  z = __ldg(keys+j);
                  if (KW == 2) zw = __ldg(keys_lo+j);
                }
            }
        }

      /* ---- expand survivors into the warp queue; resolve 32 at a time ---- */
      while (true)
        { uint64_t anyhi = mhi[0];
#pragma unroll
          for (int w = 1; w < MW; w++)
            anyhi |= mhi[w];
          const bool has = ((ma | mb) != 0) || (anyhi != 0);
          if (!__any_sync(FULL,has))
            break;
          uint64_t y = x, yw = xw;
          if (has)
            { int p, cc;
              if (ma != 0)
                { int t = 31-__clz((int) ma);
                  ma &= ~(1u << t);
                  int q = 3*NA-1-t;
                  p = q/3; cc = q-3*p+1;
                }
              else if (mb != 0)
                { int t = 31-__clz((int) mb);
                  mb &= ~(1u << t);
                  int q = 3*(PH-NA)-1-t;
                  p = q/3; cc = q-3*p+1; p += NA;
                }
              else
                { int t = 0;
#pragma unroll
                  for (int w = MW-1; w >= 0; w--)
                    if (mhi[w] != 0)
                      t = 64*w + __ffsll((long long) mhi[w])-1;
#pragma unroll
                  for (int w = 0; w < MW; w++)
                    if ((t>>6) == w)
                      mhi[w] &= mhi[w]-1;
                  p = t/3; cc = t-3*p+1; p += PH;
                }
              const int sh = 62-2*(p&31);
              if (KW == 1 || p < 32)
                y = (x & ~((uint64_t) 3 << sh)) | ((uint64_t) cc << sh);
              else
                yw = (xw & ~((uint64_t) 3 << sh)) | ((uint64_t) cc << sh);
            }
          const unsigned bal = __ballot_sync(FULL,has);
          if (has)
            { int pos = qn + __popc(bal & lt);
              qy[pos] = y;
              if (KW == 2) ql[pos] = yw;
              qi[pos] = (IdxT) i;
            }
          qn += __popc(bal);
          __syncwarp();
          if (qn >= 32)
            { qn -= 32;
              uint64_t yy = qy[qn+lane];
              uint64_t yl = KW == 2 ? ql[qn+lane] : 0;
              int64_t  oi = (int64_t) qi[qn+lane];
              __syncwarp();
              int64_t j = bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,yy,yl);
              if (j >= 0)
                book_pair<IdxT>(cnt,oi,j,lo,dv,up);
            }
        }
    }

  if (lane < qn)                                          /* left-overs */
    { uint64_t yy = qy[lane];
      uint64_t yl = KW == 2 ? ql[lane] : 0;
      int64_t  oi = (int64_t) qi[lane];
      int64_t  j  = bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,yy,yl);
      if (j >= 0)
        book_pair<IdxT>(cnt,oi,j,lo,dv,up);
    }
}

template <typename IdxT, int F, int KW>
static cudaError_t launch_pass1(const uint64_t *keys, const uint64_t *keys_lo, const uint16_t *cnt, int64_t n,
                                const void *bucket, int bits, const uint32_t *filter, int kmer,
                                int64_t lo, int64_t hi, const DegView &dv, void *up, cudaStream_t st)
{ int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  int64_t nchunks = (hi-lo+31)>>5;
  int64_t want    = (nchunks+P1_WARPS-1)/P1_WARPS;
  int64_t cap     = (int64_t) sms*P1_GRID_PER_SM;
  int     grid    = (int) (want < cap ? want : cap);
  pass1_filter_kernel<IdxT,F,KW><<<grid,P1_WARPS*32,0,st>>>
      (keys,keys_lo,cnt,n,(const IdxT *) bucket,64-bits,filter,kmer,lo,hi,dv,(IdxT *) up);
  return cudaGetLastError();
}

template <typename IdxT, int KW>
static cudaError_t dispatch_pass1(int fb, const uint64_t *keys, const uint64_t *keys_lo,
                                  const uint16_t *cnt, int64_t n,
                                  const void *bucket, int bits, const uint32_t *filter, int kmer,
                                  int64_t lo, int64_t hi, const DegView &dv, void *up, cudaStream_t st)
{ switch (fb)
  {
#define CASE(P) case P: return launch_pass1<IdxT,P,KW>(keys,keys_lo,cnt,n,bucket,bits,filter,kmer,lo,hi,dv,up,st);
    CASE(22) CASE(23) CASE(24) CASE(25) CASE(26) CASE(27) CASE(28) CASE(29)
    CASE(30) CASE(31) CASE(32) CASE(33) CASE(34) CASE(35) CASE(36) CASE(37)
#undef CASE
  }
  return cudaErrorInvalidValue;
}

extern "C" int hm_k_pass1_degree(const uint64_t *d_keys, const uint64_t *d_keys_lo,
                                 const uint16_t *d_cnt, int64_t n,
                                 const void *d_bucket, int bits, int idx64,
                                 const uint32_t *d_filter, int filter_bits, int kmer,
                                 int64_t lo, int64_t hi, uint8_t *d_deg, void *d_up,
                                 const hm_shards *shards, void *stream)
{ if (kmer < 1 || kmer > HM_MAX_KMER)
    return hm_set_error(HM_EUNSUPPORTED,"k-mer length %d not supported (1..%d)",kmer,HM_MAX_KMER);
  if (lo < 0 || hi > n || lo > hi || bits < 1 || bits > 30)
    return hm_set_error(HM_EINVAL,"pass1: bad range [%lld,%lld) of %lld or bits %d",
                        (long long) lo,(long long) hi,(long long) n,bits);
  if (filter_bits < HM_FILTER_MIN_BITS || filter_bits > HM_FILTER_MAX_BITS)
    return hm_set_error(HM_EINVAL,"pass1: filter bits %d out of range",filter_bits);
  if ((kmer > 32) != (d_keys_lo != NULL))
    return hm_set_error(HM_EINVAL,"pass1: second key word array %s for k=%d",
                        d_keys_lo ? "given" : "missing",kmer);
  if (hi == lo)
    return HM_OK;
  if (shards != NULL && shards->n_shards > 1 &&
      (shards->n_shards > HM_MAX_SHARDS || shards->self < 0 || shards->self >= shards->n_shards ||
       shards->off[shards->self] != lo || shards->off[shards->self+1] != hi))
    return hm_set_error(HM_EINVAL,"pass1: [lo,hi) is not shard %d of the shard table",shards->self);
  cudaStream_t st = (cudaStream_t) stream;
  DegView dv = make_deg_view(d_deg,lo,hi,shards);
  HM_CUDA(cudaMemsetAsync(d_up,0xFF,(idx64 ? 8 : 4)*(size_t) (hi-lo),st));   /* all-ones = none */
  cudaError_t e;
  if (kmer <= 32)
    e = idx64
      ? dispatch_pass1<uint64_t,1>(filter_bits,d_keys,NULL,d_cnt,n,d_bucket,bits,d_filter,kmer,lo,hi,dv,d_up,st)
      : dispatch_pass1<uint32_t,1>(filter_bits,d_keys,NULL,d_cnt,n,d_bucket,bits,d_filter,kmer,lo,hi,dv,d_up,st);
  else
    e = idx64
      ? dispatch_pass1<uint64_t,2>(filter_bits,d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,d_filter,kmer,lo,hi,dv,d_up,st)
      : dispatch_pass1<uint32_t,2>(filter_bits,d_keys,d_keys_lo,d_cnt,n,d_bucket,bits,d_filter,kmer,lo,hi,dv,d_up,st);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"pass1_filter_kernel");
  return HM_OK;
}

/* -------------------------------------------------------------------------- pass 2 ------ */

#define P2_TS 192      /* shared-memory tile: sums  < 192 */
#define P2_TM 96       /*                     mins  <  96   (72 KB -> 3 CTAs per SM) */
#define P2_THREADS 512
#define P2_CTAS_PER_SM 3
#define P2_ILP 4

/* deg[x] <= 1 and deg[y] <= 1 for a recorded qualifying pair means both are exactly 1, i.e. the
 * pair is isolated: one count in plot[cx+cy][min].  Persistent CTAs keep the dense corner of the
 * plot in shared memory (uint32) and flush once; the rest goes to 64-bit global atomics.      */
template <typename IdxT>
__global__ void __launch_bounds__(P2_THREADS,P2_CTAS_PER_SM)
pass2_plot_kernel(const uint16_t *__restrict__ cnt, const DegView dv,
                  const IdxT *__restrict__ up, int64_t lo, int64_t hi,
                  unsigned long long *__restrict__ plot)
{ extern __shared__ uint32_t tile[];
  __shared__ unsigned s_defer;
  for (int t = threadIdx.x; t < P2_TS*P2_TM; t += blockDim.x)
    tile[t] = 0;
  if (threadIdx.x == 0)
    s_defer = 0;
  __syncthreads();
  IdxT *const defer = (IdxT *) dv.defer_ent + 2*dv.defer_cap*blockIdx.x;
  /* P2_ILP entries per thread and trip: all their independent loads (degree bytes, partner
   * indices, then both partner look-ups at once) are in flight together -- the kernel is bound by
   * the latency of the two dependent gathers, not by bytes or instructions                      */
  const int64_t stride = (int64_t) gridDim.x * blockDim.x * P2_ILP;
  for (int64_t i0 = lo + (int64_t) blockIdx.x * blockDim.x * P2_ILP + threadIdx.x; i0 < hi; i0 += stride)
    { uint8_t di[P2_ILP];
      IdxT    j[P2_ILP];
#pragma unroll
      for (int u = 0; u < P2_ILP; u++)
        { int64_t i = i0 + (int64_t) u * blockDim.x;
          di[u] = (i < hi) ? ((const uint8_t *) dv.self)[i] : (uint8_t) 0;
        }
#pragma unroll
      for (int u = 0; u < P2_ILP; u++)       /* 0: no pair at all; >1 (reference: Pair > 1): not isolated */
        j[u] = (di[u] == 1) ? up[i0 + (int64_t) u * blockDim.x - lo] : IdxNone<IdxT>::value;
      uint8_t dj[P2_ILP];
      int     ci[P2_ILP], cj[P2_ILP];
#pragma unroll
      for (int u = 0; u < P2_ILP; u++)
        { dj[u] = 2; ci[u] = cj[u] = 0;
          if (j[u] != IdxNone<IdxT>::value)
            { const uint8_t *pj = (const uint8_t *) deg_words(dv,(int64_t) j[u]);
              if (pj != (const uint8_t *) dv.self)
                { /* partner owned by another GPU: an NVLink round trip.  Park the pair in this
                   * CTA's slice of the defer list; pass2_deferred_kernel resolves all of them with
                   * every remote load in flight at once (inline only when the slice is full)      */
                  unsigned at = dv.defer_cap > 0 ? atomicAdd(&s_defer,1u) : 0xffffffffu;
                  if ((int64_t) at < dv.defer_cap)
                    { defer[2*at] = (IdxT) (i0 + (int64_t) u * blockDim.x); defer[2*at+1] = j[u]; continue; }
                  dj[u] = __ldcv(pj+j[u]);
                }
              else
                dj[u] = __ldg(pj+j[u]);
              cj[u] = __ldg(cnt+j[u]);
              ci[u] = cnt[i0 + (int64_t) u * blockDim.x];
            }
        }
#pragma unroll
      for (int u = 0; u < P2_ILP; u++)
        if (dj[u] <= 1)
          { int s = ci[u]+cj[u];
            int m = ci[u] < cj[u] ? ci[u] : cj[u];
            if (s < P2_TS && m < P2_TM)
              atomicAdd(tile + s*P2_TM + m, 1u);
            else
              atomicAdd(plot + s*HM_PLOT_W + m, 1ull);
          }
    }
  __syncthreads();
  if (threadIdx.x == 0 && dv.defer_cap > 0)
    dv.defer_cnt[blockIdx.x] = (s_defer < (unsigned) dv.defer_cap) ? s_defer : (unsigned) dv.defer_cap;
  for (int t = threadIdx.x; t < P2_TS*P2_TM; t += blockDim.x)
    { uint32_t v = tile[t];
      if (v != 0)
        atomicAdd(plot + (t/P2_TM)*HM_PLOT_W + (t%P2_TM), (unsigned long long) v);
    }
}

/* the pairs pass2_plot_kernel parked: partner's incidence byte lives on another GPU */
template <typename IdxT>
__global__ void __launch_bounds__(256)
pass2_deferred_kernel(const uint16_t *__restrict__ cnt, const DegView dv,
                      unsigned long long *__restrict__ plot)
{ const unsigned nb = dv.defer_cnt[blockIdx.x];
  const IdxT *defer = (const IdxT *) dv.defer_ent + 2*dv.defer_cap*blockIdx.x;
  for (unsigned e = threadIdx.x; e < nb; e += blockDim.x)
    { int64_t i = (int64_t) defer[2*e], j = (int64_t) defer[2*e+1];
      const uint8_t *pj = (const uint8_t *) deg_words(dv,j);
      if (__ldcv(pj+j) > 1)
        continue;
      int ci = cnt[i], cj = __ldg(cnt+j);
      int s  = ci+cj;
      int m  = ci < cj ? ci : cj;
      atomicAdd(plot + s*HM_PLOT_W + m, 1ull);
    }
}

extern "C" int64_t hm_pass2_scratch_bytes(int64_t range, int idx64)
{ int64_t cap = range/16 + 65536;            /* foreign partners are a few % of the isolated pairs */
  return P2_DEFER_HEADER + cap * 2 * (idx64 ? 8 : 4);
}

extern "C" int hm_k_pass2_plot(const uint16_t *d_cnt, const uint8_t *d_deg, const void *d_up,
                               int idx64, int64_t lo, int64_t hi, unsigned long long *d_plot,
                               const hm_shards *shards, void *stream)
{ static int configured[64] = {0};
  if (lo > hi)
    return hm_set_error(HM_EINVAL,"pass2: bad range");
  if (hi == lo)
    return HM_OK;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  size_t smem = (size_t) P2_TS*P2_TM*sizeof(uint32_t);
  if (dev < 64 && !configured[dev])
    { cudaError_t e1 = cudaFuncSetAttribute(pass2_plot_kernel<uint32_t>,
                                            cudaFuncAttributeMaxDynamicSharedMemorySize,(int) smem);
      cudaError_t e2 = cudaFuncSetAttribute(pass2_plot_kernel<uint64_t>,
                                            cudaFuncAttributeMaxDynamicSharedMemorySize,(int) smem);
      if (e1 != cudaSuccess || e2 != cudaSuccess)
        return hm_cuda_fail(e1 != cudaSuccess ? e1 : e2,"cudaFuncSetAttribute(pass2)");
      configured[dev] = 1;
    }
  int64_t want = (hi-lo+P2_THREADS*P2_ILP-1)/(P2_THREADS*P2_ILP);
  int     grid = (int) (want < sms*P2_CTAS_PER_SM ? want : sms*P2_CTAS_PER_SM);
  DegView dv   = make_deg_view((uint8_t *) d_deg,lo,hi,shards);
  if (grid > P2_DEFER_HEADER/4) grid = P2_DEFER_HEADER/4;
  if (dv.n > 1 && shards->scratch != NULL &&
      shards->scratch_bytes >= P2_DEFER_HEADER + (int64_t) grid*2*(idx64 ? 8 : 4))
    { dv.defer_cnt = (uint32_t *) shards->scratch;
      dv.defer_ent = (uint8_t *) shards->scratch + P2_DEFER_HEADER;
      dv.defer_cap = (shards->scratch_bytes-P2_DEFER_HEADER) / (2*(idx64 ? 8 : 4)) / grid;
    }
  if (idx64)
    pass2_plot_kernel<uint64_t><<<grid,P2_THREADS,smem,(cudaStream_t) stream>>>
        (d_cnt,dv,(const uint64_t *) d_up,lo,hi,d_plot);
  else
    pass2_plot_kernel<uint32_t><<<grid,P2_THREADS,smem,(cudaStream_t) stream>>>
        (d_cnt,dv,(const uint32_t *) d_up,lo,hi,d_plot);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"pass2_plot_kernel");
  if (dv.defer_cap > 0)
    { if (idx64) pass2_deferred_kernel<uint64_t><<<grid,256,0,(cudaStream_t) stream>>>(d_cnt,dv,d_plot);
      else       pass2_deferred_kernel<uint32_t><<<grid,256,0,(cudaStream_t) stream>>>(d_cnt,dv,d_plot);
      e = cudaGetLastError();
      if (e != cudaSuccess)
        return hm_cuda_fail(e,"pass2_deferred_kernel");
    }
  return HM_OK;
}

/* ------------------------------------------------------------- pass 2, extract variant -- */

/* extract_kmer_pairs (src/lib/PloidyList.c): same isolated pairs as pass 2, but instead of
 * counting pixel (sum, min) the pair is written out when the pixel carries a smudge label
 * (PLOT[x][min] > 0, PloidyList.c:433-447,688-702).  The k-mer printed is the one with the HIGHER
 * count (on a tie the one with the smaller base), annotated with the other one's base at the
 * varying position -- print_het(seq,len,half,alt), PloidyList.c:128-165.                       */
/* entry i's record, if it has one (an isolated pair whose pixel carries a label) */
template <typename IdxT>
__device__ __forceinline__ bool pass2_pair(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                                           const uint16_t *__restrict__ cnt, const DegView &dv,
                                           const IdxT *__restrict__ up, int64_t lo, int64_t i,
                                           const uint16_t *__restrict__ pixmap, hm_pair_rec &r)
{ if (((const uint8_t *) dv.self)[i] != 1)
    return false;
  IdxT j = up[i-lo];
  if (j == IdxNone<IdxT>::value)
    return false;
  const uint8_t *dj = (const uint8_t *) deg_words(dv,(int64_t) j);
  if ((dj == (const uint8_t *) dv.self ? __ldg(dj+j) : __ldcv(dj+j)) > 1)
    return false;
  int ci = cnt[i], cj = __ldg(cnt+j);
  int s  = ci+cj;
  int m  = ci < cj ? ci : cj;
  unsigned pix = pixmap[s*HM_PLOT_W + m];
  if (pix == 0)
    return false;
  uint64_t xh = keys[i], yh = __ldg(keys+j);
  uint64_t xl = keys_lo ? keys_lo[i] : 0, yl = keys_lo ? __ldg(keys_lo+j) : 0;
  int pos = (xh != yh) ? (__clzll((long long) (xh ^ yh)) >> 1)
                       : 32 + (__clzll((long long) (xl ^ yl)) >> 1);
  int sh  = 62-2*(pos&31);
  int bi  = (int) (((pos < 32 ? xh : xl) >> sh) & 3);      /* i < j: bi < bj */
  int bj  = (int) (((pos < 32 ? yh : yl) >> sh) & 3);
  if (ci < cj) { r.key_hi = yh; r.key_lo = yl; r.alt = (uint8_t) bi; }   /* PloidyList.c:433-439 */
  else         { r.key_hi = xh; r.key_lo = xl; r.alt = (uint8_t) bj; }   /*              :441-447 */
  r.smudge = pix; r.pos = (uint8_t) pos; r.pad = 0;
  return true;
}

template <typename IdxT>
__global__ void __launch_bounds__(256)
pass2_extract_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                     const uint16_t *__restrict__ cnt, const DegView dv,
                     const IdxT *__restrict__ up, int64_t lo, int64_t hi,
                     const uint16_t *__restrict__ pixmap, hm_pair_rec *__restrict__ out,
                     unsigned long long cap, unsigned long long *__restrict__ count)
{ int64_t stride = (int64_t) gridDim.x * blockDim.x;
  for (int64_t i = lo + (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < hi; i += stride)
    { hm_pair_rec r;
      if (!pass2_pair<IdxT>(keys,keys_lo,cnt,dv,up,lo,i,pixmap,r))
        continue;
      unsigned long long at = atomicAdd(count,1ull);
      if (at < cap)
        out[at] = r;
    }
}

/* pass2_extract_kernel's records by key prefix (the top hb bits of key_hi), as PrefixSink takes the symmetric
 * route's: HIST = true adds each to hist[prefix]; HIST = false stores those with p0 <= prefix < p1 into out, one
 * atomic per warp on the counter, which counts past cap.  The warps stride together so that every lane of a
 * warp reaches the warp-wide steps.                                                                           */
template <typename IdxT, bool HIST>
__global__ void __launch_bounds__(256)
pass2_pairs_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                   const uint16_t *__restrict__ cnt, const DegView dv,
                   const IdxT *__restrict__ up, int64_t lo, int64_t hi,
                   const uint16_t *__restrict__ pixmap, int hb, unsigned long long *__restrict__ hist,
                   uint64_t p0, uint64_t p1, hm_pair_rec *__restrict__ out,
                   unsigned long long cap, unsigned long long *__restrict__ count)
{ const int      lane = threadIdx.x & 31;
  const unsigned lt = (1u << lane) - 1;
  int64_t stride = (int64_t) gridDim.x * blockDim.x;
  for (int64_t w = lo + (int64_t) blockIdx.x * blockDim.x + (threadIdx.x & ~31); w < hi; w += stride)
    { const int64_t i = w + lane;
      hm_pair_rec   r;
      const bool    has = i < hi && pass2_pair<IdxT>(keys,keys_lo,cnt,dv,up,lo,i,pixmap,r);
      const uint64_t f  = has ? r.key_hi >> (64-hb) : 0;
      if (HIST)
        { warp_count(hist,has,f);
          continue;
        }
      const bool     in = has && f >= p0 && f < p1;
      const unsigned b  = __ballot_sync(0xffffffffu,in);
      if (b == 0)
        continue;
      unsigned long long at = 0;
      if (lane == 0)
        at = atomicAdd(count,(unsigned long long) __popc(b));
      at = __shfl_sync(0xffffffffu,at,0) + (unsigned long long) __popc(b & lt);
      if (in && at < cap)
        out[at] = r;
    }
}

extern "C" int hm_k_pass2_extract(const uint64_t *d_keys, const uint64_t *d_keys_lo,
                                  const uint16_t *d_cnt, const uint8_t *d_deg, const void *d_up,
                                  int idx64, int64_t lo, int64_t hi, const uint16_t *d_pixmap,
                                  hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count,
                                  const hm_shards *shards, void *stream)
{ if (lo > hi || cap < 0)
    return hm_set_error(HM_EINVAL,"extract: bad range or capacity");
  if (hi == lo)
    return HM_OK;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  int64_t want = (hi-lo+255)/256;
  int     grid = (int) (want < sms*8 ? want : sms*8);
  DegView dv   = make_deg_view((uint8_t *) d_deg,lo,hi,shards);
  if (idx64)
    pass2_extract_kernel<uint64_t><<<grid,256,0,(cudaStream_t) stream>>>
        (d_keys,d_keys_lo,d_cnt,dv,(const uint64_t *) d_up,lo,hi,d_pixmap,d_out,(unsigned long long) cap,d_count);
  else
    pass2_extract_kernel<uint32_t><<<grid,256,0,(cudaStream_t) stream>>>
        (d_keys,d_keys_lo,d_cnt,dv,(const uint32_t *) d_up,lo,hi,d_pixmap,d_out,(unsigned long long) cap,d_count);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"pass2_extract_kernel");
  return HM_OK;
}

int hm_pass2_pairs_sweep(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                         const uint8_t *d_deg, const void *d_up, int idx64, int64_t lo, int64_t hi,
                         const uint16_t *d_pixmap, int hb, unsigned long long *d_hist, uint64_t p0,
                         uint64_t p1, hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count,
                         const hm_shards *shards, void *stream)
{ if (lo > hi || cap < 0 || hb < 1 || hb > 32 || d_pixmap == NULL ||
      (d_hist == NULL && (d_count == NULL || (cap > 0 && d_out == NULL))))
    return hm_set_error(HM_EINVAL,"pass2_pairs_sweep: bad arguments");
  if (hi == lo)
    return HM_OK;
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms,cudaDevAttrMultiProcessorCount,dev);
  int64_t want = (hi-lo+255)/256;
  int     grid = (int) (want < sms*8 ? want : sms*8);
  DegView dv   = make_deg_view((uint8_t *) d_deg,lo,hi,shards);
  cudaStream_t st = (cudaStream_t) stream;
  const unsigned long long c = (unsigned long long) cap;
  if (idx64 && d_hist != NULL)
    pass2_pairs_kernel<uint64_t,true><<<grid,256,0,st>>>
        (d_keys,d_keys_lo,d_cnt,dv,(const uint64_t *) d_up,lo,hi,d_pixmap,hb,d_hist,p0,p1,d_out,c,d_count);
  else if (idx64)
    pass2_pairs_kernel<uint64_t,false><<<grid,256,0,st>>>
        (d_keys,d_keys_lo,d_cnt,dv,(const uint64_t *) d_up,lo,hi,d_pixmap,hb,d_hist,p0,p1,d_out,c,d_count);
  else if (d_hist != NULL)
    pass2_pairs_kernel<uint32_t,true><<<grid,256,0,st>>>
        (d_keys,d_keys_lo,d_cnt,dv,(const uint32_t *) d_up,lo,hi,d_pixmap,hb,d_hist,p0,p1,d_out,c,d_count);
  else
    pass2_pairs_kernel<uint32_t,false><<<grid,256,0,st>>>
        (d_keys,d_keys_lo,d_cnt,dv,(const uint32_t *) d_up,lo,hi,d_pixmap,hb,d_hist,p0,p1,d_out,c,d_count);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"pass2_pairs_kernel");
  return HM_OK;
}

/* ------------------------------------------------------------------------- examine ------ */

__global__ void __launch_bounds__(256)
min_count_kernel(const uint16_t *__restrict__ cnt, int64_t frst, int64_t last, int *out)
{ int     best = 0x8000;
  int64_t stride = (int64_t) gridDim.x * blockDim.x;
  for (int64_t i = frst + (int64_t) blockIdx.x * blockDim.x + threadIdx.x; i < last; i += stride)
    { int v = (int) (int16_t) cnt[i];          /* the reference reads counts as int16 (:1189) */
      if (v >= 1 && v < best) best = v;
    }
  for (int o = 16; o > 0; o >>= 1)
    { int w = __shfl_xor_sync(0xffffffffu,best,o);
      if (w < best) best = w;
    }
  if ((threadIdx.x & 31) == 0 && best < 0x8000)
    atomicMin(out,best);
}

extern "C" int hm_k_min_count(const uint16_t *d_cnt, int64_t frst, int64_t last, int *d_min,
                              void *stream)
{ if (last <= frst)
    return HM_OK;
  int64_t want = (last-frst+255)/256;
  int     grid = (int) (want < 132*8 ? want : 132*8);
  min_count_kernel<<<grid,256,0,(cudaStream_t) stream>>>(d_cnt,frst,last,d_min);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"min_count_kernel");
  return HM_OK;
}

template <typename IdxT, int KW>
__global__ void __launch_bounds__(128)
find_keys_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ keys_lo,
                 const IdxT *__restrict__ bucket, int bshift,
                 const uint64_t *__restrict__ query, const uint64_t *__restrict__ query_lo,
                 int64_t nq, int64_t *__restrict__ pos)
{ int64_t q = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (q < nq)
    pos[q] = bucket_find<IdxT,KW>(keys,keys_lo,bucket,bshift,query[q],KW == 2 ? query_lo[q] : 0);
}

extern "C" int hm_k_find_keys(const uint64_t *d_keys, const uint64_t *d_keys_lo, int64_t n,
                              const void *d_bucket, int bits, int idx64,
                              const uint64_t *d_query, const uint64_t *d_query_lo, int64_t nq,
                              int64_t *d_pos, void *stream)
{ (void) n;
  if (nq <= 0)
    return HM_OK;
  if ((d_keys_lo != NULL) != (d_query_lo != NULL))
    return hm_set_error(HM_EINVAL,"find_keys: table and queries must have the same number of key words");
  int64_t      nblk = (nq+127)/128;
  cudaStream_t st = (cudaStream_t) stream;
  int          sh = 64-bits;
  if (d_keys_lo == NULL)
    { if (idx64)
        find_keys_kernel<uint64_t,1><<<(unsigned) nblk,128,0,st>>>(d_keys,NULL,(const uint64_t *) d_bucket,sh,d_query,NULL,nq,d_pos);
      else
        find_keys_kernel<uint32_t,1><<<(unsigned) nblk,128,0,st>>>(d_keys,NULL,(const uint32_t *) d_bucket,sh,d_query,NULL,nq,d_pos);
    }
  else
    { if (idx64)
        find_keys_kernel<uint64_t,2><<<(unsigned) nblk,128,0,st>>>(d_keys,d_keys_lo,(const uint64_t *) d_bucket,sh,d_query,d_query_lo,nq,d_pos);
      else
        find_keys_kernel<uint32_t,2><<<(unsigned) nblk,128,0,st>>>(d_keys,d_keys_lo,(const uint32_t *) d_bucket,sh,d_query,d_query_lo,nq,d_pos);
    }
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"find_keys_kernel");
  return HM_OK;
}

/*******************************************************************************************
 * hm_condition.cu -- table conditioning on the GPU: the two things the reference delegates to external
 * FastK executables before it scans (PloidyPlot.c:1381-1426):
 *
 *   trim        `Logex -T<t> '<tmp>.trim=A[<L>-]' <table>`   keep entries with count >= L
 *   symmetrise  `Symmex -T<t> -P<dir> <table> <tmp>.symx`     add the reverse complement of every
 *                                                             k-mer (same count), keep the table sorted
 *
 * FastK's tools are not part of the reference tree and are not pinned to a version (SURVEY.md §8c), so this
 * restates their documented effect, not their code: parity for THIS step is pinned only against a numpy
 * restatement in tests/.  Where a reverse complement equals an original (palindromes at even k, a source
 * holding both strands) the original wins.
 *
 * One algorithm, a key range at a time (DESIGN.md §4d), behind three drivers: hm_scan_condition (the resident
 * table, in place) and hm_scan_condition_files (new FastK files) in hm_scan.cu, and the ranks of a
 * one-process-per-GPU job in hm_shard_condition.cu.  The steps here:
 *
 *   cond_hist_kernel     output histogram: kept originals + their reverse complements per key prefix
 *   cond_gather_kernel   one source chunk -> the range's reverse complements (warp-aggregated appends)
 *                        and the tile counts of its kept originals
 *   cond_scan_kernel     tile counts -> tile offsets (one CTA)
 *   cond_orig_kernel     the range's kept originals, in source order (so already sorted)
 *   cond_dup_kernel      merge, step 1: which entries have an equal key on the other side
 *   cond_merge_kernel    merge, step 2: every entry to its output rank; reverse complements that equal an
 *                        original are dropped
 *   cond_pack_kernel     (keys, counts) -> FastK records (the inverse of unpack_records_kernel) + the range's
 *                        stub-index bucket counts
 * The reverse complements are sorted with CUB's radix sort (not the hot path).  The merge ranks by binary
 * search instead of a merge path: every entry finds its rank on the other side (log n probes into L2-resident
 * neighbourhoods), and duplicates are settled with tile-count prefix sums.  hm_sort_keys (the streamed scan's
 * S list) sorts with the same two-pass scheme.
 *******************************************************************************************/
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "hetmers_b200.h"
#include "hm_internal.h"
#include "hm_device.cuh"

#define FULL 0xffffffffu

__device__ __forceinline__ uint64_t kmer_prefix(uint64_t x, int bits) { return x >> (64-bits); }

template <int KW>
__device__ __forceinline__ void load_key(const uint64_t *keys, const uint64_t *klo, int64_t i, uint64_t &x, uint64_t &xl)
{ x = keys[i]; xl = KW == 2 ? klo[i] : 0; }

template <int KW>
__device__ __forceinline__ bool key_less(uint64_t a, uint64_t al, uint64_t b, uint64_t bl)
{ return a < b || (KW == 2 && a == b && al < bl); }

/* first index in sorted (keys, klo)[0, n) whose key is not below (x, xl) */
template <int KW>
__device__ __forceinline__ int64_t lower_bound(const uint64_t *keys, const uint64_t *klo, int64_t n, uint64_t x, uint64_t xl)
{ int64_t l = 0, r = n;
  while (l < r)
    { int64_t m = (l+r) >> 1;
      if (key_less<KW>(keys[m],KW == 2 ? klo[m] : 0,x,xl)) l = m+1;
      else                                                 r = m;
    }
  return l;
}

template <int KW>
__global__ void __launch_bounds__(CT)
cond_hist_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ klo, const uint16_t *__restrict__ cnt,
                 int64_t m, int kmer, int ethresh, int do_symm, int hb, unsigned long long *__restrict__ hist)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  const bool    kept = i < m && cnt[i] >= ethresh;
  uint64_t x = 0, xl = 0;
  if (kept) load_key<KW>(keys,klo,i,x,xl);
  warp_count(hist,kept,kmer_prefix(x,hb));
  if (do_symm)
    { uint64_t r, rl;
      revcomp_kmer<KW>(x,xl,kmer,r,rl);
      warp_count(hist,kept,kmer_prefix(r,hb));
    }
}

/* ctr: [0] originals gathered, [1] reverse complements gathered, [3] overflow (hm_cond_bufs) */
template <int KW>
__global__ void __launch_bounds__(CT)
cond_gather_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ klo, const uint16_t *__restrict__ cnt,
                   int64_t m, int kmer, int ethresh, int do_symm, int hb, uint64_t p0, uint64_t p1,
                   unsigned long long *__restrict__ tiles, uint64_t *__restrict__ c_key, uint64_t *__restrict__ c_lo,
                   uint16_t *__restrict__ c_cnt, int64_t c_room, unsigned long long *__restrict__ ctr)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  const bool    kept = i < m && cnt[i] >= ethresh;
  uint64_t x = 0, xl = 0;
  uint16_t c = 0;
  if (kept) { load_key<KW>(keys,klo,i,x,xl); c = cnt[i]; }
  const uint64_t p = kmer_prefix(x,hb);
  const int n_in = __syncthreads_count(kept && p >= p0 && p < p1);
  if (threadIdx.x == 0) tiles[blockIdx.x] = (unsigned long long) n_in;
  if (!do_symm)
    return;
  uint64_t r, rl;
  revcomp_kmer<KW>(x,xl,kmer,r,rl);
  const uint64_t rp = kmer_prefix(r,hb);
  const bool     in = kept && rp >= p0 && rp < p1;
  const unsigned b = __ballot_sync(FULL,in);
  if (b == 0)
    return;
  const int lane = threadIdx.x & 31, leader = __ffs(b)-1;
  unsigned long long base = 0;
  if (lane == leader) base = atomicAdd(ctr+1,(unsigned long long) __popc(b));
  base = __shfl_sync(FULL,base,leader);
  if (in)
    { const int64_t slot = (int64_t) base + __popc(b & ((1u << lane)-1));
      if (slot < c_room)                      /* c_key etc. point at the END of the shared region: fill downwards */
        { c_key[-1-slot] = r; if (KW == 2) c_lo[-1-slot] = rl; c_cnt[-1-slot] = c; }
      else
        atomicOr(ctr+3,1ull);
    }
}

/* tiles[0, nt): counts -> exclusive offsets + *base; *base += total (one CTA of 1024 threads) */
__global__ void __launch_bounds__(1024)
cond_scan_kernel(unsigned long long *__restrict__ tiles, int64_t nt, unsigned long long *__restrict__ base)
{ __shared__ unsigned long long s[1024];
  const int64_t per = (nt+1023)/1024, a = threadIdx.x*per, e = a+per < nt ? a+per : nt;
  unsigned long long sum = 0;
  for (int64_t t = a; t < e; t++) sum += tiles[t];
  s[threadIdx.x] = sum;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1)                       /* inclusive Hillis-Steele scan of the sums */
    { unsigned long long v = threadIdx.x >= (unsigned) o ? s[threadIdx.x-o] : 0;
      __syncthreads();
      s[threadIdx.x] += v;
      __syncthreads();
    }
  const unsigned long long b0 = *base;
  unsigned long long run = b0 + s[threadIdx.x] - sum;
  for (int64_t t = a; t < e; t++)
    { unsigned long long v = tiles[t];
      tiles[t] = run;
      run += v;
    }
  __syncthreads();
  if (threadIdx.x == 1023) *base = b0 + s[1023];
}

template <int KW>
__global__ void __launch_bounds__(CT)
cond_orig_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ klo, const uint16_t *__restrict__ cnt,
                 int64_t m, int ethresh, int hb, uint64_t p0, uint64_t p1, const unsigned long long *__restrict__ tiles,
                 uint64_t *__restrict__ o_key, uint64_t *__restrict__ o_lo, uint16_t *__restrict__ o_cnt, int64_t o_room,
                 unsigned long long *__restrict__ ctr)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  const bool    kept = i < m && cnt[i] >= ethresh;
  uint64_t x = 0, xl = 0;
  if (kept) load_key<KW>(keys,klo,i,x,xl);
  const uint64_t p = kmer_prefix(x,hb);
  const bool     in = kept && p >= p0 && p < p1;
  const int rank = cta_rank(in);
  if (in)
    { const int64_t slot = (int64_t) tiles[blockIdx.x] + rank;
      if (slot < o_room) { o_key[slot] = x; if (KW == 2) o_lo[slot] = xl; o_cnt[slot] = cnt[i]; }
      else               atomicOr(ctr+3,1ull);
    }
}

/* tiles[t] = entries of tile t of (a) that also occur in (b) */
template <int KW>
__global__ void __launch_bounds__(CT)
cond_dup_kernel(const uint64_t *__restrict__ a, const uint64_t *__restrict__ al, int64_t na,
                const uint64_t *__restrict__ b, const uint64_t *__restrict__ bl, int64_t nb,
                unsigned long long *__restrict__ tiles)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  bool dup = false;
  if (i < na)
    { uint64_t x, xl;
      load_key<KW>(a,al,i,x,xl);
      const int64_t j = lower_bound<KW>(b,bl,nb,x,xl);
      dup = j < nb && b[j] == x && (KW == 1 || bl[j] == xl);
    }
  const int n = __syncthreads_count(dup);
  if (threadIdx.x == 0) tiles[blockIdx.x] = (unsigned long long) n;
}

/* entry i of (a) goes to i + (entries of b below it) - (entries of a before i that occur in b): the equal
 * entries of b are the ones the merge drops (originals = a) or a's own dropped entries (reverse
 * complements = a, drop_dups)                                                                          */
template <int KW>
__global__ void __launch_bounds__(CT)
cond_merge_kernel(const uint64_t *__restrict__ a, const uint64_t *__restrict__ al, const uint16_t *__restrict__ ac,
                  int64_t na, const uint64_t *__restrict__ b, const uint64_t *__restrict__ bl, int64_t nb,
                  const unsigned long long *__restrict__ tiles, int drop_dups,
                  uint64_t *__restrict__ o_key, uint64_t *__restrict__ o_lo, uint16_t *__restrict__ o_cnt)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  bool     dup = false;
  uint64_t x = 0, xl = 0;
  int64_t  j = 0;
  if (i < na)
    { load_key<KW>(a,al,i,x,xl);
      j = lower_bound<KW>(b,bl,nb,x,xl);
      dup = j < nb && b[j] == x && (KW == 1 || bl[j] == xl);
    }
  const int before = (int) tiles[blockIdx.x] + cta_rank(dup);
  if (i < na && !(drop_dups && dup))
    { const int64_t at = i + j - before;
      o_key[at] = x; if (KW == 2) o_lo[at] = xl; o_cnt[at] = ac[i];
    }
}

/* FastK records: key bytes ibyte..kbyte-1 (big-endian packing), then the count little-endian; bcount[bucket-b0]
 * += 1 for the stub-index bucket (the first ibyte bytes) of every record                                     */
template <int KW>
__global__ void __launch_bounds__(CT)
cond_pack_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ klo, const uint16_t *__restrict__ cnt,
                 int64_t n, int ibyte, int kbyte, uint64_t b0, uint8_t *__restrict__ rec,
                 unsigned long long *__restrict__ bcount)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  const int     pbyte = kbyte-ibyte+2;
  uint64_t x = 0, xl = 0;
  if (i < n)
    { load_key<KW>(keys,klo,i,x,xl);
      uint8_t *r = rec + i*pbyte;
      for (int j = ibyte; j < kbyte; j++)
        r[j-ibyte] = (uint8_t) (j < 8 ? x >> (56-8*j) : xl >> (56-8*(j-8)));
      const uint16_t c = cnt[i];
      r[kbyte-ibyte]   = (uint8_t) (c & 0xFF);
      r[kbyte-ibyte+1] = (uint8_t) (c >> 8);
    }
  warp_count(bcount,i < n,kmer_prefix(x,8*ibyte)-b0);
}

__global__ void __launch_bounds__(CT)
cond_iota_kernel(uint32_t *__restrict__ idx, int64_t n)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  if (i < n) idx[i] = (uint32_t) i;
}

template <typename T>
__global__ void __launch_bounds__(CT)
cond_permute_kernel(const T *__restrict__ src, const uint32_t *__restrict__ idx, int64_t n, T *__restrict__ dst)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

#define LAUNCHED(what) do { cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return hm_cuda_fail(_e,what); } while (0)

/* ---- sizes and plan (host only, no CUDA calls) ------------------------------------------------------- */

static int64_t align256(int64_t b) { return (b+255) & ~255ll; }

/* CUB's scratch for a double-buffered radix sort of c pairs: histograms and look-back state, well under a
 * byte per entry; checked against CUB's own figure before every sort                                 */
static int64_t sort_room(int64_t c) { return align256(c + (16ll << 20)); }

static int64_t tiles_bytes(int64_t n) { return align256(8*(n/CT+2)); }

extern "C" int64_t hm_condition_range_bytes(int64_t t, int do_symm, int kmer, int ibyte)
{ const int64_t KW = kmer > 32 ? 2 : 1, E = 8*KW+2, pbyte = ((kmer+3)>>2) - ibyte + 2;
  int64_t b = E*align256(t) + pbyte*t + 256;               /* originals + reverse complements, records */
  if (do_symm)                                             /* sort buffers, permutation pair, merged table */
    b += E*align256(t) + (KW == 2 ? 8*align256(t) : 0) + sort_room(t) + E*align256(t) + 2*tiles_bytes(t);
  return align256(b) + 8*256;
}

/* fixed bytes besides a chunk: stub index, the range's bucket counts, histogram, counters */
static int64_t base_fixed(int ibyte, int hb)
{ return align256(8ll << (8*ibyte))*2 + align256(8ll << hb) + 256; }

/* a loaded chunk of c source entries: keys (+ second words) and counts, two staging buffers, tile counts */
static int64_t chunk_fixed(int64_t c, int kmer, int ibyte)
{ const int64_t KW = kmer > 32 ? 2 : 1, pbyte = ((kmer+3)>>2) - ibyte + 2;
  return align256(8*(c+1))*KW + align256(2*(c+8)) + 2*align256(c*pbyte) + tiles_bytes(c);
}

#define COND_CHUNK     (8ll << 20)              /* source entries per chunk at most (the loader's staged chunk) */
#define COND_MIN_CHUNK 256

/* the chunk for a budget: the largest power-of-two fraction of COND_CHUNK (or n) within a quarter of it */
static int64_t pick_chunk(int64_t n, int kmer, int ibyte, int64_t budget)
{ int64_t c = n < COND_CHUNK ? (n > 0 ? n : 1) : COND_CHUNK;
  while (c > COND_MIN_CHUNK && chunk_fixed(c,kmer,ibyte) > budget/4)
    c = (c+1)/2;
  return c;
}

extern "C" int hm_condition_plan(int64_t n, int kmer, int ibyte, int64_t budget, int do_symm, const int64_t *hist,
                                 int hist_bits, int64_t *cuts, hm_condition_layout *out)
{ if (out == NULL || cuts == NULL || hist == NULL || n < 0 || kmer < 1 || kmer > HM_MAX_KMER || ibyte < 1 ||
      ibyte > 3 || budget < 0 || hist_bits < 1 || hist_bits > HM_COND_HIST_BITS || hist_bits > 2*kmer)
    return hm_set_error(HM_EINVAL,"hm_condition_plan: bad arguments");
  memset(out,0,sizeof(*out));
  out->budget = budget; out->hist_bits = hist_bits;
  out->chunk = pick_chunk(n,kmer,ibyte,budget);
  const int64_t fixed = base_fixed(ibyte,hist_bits), cb = chunk_fixed(out->chunk,kmer,ibyte);
  out->fixed_bytes = fixed + cb;
  out->range_room  = budget - budget/4 - fixed;            /* the chunk takes at most the other quarter */
  const int64_t lo = hm_cond_range_limit(out->range_room,hm_condition_range_bytes,do_symm,kmer,ibyte);
  int64_t big = 0, cap = 0;
  const int r = hm_cond_cut(hist,(int64_t) 1 << hist_bits,lo,cuts,&cap,&big);
  if (cb > budget/4 || out->range_room <= 0 || r < 1 || (lo < 1 && n > 0))
    return hm_set_error(HM_ENOMEM,"a device budget of %lld bytes cannot hold one range of the conditioning: %lld bytes "
                        "are fixed (stub index, bucket counts, histogram, a chunk of %lld entries) and the largest key "
                        "prefix needs a range of %lld entries, %lld more bytes",(long long) budget,
                        (long long) out->fixed_bytes,(long long) out->chunk,(long long) big,
                        (long long) hm_condition_range_bytes(big,do_symm,kmer,ibyte));
  out->n_ranges = r;
  out->range_cap = cap;
  out->range_bytes = hm_condition_range_bytes(cap,do_symm,kmer,ibyte);
  return HM_OK;
}

int64_t hm_cond_range_limit(int64_t room, hm_cond_bytes_fn bytes, int do_symm, int kmer, int ibyte)
{ int64_t lo = 0, hi = HM_COND_MAX_RANGE;                  /* bisection: bytes grows with t */
  while (lo < hi)
    { int64_t mid = lo + (hi-lo+1)/2;
      if (bytes(mid,do_symm,kmer,ibyte) <= room) lo = mid;
      else                                       hi = mid-1;
    }
  return lo;
}

int hm_cond_cut(const int64_t *hist, int64_t np, int64_t limit, int64_t *cuts, int64_t *range_cap, int64_t *big)
{ int64_t t = 0, tmax = 0;
  int     r = 0;
  *big = 0;
  for (int64_t p = 0; p < np; p++)
    if (hist[p] > *big) *big = hist[p];
  if (*big > limit)
    return 0;
  cuts[0] = 0;
  for (int64_t p = 0; p < np; p++)
    { if (t + hist[p] > limit)                              /* the range so far is full: p starts the next */
        { cuts[++r] = p;
          if (t > tmax) tmax = t;
          t = 0;
        }
      t += hist[p];
    }
  if (t > tmax) tmax = t;
  cuts[++r] = np;
  *range_cap = tmax;
  return r;
}

/* ---- device steps (hm_scan.cu and hm_shard_condition.cu drive them) ---------------------------------- */

int64_t hm_cond_chunk(int64_t n, int kmer, int ibyte, int64_t budget) { return pick_chunk(n,kmer,ibyte,budget); }
int64_t hm_cond_tiles_bytes(int64_t n) { return tiles_bytes(n); }
int64_t hm_cond_sort_room(int64_t c) { return sort_room(c); }

int hm_cond_hist(const uint64_t *keys, const uint64_t *klo, const uint16_t *cnt, int64_t m, int kmer, int ethresh,
                 int do_symm, int hb, unsigned long long *hist, cudaStream_t st)
{ if (m <= 0) return HM_OK;
  if (kmer > 32) cond_hist_kernel<2><<<grid(m),CT,0,st>>>(keys,klo,cnt,m,kmer,ethresh,do_symm,hb,hist);
  else           cond_hist_kernel<1><<<grid(m),CT,0,st>>>(keys,klo,cnt,m,kmer,ethresh,do_symm,hb,hist);
  LAUNCHED("cond_hist_kernel");
  return HM_OK;
}

int hm_cond_gather(const uint64_t *keys, const uint64_t *klo, const uint16_t *cnt, int64_t m, const hm_cond_bufs *B,
                   uint64_t p0, uint64_t p1, unsigned long long *tiles, cudaStream_t st)
{ if (m <= 0) return HM_OK;
  const int64_t T = B->cap;
  uint64_t *ck = B->key+T, *cl = B->lo ? B->lo+T : NULL;    /* reverse complements fill the region from its end */
  uint16_t *cc = B->cnt+T;
  if (B->kmer > 32)
    { cond_gather_kernel<2><<<grid(m),CT,0,st>>>(keys,klo,cnt,m,B->kmer,B->ethresh,B->do_symm,B->hb,p0,p1,tiles,ck,cl,cc,T,B->ctr);
      LAUNCHED("cond_gather_kernel");
      cond_scan_kernel<<<1,1024,0,st>>>(tiles,grid(m),B->ctr);
      cond_orig_kernel<2><<<grid(m),CT,0,st>>>(keys,klo,cnt,m,B->ethresh,B->hb,p0,p1,tiles,B->key,B->lo,B->cnt,T,B->ctr);
    }
  else
    { cond_gather_kernel<1><<<grid(m),CT,0,st>>>(keys,klo,cnt,m,B->kmer,B->ethresh,B->do_symm,B->hb,p0,p1,tiles,ck,cl,cc,T,B->ctr);
      LAUNCHED("cond_gather_kernel");
      cond_scan_kernel<<<1,1024,0,st>>>(tiles,grid(m),B->ctr);
      cond_orig_kernel<1><<<grid(m),CT,0,st>>>(keys,klo,cnt,m,B->ethresh,B->hb,p0,p1,tiles,B->key,B->lo,B->cnt,T,B->ctr);
    }
  LAUNCHED("cond_orig_kernel");
  return HM_OK;
}

template <typename K, typename V>
static int sort_db(cub::DoubleBuffer<K> &k, cub::DoubleBuffer<V> &v, int64_t n, int bb, const hm_cond_bufs *B,
                   cudaStream_t st)
{ size_t need = 0;
  HM_CUDA(cub::DeviceRadixSort::SortPairs(NULL,need,k,v,n,bb,64,st));
  if ((int64_t) need > B->sort_bytes)
    return hm_set_error(HM_ECUDA,"the radix sort of %lld reverse complements asks for %lld scratch bytes, %lld planned",
                        (long long) n,(long long) need,(long long) B->sort_bytes);
  HM_CUDA(cub::DeviceRadixSort::SortPairs(B->sort_tmp,need,k,v,n,bb,64,st));
  return HM_OK;
}

/* the region's c reverse complements (at its end) sorted; *k / *l / *c: where they are now */
static int sort_rc(const hm_cond_bufs *B, int64_t c, uint64_t **pk, uint64_t **pl, uint16_t **pc, cudaStream_t st)
{ const int64_t T = B->cap;
  uint64_t *k0 = B->key+T-c, *l0 = B->lo ? B->lo+T-c : NULL;
  uint16_t *c0 = B->cnt+T-c;
  int rc;
  if (B->kmer <= 32)
    { cub::DoubleBuffer<uint64_t> k(k0,B->alt_key);
      cub::DoubleBuffer<uint16_t> v(c0,B->alt_cnt);
      if ((rc = sort_db(k,v,c,B->kmer < 32 ? 64-2*B->kmer : 0,B,st)) != HM_OK) return rc;
      *pk = k.Current(); *pl = NULL; *pc = v.Current();
      return HM_OK;
    }
  /* two words: by the second word with a permutation riding along, the first words and counts gathered in that
   * order, then (stable) by the first word; the second words and counts follow the final permutation         */
  cond_iota_kernel<<<grid(c),CT,0,st>>>(B->idx[0],c);
  cub::DoubleBuffer<uint64_t> l(l0,B->alt_lo);
  cub::DoubleBuffer<uint32_t> p(B->idx[0],B->idx[1]);
  if ((rc = sort_db(l,p,c,B->kmer < 64 ? 128-2*B->kmer : 0,B,st)) != HM_OK) return rc;
  cond_permute_kernel<uint64_t><<<grid(c),CT,0,st>>>(k0,p.Current(),c,B->alt_key);
  cond_permute_kernel<uint16_t><<<grid(c),CT,0,st>>>(c0,p.Current(),c,B->alt_cnt);
  cond_iota_kernel<<<grid(c),CT,0,st>>>(p.Alternate(),c);
  cub::DoubleBuffer<uint64_t> h(B->alt_key,k0);
  cub::DoubleBuffer<uint32_t> q(p.Alternate(),p.Current());
  if ((rc = sort_db(h,q,c,0,B,st)) != HM_OK) return rc;
  cond_permute_kernel<uint64_t><<<grid(c),CT,0,st>>>(l.Current(),q.Current(),c,l.Alternate());
  cond_permute_kernel<uint16_t><<<grid(c),CT,0,st>>>(B->alt_cnt,q.Current(),c,c0);
  LAUNCHED("cond_permute_kernel");
  *pk = h.Current(); *pl = l.Alternate(); *pc = c0;
  return HM_OK;
}

template <int KW>
static int merge_ranked(const hm_cond_bufs *B, int64_t o, const uint64_t *rk, const uint64_t *rl, const uint16_t *rc_,
                        int64_t c, cudaStream_t st)
{ unsigned long long *to = B->mtiles, *tc = B->mtiles + (B->cap/CT+2);
  cond_dup_kernel<KW><<<grid(o),CT,0,st>>>(B->key,B->lo,o,rk,rl,c,to);
  cond_dup_kernel<KW><<<grid(c),CT,0,st>>>(rk,rl,c,B->key,B->lo,o,tc);
  HM_CUDA(cudaMemsetAsync(B->ctr+4,0,2*sizeof(unsigned long long),st));
  cond_scan_kernel<<<1,1024,0,st>>>(to,grid(o),B->ctr+4);
  cond_scan_kernel<<<1,1024,0,st>>>(tc,grid(c),B->ctr+5);
  cond_merge_kernel<KW><<<grid(o),CT,0,st>>>(B->key,B->lo,B->cnt,o,rk,rl,c,to,0,B->m_key,B->m_lo,B->m_cnt);
  cond_merge_kernel<KW><<<grid(c),CT,0,st>>>(rk,rl,rc_,c,B->key,B->lo,o,tc,1,B->m_key,B->m_lo,B->m_cnt);
  LAUNCHED("cond_merge_kernel");
  return HM_OK;
}

int hm_cond_scan_tiles(unsigned long long *tiles, int64_t nt, unsigned long long *base, cudaStream_t st)
{ cond_scan_kernel<<<1,1024,0,st>>>(tiles,nt,base);
  LAUNCHED("cond_scan_kernel");
  return HM_OK;
}

int hm_cond_settle(const hm_cond_bufs *B, int64_t *n_out, cudaStream_t st)
{ unsigned long long h[6];
  HM_CUDA(cudaMemcpyAsync(h,B->ctr,sizeof(h),cudaMemcpyDeviceToHost,st));
  HM_CUDA(cudaStreamSynchronize(st));
  if (h[3] != 0)
    return hm_set_error(HM_ECUDA,"conditioning: a range outgrew its planned %lld entries",(long long) B->cap);
  const int64_t o = (int64_t) h[0], c = (int64_t) h[1];
  if (o+c > B->cap)
    return hm_set_error(HM_ECUDA,"conditioning: a range of %lld entries outgrew its planned %lld",(long long) (o+c),
                        (long long) B->cap);
  *n_out = o;
  if (B->m_key == NULL)                                    /* trimming only: the originals are the range */
    return HM_OK;
  if (c == 0)
    { if (o > 0)
        { HM_CUDA(cudaMemcpyAsync(B->m_key,B->key,8*(size_t) o,cudaMemcpyDeviceToDevice,st));
          if (B->lo != NULL) HM_CUDA(cudaMemcpyAsync(B->m_lo,B->lo,8*(size_t) o,cudaMemcpyDeviceToDevice,st));
          HM_CUDA(cudaMemcpyAsync(B->m_cnt,B->cnt,2*(size_t) o,cudaMemcpyDeviceToDevice,st));
        }
      HM_CUDA(cudaStreamSynchronize(st));
      return HM_OK;
    }
  uint64_t *rk = NULL, *rl = NULL;
  uint16_t *rc_ = NULL;
  int rc = sort_rc(B,c,&rk,&rl,&rc_,st);
  if (rc == HM_OK)
    rc = B->kmer > 32 ? merge_ranked<2>(B,o,rk,rl,rc_,c,st) : merge_ranked<1>(B,o,rk,rl,rc_,c,st);
  if (rc != HM_OK) return rc;
  HM_CUDA(cudaMemcpyAsync(h+4,B->ctr+4,2*sizeof(unsigned long long),cudaMemcpyDeviceToHost,st));
  HM_CUDA(cudaStreamSynchronize(st));
  *n_out = o + c - (int64_t) h[5];                         /* the reverse complements equal to an original go */
  return HM_OK;
}

int hm_cond_pack(const hm_cond_bufs *B, int64_t n, uint64_t b0, int64_t nb, cudaStream_t st)
{ const uint64_t *k = B->m_key ? B->m_key : B->key, *l = B->m_key ? B->m_lo : B->lo;
  const uint16_t *cn = B->m_key ? B->m_cnt : B->cnt;
  HM_CUDA(cudaMemsetAsync(B->bcount,0,8*(size_t) (nb > 0 ? nb : 1),st));
  const int kbyte = (B->kmer+3)>>2;
  if (n > 0)
    { if (B->kmer > 32) cond_pack_kernel<2><<<grid(n),CT,0,st>>>(k,l,cn,n,B->ibyte,kbyte,b0,B->rec,B->bcount);
      else              cond_pack_kernel<1><<<grid(n),CT,0,st>>>(k,l,cn,n,B->ibyte,kbyte,b0,B->rec,B->bcount);
      LAUNCHED("cond_pack_kernel");
    }
  HM_CUDA(cudaStreamSynchronize(st));
  return HM_OK;
}

/* ---- sorting the streamed scan's S list ------------------------------------------------------------- */

/* scratch of hm_sort_keys for up to n keys: the other buffers of the radix sort + CUB's temporary storage */
int64_t hm_sort_keys_bytes(int64_t n, int kmer)
{ size_t need = 0;
  if (n < 1) n = 1;
  if (kmer <= 32)
    cub::DeviceRadixSort::SortKeys(NULL,need,(const uint64_t *) NULL,(uint64_t *) NULL,n,0,64);
  else
    cub::DeviceRadixSort::SortPairs(NULL,need,(const uint64_t *) NULL,(uint64_t *) NULL,(const uint64_t *) NULL,
                                    (uint64_t *) NULL,n,0,64);
  return ((8*n+255) & ~255ll)*(kmer > 32 ? 2 : 1) + (int64_t) need + 256;
}

/* Sort n packed keys in place, in the caller's scratch (hm_sort_keys_bytes), enqueued on st: one radix sort
 * for one-word keys; for two-word keys the least significant word first, then a stable sort on the most
 * significant word (the other word riding along as the value).                                          */
int hm_sort_keys(uint64_t *keys, uint64_t *lo, int64_t n, int kmer, void *scratch, int64_t scratch_bytes,
                 cudaStream_t st)
{ if (n <= 1)
    return HM_OK;
  if (scratch_bytes < hm_sort_keys_bytes(n,kmer))
    return hm_set_error(HM_EINVAL,"hm_sort_keys: %lld bytes of scratch for %lld keys",(long long) scratch_bytes,(long long) n);
  uint8_t  *b   = (uint8_t *) scratch;
  int64_t   arr = (8*n+255) & ~255ll;
  uint64_t *k2  = (uint64_t *) b;
  uint64_t *l2  = (uint64_t *) (b + arr);
  void     *tmp = b + arr*(kmer > 32 ? 2 : 1);
  size_t    tb  = (size_t) (scratch_bytes - arr*(kmer > 32 ? 2 : 1));
  if (kmer <= 32)
    { int bb = kmer < 32 ? 64-2*kmer : 0;
      HM_CUDA(cub::DeviceRadixSort::SortKeys(tmp,tb,keys,k2,n,bb,64,st));
      HM_CUDA(cudaMemcpyAsync(keys,k2,sizeof(uint64_t)*(size_t) n,cudaMemcpyDeviceToDevice,st));
    }
  else
    { int bb = kmer < 64 ? 128-2*kmer : 0;
      HM_CUDA(cub::DeviceRadixSort::SortPairs(tmp,tb,lo,l2,keys,k2,n,bb,64,st));     /* by the second word */
      HM_CUDA(cub::DeviceRadixSort::SortPairs(tmp,tb,k2,keys,l2,lo,n,0,64,st));      /* stable, by the first */
    }
  return HM_OK;
}

/* CUB's temporary storage for hm_sort_perm of up to n keys */
int64_t hm_sort_perm_bytes(int64_t n)
{ size_t need = 0;
  if (n < 1) n = 1;
  cub::DeviceRadixSort::SortPairs(NULL,need,(const uint64_t *) NULL,(uint64_t *) NULL,(const uint32_t *) NULL,
                                  (uint32_t *) NULL,n,0,64);
  return (int64_t) need + 256;
}

/* one stable radix sort of n keys k_in -> k_out carrying v_in -> v_out, enqueued on st */
int hm_sort_perm(const uint64_t *k_in, uint64_t *k_out, const uint32_t *v_in, uint32_t *v_out, int64_t n,
                 void *tmp, int64_t tmp_bytes, cudaStream_t st)
{ size_t tb = (size_t) tmp_bytes;
  if (tmp_bytes < hm_sort_perm_bytes(n))
    return hm_set_error(HM_EINVAL,"hm_sort_perm: %lld bytes of scratch for %lld keys",(long long) tmp_bytes,(long long) n);
  HM_CUDA(cub::DeviceRadixSort::SortPairs(tmp,tb,k_in,k_out,v_in,v_out,n,0,64,st));
  return HM_OK;
}

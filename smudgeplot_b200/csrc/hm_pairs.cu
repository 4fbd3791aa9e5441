/*******************************************************************************************
 * hm_pairs.cu -- the file phase of extract_kmer_pairs' output in a one-process-per-GPU job (dist.ShardedScan /
 * StreamedShardedScan.write_pairs, DESIGN.md §6b).  The pair records of the job are cut by key prefix into
 * contiguous windows; the owner of a window sorts its records into hm_scan_extract's order and formats their
 * print_het lines, so that every smudge file is the concatenation, window by window, of each window's lines for
 * that smudge, at offsets that follow from the per-window line counts alone.
 *
 *   hm_k_pairs_hist            records per key prefix (the top hb bits of key_hi, hb = min(HM_COND_HIST_BITS, 2k))
 *   pairs_route_kernel<false>  per destination rank: the records of this pass's windows (dest[prefix] >= 0)
 *   pairs_route_kernel<true>   those records scattered into per-destination segments (any order inside one)
 *   hm_k_pairs_sort            CUB DeviceRadixSort over (smudge, key_hi, key_lo, pos, alt): rec_cmp's order
 *   label_bounds_kernel        lines per smudge of a sorted window
 *   format_kernel              the window's lines, staged per tile in shared memory, stored as aligned words
 * The collectives between the calls are the caller's.
 *******************************************************************************************/
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include <cub/device/device_radix_sort.cuh>
#include <cuda/std/tuple>

#include "hetmers_b200.h"
#include "hm_internal.h"
#include "hm_device.cuh"

#define LAUNCHED(what) do { cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return hm_cuda_fail(_e,what); } while (0)

static int hist_bits_of(int kmer) { return 2*kmer < HM_COND_HIST_BITS ? 2*kmer : HM_COND_HIST_BITS; }

static int64_t a512(int64_t b) { return (b+511) & ~511ll; }

__global__ void __launch_bounds__(CT)
pairs_hist_kernel(const hm_pair_rec *__restrict__ rec, int64_t n, int hb, unsigned long long *__restrict__ hist)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  const bool    in = i < n;
  warp_count(hist,in,in ? rec[i].key_hi >> (64-hb) : 0ull);
}

/* SCATTER = false: counts[d] += the records bound for rank d.  SCATTER = true: each CTA reserves its records'
 * slots in every destination's segment with one atomic per destination (cursor[d]: the next free slot, preset by
 * the caller to segment starts), then places them; *flag is set when a slot lies at or beyond `cap`.  The block's
 * per-destination counters live in dynamic shared memory (2 * world ints).                                    */
template <bool SCATTER>
__global__ void __launch_bounds__(CT)
pairs_route_kernel(const hm_pair_rec *__restrict__ rec, int64_t n, int hb, const int16_t *__restrict__ dest, int world,
                   unsigned long long *__restrict__ counts, hm_pair_rec *__restrict__ out, int64_t cap,
                   unsigned long long *__restrict__ flag)
{ extern __shared__ int s_cnt[];                         /* [world] counts, then [world] base offsets (as ints) */
  __shared__ unsigned long long s_base[64];
  const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  for (int d = threadIdx.x; d < world; d += CT) s_cnt[d] = 0;
  __syncthreads();
  hm_pair_rec r;
  int d = -1, slot = 0;
  if (i < n)
    { r = rec[i];
      d = dest[r.key_hi >> (64-hb)];
      if (d >= 0) slot = atomicAdd(&s_cnt[d],1);
    }
  __syncthreads();
  if (!SCATTER)
    { for (int q = threadIdx.x; q < world; q += CT)
        if (s_cnt[q]) atomicAdd(counts+q,(unsigned long long) s_cnt[q]);
      return;
    }
  for (int q = threadIdx.x; q < world; q += CT)
    s_base[q] = s_cnt[q] ? atomicAdd(counts+q,(unsigned long long) s_cnt[q]) : 0ull;
  __syncthreads();
  if (d >= 0)
    { const unsigned long long g = s_base[d] + (unsigned long long) slot;
      if (g < (unsigned long long) cap)
        out[g] = r;
      else
        atomicOr(flag,1ull);
    }
}

extern "C" int hm_k_pairs_hist(const hm_pair_rec *d_rec, int64_t n, int kmer, uint64_t *d_hist, void *stream)
{ if (kmer < 1 || kmer > HM_MAX_KMER || n < 0 || (n > 0 && (d_rec == NULL || d_hist == NULL)))
    return hm_set_error(HM_EINVAL,"hm_k_pairs_hist: bad arguments");
  if (n == 0)
    return HM_OK;
  pairs_hist_kernel<<<grid(n),CT,0,(cudaStream_t) stream>>>(d_rec,n,hist_bits_of(kmer),(unsigned long long *) d_hist);
  LAUNCHED("pairs_hist_kernel");
  return HM_OK;
}

static int route_args(const hm_pair_rec *d_rec, int64_t n, int kmer, const int16_t *d_dest, int world, uint64_t *d_c)
{ return kmer < 1 || kmer > HM_MAX_KMER || n < 0 || world < 1 || world > 64 ||
         (n > 0 && (d_rec == NULL || d_dest == NULL || d_c == NULL));
}

extern "C" int hm_k_pairs_route_count(const hm_pair_rec *d_rec, int64_t n, int kmer, const int16_t *d_dest, int world,
                                      uint64_t *d_counts, void *stream)
{ if (route_args(d_rec,n,kmer,d_dest,world,d_counts))
    return hm_set_error(HM_EINVAL,"hm_k_pairs_route_count: bad arguments");
  if (n == 0)
    return HM_OK;
  pairs_route_kernel<false><<<grid(n),CT,2*world*sizeof(int),(cudaStream_t) stream>>>(
      d_rec,n,hist_bits_of(kmer),d_dest,world,(unsigned long long *) d_counts,NULL,0,NULL);
  LAUNCHED("pairs_route_kernel<count>");
  return HM_OK;
}

extern "C" int hm_k_pairs_route_scatter(const hm_pair_rec *d_rec, int64_t n, int kmer, const int16_t *d_dest,
                                        int world, uint64_t *d_cursor, hm_pair_rec *d_send, int64_t cap,
                                        uint64_t *d_flag, void *stream)
{ if (route_args(d_rec,n,kmer,d_dest,world,d_cursor) || cap < 0 || (n > 0 && (d_flag == NULL || (cap > 0 && d_send == NULL))))
    return hm_set_error(HM_EINVAL,"hm_k_pairs_route_scatter: bad arguments");
  if (n == 0)
    return HM_OK;
  pairs_route_kernel<true><<<grid(n),CT,2*world*sizeof(int),(cudaStream_t) stream>>>(
      d_rec,n,hist_bits_of(kmer),d_dest,world,(unsigned long long *) d_cursor,d_send,cap,
      (unsigned long long *) d_flag);
  LAUNCHED("pairs_route_kernel<scatter>");
  return HM_OK;
}

/* rec_cmp's fields, most significant first (pad is carried along, never compared) */
struct pair_decomposer
{ __host__ __device__ ::cuda::std::tuple<uint32_t &, uint64_t &, uint64_t &, uint8_t &, uint8_t &>
  operator()(hm_pair_rec &r) const
  { return ::cuda::std::tuple<uint32_t &, uint64_t &, uint64_t &, uint8_t &, uint8_t &>(r.smudge,r.key_hi,r.key_lo,
                                                                                        r.pos,r.alt); }
};

static size_t sort_scratch(int64_t n, cudaStream_t st, int *rc)
{ size_t bytes = 0;
  cub::DoubleBuffer<hm_pair_rec> db(NULL,NULL);
  cudaError_t e = cub::DeviceRadixSort::SortKeys(NULL,bytes,db,n,pair_decomposer{},st);
  *rc = e == cudaSuccess ? HM_OK : hm_cuda_fail(e,"cub::DeviceRadixSort::SortKeys (size query)");
  return bytes;
}

/* the scratch the sort of n records asks for (0 on failure; the error is set) */
extern "C" int64_t hm_pairs_sort_scratch_bytes(int64_t n)
{ if (n < 0)
    { hm_set_error(HM_EINVAL,"hm_pairs_sort_scratch_bytes: bad arguments");
      return 0;
    }
  int rc;
  size_t b = sort_scratch(n,0,&rc);
  return rc == HM_OK ? (int64_t) b : 0;
}

/* the model's allowance for that scratch: the onesweep bins and lookback, at most a few bytes per record */
static int64_t sort_scratch_model(int64_t r) { return a512(8*r + (1ll << 20)); }

extern "C" int64_t hm_pairs_bytes(int kmer, int64_t records)
{ if (kmer < 1 || kmer > HM_MAX_KMER || records < 0)
    return -1;
  const int64_t r = records, rec = a512(24*r);
  const int64_t fixed = a512(8ll << hist_bits_of(kmer)) + a512(2ll << hist_bits_of(kmer)) + (2ll << 20);
  const int64_t route = rec + 2*a512(24*(r/2)) + 1024;
  const int64_t sort  = 2*rec + sort_scratch_model(r);
  const int64_t fmt   = rec + a512((int64_t) (kmer+5)*r);
  int64_t m = route > sort ? route : sort;
  return fixed + (m > fmt ? m : fmt);
}

int64_t hm_pairs_window_bytes(int kmer, int64_t records)
{ if (kmer < 1 || kmer > HM_MAX_KMER || records < 0)
    return -1;
  const int64_t r = records, rec = a512(24*r);
  const int64_t fixed = a512(8ll << hist_bits_of(kmer)) + a512(2ll << hist_bits_of(kmer)) + (2ll << 20);
  const int64_t sort  = 2*rec + sort_scratch_model(r);
  const int64_t fmt   = rec + a512((int64_t) (kmer+5)*r);
  return fixed + (sort > fmt ? sort : fmt);
}

/* The plan of the pair files (DESIGN.md §6b, §6c): the key prefixes cut into windows of near-equal record counts
 * on prefix boundaries -- cut r of W is the boundary nearest to r/W of the total, the lower one on a tie -- with
 * the fewest passes P such that no window of the P * world holds more than `room` records.  dist.pair_windows
 * and dist.condition_cuts are the same rule in Python; a CPU test holds the two together.                      */
static void nearest_cuts(const int64_t *before, int64_t np, int64_t W, int64_t *cuts)
{ const int64_t total = before[np];
  cuts[0] = 0;
  for (int64_t r = 1; r < W; r++)
    { const int64_t want = (int64_t) (((__int128) total * r) / W);
      int64_t lo = 0, hi = np;                                  /* the largest p with before[p] <= want */
      while (lo < hi)
        { const int64_t m = (lo+hi+1) >> 1;
          if (before[m] <= want) lo = m; else hi = m-1;
        }
      int64_t p = lo;
      if (p < np && before[p+1] - want < want - before[p])
        p += 1;
      cuts[r] = p > cuts[r-1] ? p : cuts[r-1];
    }
  cuts[W] = np;
}

extern "C" int hm_pair_windows(const int64_t *hist, int64_t np, int world, int64_t room, int64_t *passes,
                               int64_t *cuts)
{ if (hist == NULL || np < 1 || world < 1 || passes == NULL)
    return hm_set_error(HM_EINVAL,"hm_pair_windows: bad arguments");
  int64_t *before = (int64_t *) malloc(sizeof(int64_t)*(size_t) (np+1));
  if (before == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory");
  int64_t big = 0, at = 0;
  before[0] = 0;
  for (int64_t p = 0; p < np; p++)
    { if (hist[p] > big) { big = hist[p]; at = p; }
      before[p+1] = before[p] + hist[p];
    }
  if (big > room)
    { free(before);
      return hm_set_error(HM_ENOMEM,"writing the pair files: key prefix %lld holds %lld records, beyond the %lld "
                          "records one window has room for",(long long) at,(long long) big,(long long) room);
    }
  const int64_t total = before[np], per = (room > 1 ? room : 1) * (int64_t) world;
  int64_t P = (total + per - 1) / per;
  if (P < 1) P = 1;
  int64_t *c = NULL;
  for (;; P++)                                 /* ends: with a window per record every window fits */
    { int64_t *c2 = (int64_t *) realloc(c,sizeof(int64_t)*(size_t) (P*world+1));
      if (c2 == NULL)
        { free(c); free(before); return hm_set_error(HM_ENOMEM,"out of host memory"); }
      c = c2;
      nearest_cuts(before,np,P*world,c);
      int64_t most = 0;
      for (int64_t j = 0; j < P*world; j++)
        if (before[c[j+1]] - before[c[j]] > most) most = before[c[j+1]] - before[c[j]];
      if (most <= room)
        break;
    }
  *passes = P;
  if (cuts != NULL)
    memcpy(cuts,c,sizeof(int64_t)*(size_t) (P*world+1));
  free(c); free(before);
  return HM_OK;
}

extern "C" int hm_k_pairs_sort(hm_pair_rec *d_rec, hm_pair_rec *d_alt, int64_t n, void *d_scratch,
                               int64_t scratch_bytes, int *in_alt, void *stream)
{ if (n < 0 || in_alt == NULL || (n > 1 && (d_rec == NULL || d_alt == NULL || d_scratch == NULL)))
    return hm_set_error(HM_EINVAL,"hm_k_pairs_sort: bad arguments");
  *in_alt = 0;
  if (n <= 1)
    return HM_OK;
  cudaStream_t st = (cudaStream_t) stream;
  int rc;
  size_t need = sort_scratch(n,st,&rc);
  if (rc != HM_OK)
    return rc;
  if ((int64_t) need > scratch_bytes)
    return hm_set_error(HM_ENOMEM,"hm_k_pairs_sort: %lld records need %lld scratch bytes, %lld given",
                        (long long) n,(long long) need,(long long) scratch_bytes);
  cub::DoubleBuffer<hm_pair_rec> db(d_rec,d_alt);
  size_t bytes = (size_t) scratch_bytes;
  cudaError_t e = cub::DeviceRadixSort::SortKeys(d_scratch,bytes,db,n,pair_decomposer{},st);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"cub::DeviceRadixSort::SortKeys");
  *in_alt = db.Current() == d_alt;
  return HM_OK;
}

/* bounds[2s], bounds[2s+1]: first and one-past-last index of smudge s in a sorted window (both 0 if absent) */
__global__ void __launch_bounds__(CT)
label_bounds_kernel(const hm_pair_rec *__restrict__ rec, int64_t n, int n_labels, unsigned long long *__restrict__ bounds)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  if (i >= n)
    return;
  const uint32_t s = rec[i].smudge;
  if (s > (uint32_t) n_labels)
    return;
  if (i == 0 || rec[i-1].smudge != s)     bounds[2*s]   = (unsigned long long) i;
  if (i == n-1 || rec[i+1].smudge != s)   bounds[2*s+1] = (unsigned long long) i+1;
}

extern "C" int hm_k_pairs_label_bounds(const hm_pair_rec *d_sorted, int64_t n, int n_labels, uint64_t *d_bounds,
                                       void *stream)
{ if (n < 0 || n_labels < 0 || (n > 0 && (d_sorted == NULL || d_bounds == NULL)))
    return hm_set_error(HM_EINVAL,"hm_k_pairs_label_bounds: bad arguments");
  if (n == 0)
    return HM_OK;
  label_bounds_kernel<<<grid(n),CT,0,(cudaStream_t) stream>>>(d_sorted,n,n_labels,(unsigned long long *) d_bounds);
  LAUNCHED("label_bounds_kernel");
  return HM_OK;
}

/* print_het's line of every record (hetmers_main.c): k lower-case bases, the varying one as "(x/y)", and '\n' --
 * k + 5 bytes.  A CTA formats FT records into shared memory, then stores the tile's bytes as 4-byte words on
 * 4-byte aligned addresses (bytes only at the tile's two ends), so that a warp's stores are 128 coalesced bytes. */
static constexpr int FT = 128;

__global__ void __launch_bounds__(FT)
format_kernel(const hm_pair_rec *__restrict__ rec, int64_t n, int kmer, char *__restrict__ text)
{ __shared__ char s_txt[FT*(HM_MAX_KMER+5)];
  const int     lw = kmer + 5;
  const int64_t t0 = (int64_t) blockIdx.x*FT;
  const int     nt = (int) (n - t0 < FT ? n - t0 : FT);
  if ((int) threadIdx.x < nt)
    { const hm_pair_rec q = rec[t0+threadIdx.x];
      char *o = s_txt + threadIdx.x*lw;
      const char dna[4] = { 'a', 'c', 'g', 't' };
      for (int p = 0; p < kmer; p++)
        { const int b = (int) (((p < 32 ? q.key_hi : q.key_lo) >> (62-2*(p&31))) & 3);
          if (p == q.pos)
            { *o++ = '('; *o++ = dna[b]; *o++ = '/'; *o++ = dna[q.alt & 3]; *o++ = ')'; }
          else
            *o++ = dna[b];
        }
      *o = '\n';
    }
  __syncthreads();
  const int64_t g0 = t0*lw;
  const int     nb = nt*lw;
  const int     head = (int) ((4 - (g0 & 3)) & 3) < nb ? (int) ((4 - (g0 & 3)) & 3) : nb;
  const int     words = (nb - head) >> 2;
  if ((int) threadIdx.x < head)
    text[g0+threadIdx.x] = s_txt[threadIdx.x];
  uint32_t *tw = (uint32_t *) (text + g0 + head);
  for (int w = threadIdx.x; w < words; w += FT)
    { const char *s = s_txt + head + 4*w;
      tw[w] = (uint32_t) (uint8_t) s[0] | (uint32_t) (uint8_t) s[1] << 8 | (uint32_t) (uint8_t) s[2] << 16 |
              (uint32_t) (uint8_t) s[3] << 24;
    }
  for (int j = head + 4*words + threadIdx.x; j < nb; j += FT)
    text[g0+j] = s_txt[j];
}

extern "C" int hm_k_pairs_format(const hm_pair_rec *d_sorted, int64_t n, int kmer, char *d_text, void *stream)
{ if (kmer < 1 || kmer > HM_MAX_KMER || n < 0 || (n > 0 && (d_sorted == NULL || d_text == NULL)))
    return hm_set_error(HM_EINVAL,"hm_k_pairs_format: bad arguments");
  if (n == 0)
    return HM_OK;
  format_kernel<<<(unsigned) ((n+FT-1)/FT),FT,0,(cudaStream_t) stream>>>(d_sorted,n,kmer,d_text);
  LAUNCHED("format_kernel");
  return HM_OK;
}

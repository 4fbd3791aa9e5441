/*******************************************************************************************
 * hm_shard_condition.cu -- trim + symmetrise a FastK table across the ranks of a one-process-per-GPU job
 * (smudgeplot_b200/dist.py, ShardedScan.from_ktab(L=...); DESIGN.md §4e).  Rank r holds source ordinals
 * [n r/W, n (r+1)/W); rank d owns the output key prefixes [cut_d, cut_d+1), so the ranks' conditioned shares,
 * concatenated in rank order, are the sorted conditioned table.
 *
 *   hm_k_cond_hist              hm_cond_hist over a share: kept originals (+ their reverse complements) per prefix
 *   route_count_kernel          per destination rank: kept originals, reverse complements; per tile: kept originals
 *   route_scatter_kernel        the share into one send buffer: the kept originals in source order (their tile
 *                               offsets), then the reverse complements in per-destination segments (warp-aggregated
 *                               cursors; any order inside a segment)
 *   hm_k_shard_settle           the received reverse complements sorted and merged with the received originals
 *                               (already sorted): hm_cond_settle, the step every conditioning driver settles with
 * Into new table files (dist.condition_ktab, §4f) the same steps run in passes, each over one window of key prefixes
 * per rank: the route kernels' WIN instantiations skip the entries outside the pass's windows, hm_k_cond_pack packs
 * the settled entries into FastK records, and hm_rank_condition_cut / _bytes plan the passes.
 * The collectives between the calls are the caller's.
 *******************************************************************************************/
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include "hetmers_b200.h"
#include "hm_internal.h"
#include "hm_device.cuh"

#define FULL 0xffffffffu

/* counts[d]: kept originals bound for rank d; counts[world+d]: reverse complements; tiles[t]: kept originals of tile t.
 * WIN (one pass of a windowed conditioning): dest[prefix] < 0 marks a prefix outside this pass; an entry there
 * is neither counted nor written, and the tile counts cover the in-window kept originals only                  */
template <int KW, bool WIN>
__global__ void __launch_bounds__(CT)
route_count_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ klo, const uint16_t *__restrict__ cnt,
                   int64_t m, int kmer, int ethresh, int do_symm, int hb, const int16_t *__restrict__ dest, int world,
                   unsigned long long *__restrict__ counts, unsigned long long *__restrict__ tiles)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  const bool    kept = i < m && cnt[i] >= ethresh;
  uint64_t x = 0, xl = 0;
  if (kept) { x = keys[i]; if (KW == 2) xl = klo[i]; }
  const int  d  = WIN && kept ? dest[x >> (64-hb)] : -1;
  const bool in = WIN ? d >= 0 : kept;
  const int n_in = __syncthreads_count(in);
  if (threadIdx.x == 0) tiles[blockIdx.x] = (unsigned long long) n_in;
  if (WIN) warp_count(counts,in,in ? d : 0);
  else     warp_count(counts,kept,kept ? dest[x >> (64-hb)] : 0);
  if (do_symm)
    { uint64_t r, rl;
      revcomp_kmer<KW>(x,xl,kmer,r,rl);
      if (WIN)
        { const int rd = kept ? dest[r >> (64-hb)] : -1;
          warp_count(counts+world,rd >= 0,rd >= 0 ? rd : 0);
        }
      else
        warp_count(counts+world,kept,kept ? dest[r >> (64-hb)] : 0);
    }
}

/* tiles: exclusive offsets of the kept originals (hm_cond_scan_tiles); cursor[d]: the next free slot of rank d's
 * reverse-complement segment, counted from s_* + n_orig; flag: set when a slot lies beyond the buffer.  WIN: as
 * route_count_kernel                                                                                            */
template <int KW, bool WIN>
__global__ void __launch_bounds__(CT)
route_scatter_kernel(const uint64_t *__restrict__ keys, const uint64_t *__restrict__ klo, const uint16_t *__restrict__ cnt,
                     int64_t m, int kmer, int ethresh, int do_symm, int hb, const int16_t *__restrict__ dest,
                     const unsigned long long *__restrict__ tiles, uint64_t *__restrict__ s_key,
                     uint64_t *__restrict__ s_lo, uint16_t *__restrict__ s_cnt, int64_t n_orig, int64_t n_rc,
                     unsigned long long *__restrict__ cursor, unsigned long long *__restrict__ flag)
{ const int64_t i = (int64_t) blockIdx.x*CT + threadIdx.x;
  const bool    kept = i < m && cnt[i] >= ethresh;
  uint64_t x = 0, xl = 0;
  uint16_t c = 0;
  if (kept) { x = keys[i]; if (KW == 2) xl = klo[i]; c = cnt[i]; }
  const bool in = WIN ? kept && dest[x >> (64-hb)] >= 0 : kept;
  const int rank = cta_rank(in);
  if (in)
    { const int64_t g = (int64_t) tiles[blockIdx.x] + rank;   /* originals keep their order: the destination is */
      if (g < n_orig)                                         /* monotone in the key, so rank d's are one slice */
        { s_key[g] = x; if (KW == 2) s_lo[g] = xl; s_cnt[g] = c; }
      else
        atomicOr(flag,1ull);
    }
  if (!do_symm)
    return;
  uint64_t r, rl;
  revcomp_kmer<KW>(x,xl,kmer,r,rl);
  const int  rd  = WIN && kept ? dest[r >> (64-hb)] : -1;
  const bool rin = WIN ? rd >= 0 : kept;
  const unsigned act = __ballot_sync(FULL,rin);
  if (rin)
    { const int      d = WIN ? rd : dest[r >> (64-hb)];
      const unsigned peers = __match_any_sync(act,d);
      const int      lane = threadIdx.x & 31, leader = __ffs(peers)-1;
      unsigned long long base = 0;
      if (lane == leader) base = atomicAdd(cursor+d,(unsigned long long) __popc(peers));
      base = __shfl_sync(peers,base,leader);
      const int64_t slot = (int64_t) base + __popc(peers & ((1u << lane)-1));
      if (slot < n_rc)
        { s_key[n_orig+slot] = r; if (KW == 2) s_lo[n_orig+slot] = rl; s_cnt[n_orig+slot] = c; }
      else
        atomicOr(flag,1ull);
    }
}

static int64_t a256(int64_t b) { return (b+255) & ~255ll; }

static int hist_bits_of(int kmer) { return 2*kmer < HM_COND_HIST_BITS ? 2*kmer : HM_COND_HIST_BITS; }

#define LAUNCHED(what) do { cudaError_t _e = cudaGetLastError(); if (_e != cudaSuccess) return hm_cuda_fail(_e,what); } while (0)

extern "C" int hm_k_cond_hist(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m,
                              int kmer, int ethresh, int do_symm, uint64_t *d_hist, void *stream)
{ if (kmer < 1 || kmer > HM_MAX_KMER || m < 0 || (m > 0 && (kmer > 32) != (d_keys_lo != NULL)))
    return hm_set_error(HM_EINVAL,"hm_k_cond_hist: bad arguments");
  return hm_cond_hist(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,hist_bits_of(kmer),
                      (unsigned long long *) d_hist,(cudaStream_t) stream);
}

template <bool WIN>
static int route_count(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m, int kmer,
                       int ethresh, int do_symm, const int16_t *d_dest, int world, uint64_t *d_counts,
                       uint64_t *d_tiles, void *stream, const char *name)
{ if (kmer < 1 || kmer > HM_MAX_KMER || m < 0 || world < 1 || (m > 0 && (kmer > 32) != (d_keys_lo != NULL)))
    return hm_set_error(HM_EINVAL,"%s: bad arguments",name);
  cudaStream_t st = (cudaStream_t) stream;
  unsigned long long *counts = (unsigned long long *) d_counts, *tiles = (unsigned long long *) d_tiles;
  const int hb = hist_bits_of(kmer);
  if (m > 0)
    { if (kmer > 32) route_count_kernel<2,WIN><<<grid(m),CT,0,st>>>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,hb,d_dest,world,counts,tiles);
      else           route_count_kernel<1,WIN><<<grid(m),CT,0,st>>>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,hb,d_dest,world,counts,tiles);
      LAUNCHED("route_count_kernel");
    }
  return hm_cond_scan_tiles(tiles,m > 0 ? grid(m) : 0,counts+2*world,st);
}

template <bool WIN>
static int route_scatter(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m, int kmer,
                         int ethresh, int do_symm, const int16_t *d_dest, const uint64_t *d_tiles, uint64_t *d_send_key,
                         uint64_t *d_send_lo, uint16_t *d_send_cnt, int64_t n_orig, int64_t n_rc, uint64_t *d_cursor,
                         uint64_t *d_flag, void *stream, const char *name)
{ if (kmer < 1 || kmer > HM_MAX_KMER || m < 0 || n_orig < 0 || n_rc < 0 || (m > 0 && (kmer > 32) != (d_keys_lo != NULL)) ||
      (n_orig+n_rc > 0 && (kmer > 32) != (d_send_lo != NULL)))
    return hm_set_error(HM_EINVAL,"%s: bad arguments",name);
  if (m == 0)
    return HM_OK;
  cudaStream_t st = (cudaStream_t) stream;
  const unsigned long long *tiles = (const unsigned long long *) d_tiles;
  unsigned long long *cur = (unsigned long long *) d_cursor, *flag = (unsigned long long *) d_flag;
  const int hb = hist_bits_of(kmer);
  if (kmer > 32)
    route_scatter_kernel<2,WIN><<<grid(m),CT,0,st>>>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,hb,d_dest,tiles,d_send_key,
                                                     d_send_lo,d_send_cnt,n_orig,n_rc,cur,flag);
  else
    route_scatter_kernel<1,WIN><<<grid(m),CT,0,st>>>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,hb,d_dest,tiles,d_send_key,
                                                     d_send_lo,d_send_cnt,n_orig,n_rc,cur,flag);
  LAUNCHED("route_scatter_kernel");
  return HM_OK;
}

extern "C" int hm_k_shard_route_count(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t m,
                                      int kmer, int ethresh, int do_symm, const int16_t *d_dest, int world,
                                      uint64_t *d_counts, uint64_t *d_tiles, void *stream)
{ return route_count<false>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,d_dest,world,d_counts,d_tiles,stream,
                            "hm_k_shard_route_count");
}

extern "C" int hm_k_shard_route_scatter(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                                        int64_t m, int kmer, int ethresh, int do_symm, const int16_t *d_dest,
                                        const uint64_t *d_tiles, uint64_t *d_send_key, uint64_t *d_send_lo,
                                        uint16_t *d_send_cnt, int64_t n_orig, int64_t n_rc, uint64_t *d_cursor,
                                        uint64_t *d_flag, void *stream)
{ return route_scatter<false>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,d_dest,d_tiles,d_send_key,d_send_lo,d_send_cnt,
                              n_orig,n_rc,d_cursor,d_flag,stream,"hm_k_shard_route_scatter");
}

extern "C" int hm_k_shard_route_count_window(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                                             int64_t m, int kmer, int ethresh, int do_symm, const int16_t *d_dest,
                                             int world, uint64_t *d_counts, uint64_t *d_tiles, void *stream)
{ return route_count<true>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,d_dest,world,d_counts,d_tiles,stream,
                           "hm_k_shard_route_count_window");
}

extern "C" int hm_k_shard_route_scatter_window(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                                               int64_t m, int kmer, int ethresh, int do_symm, const int16_t *d_dest,
                                               const uint64_t *d_tiles, uint64_t *d_send_key, uint64_t *d_send_lo,
                                               uint16_t *d_send_cnt, int64_t n_orig, int64_t n_rc, uint64_t *d_cursor,
                                               uint64_t *d_flag, void *stream)
{ return route_scatter<true>(d_keys,d_keys_lo,d_cnt,m,kmer,ethresh,do_symm,d_dest,d_tiles,d_send_key,d_send_lo,d_send_cnt,
                             n_orig,n_rc,d_cursor,d_flag,stream,"hm_k_shard_route_scatter_window");
}

extern "C" int hm_k_cond_pack(int kmer, int ibyte, const uint64_t *d_keys, const uint64_t *d_keys_lo,
                              const uint16_t *d_cnt, int64_t n, int64_t b0, int64_t nb, uint8_t *d_rec,
                              uint64_t *d_bcount, void *stream)
{ if (kmer < 1 || kmer > HM_MAX_KMER || ibyte < 1 || ibyte > 3 || (kmer+3)/4 < ibyte || n < 0 || b0 < 0 || nb < 1 ||
      b0+nb > (1ll << (8*ibyte)) || d_bcount == NULL || (n > 0 && (d_rec == NULL || (kmer > 32) != (d_keys_lo != NULL))))
    return hm_set_error(HM_EINVAL,"hm_k_cond_pack: bad arguments");
  hm_cond_bufs B;
  memset(&B,0,sizeof(B));
  B.kmer = kmer; B.ibyte = ibyte;
  B.key = (uint64_t *) d_keys; B.lo = (uint64_t *) d_keys_lo; B.cnt = (uint16_t *) d_cnt;
  B.rec = d_rec; B.bcount = (unsigned long long *) d_bcount;
  return hm_cond_pack(&B,n,(uint64_t) b0,nb,(cudaStream_t) stream);
}

/* the settle's scratch for t received entries of which c are reverse complements: sort buffers (+ the permutation
 * pair of the two-word sort), the merge's tile counts and counters, CUB's sort scratch                         */
extern "C" int64_t hm_k_shard_settle_bytes(int kmer, int64_t t, int64_t c)
{ const int two = kmer > 32;
  if (t < 1) t = 1;
  if (c < 1) c = 1;
  return a256(8*c) + a256(2*c) + (two ? a256(8*c) + 2*a256(4*c) : 0) + 2*hm_cond_tiles_bytes(t) + 256 +
         hm_cond_sort_room(c);
}

extern "C" int hm_k_shard_settle(int kmer, uint64_t *d_key, uint64_t *d_lo, uint16_t *d_cnt, int64_t n_orig,
                                 int64_t n_rc, void *d_scratch, int64_t scratch_bytes, uint64_t *d_out_key,
                                 uint64_t *d_out_lo, uint16_t *d_out_cnt, int64_t *n_out, void *stream)
{ const int two = kmer > 32;
  if (kmer < 1 || kmer > HM_MAX_KMER || n_orig < 0 || n_rc < 0 || n_out == NULL ||
      (n_orig+n_rc > 0 && (two != (d_lo != NULL) || two != (d_out_lo != NULL))))
    return hm_set_error(HM_EINVAL,"hm_k_shard_settle: bad arguments");
  if (two && n_rc >= 0xFFFFFFF0ll)
    return hm_set_error(HM_EUNSUPPORTED,"sorting %lld reverse complements of k=%d needs 64-bit sort indices",
                        (long long) n_rc,kmer);
  const int64_t T = n_orig + n_rc;
  if (scratch_bytes < hm_k_shard_settle_bytes(kmer,T,n_rc))
    return hm_set_error(HM_EINVAL,"hm_k_shard_settle: %lld bytes of scratch, %lld needed",(long long) scratch_bytes,
                        (long long) hm_k_shard_settle_bytes(kmer,T,n_rc));
  cudaStream_t st = (cudaStream_t) stream;
  hm_cond_bufs B;
  memset(&B,0,sizeof(B));
  B.kmer = kmer; B.do_symm = 1; B.cap = T;
  B.key = d_key; B.lo = d_lo; B.cnt = d_cnt;
  B.m_key = d_out_key; B.m_lo = d_out_lo; B.m_cnt = d_out_cnt;
  uint8_t *p = (uint8_t *) d_scratch;
  const int64_t c = n_rc > 0 ? n_rc : 1;
  B.alt_key = (uint64_t *) p; p += a256(8*c);
  B.alt_cnt = (uint16_t *) p; p += a256(2*c);
  if (two)
    { B.alt_lo = (uint64_t *) p; p += a256(8*c);
      B.idx[0] = (uint32_t *) p; p += a256(4*c);
      B.idx[1] = (uint32_t *) p; p += a256(4*c);
    }
  B.mtiles = (unsigned long long *) p; p += 2*hm_cond_tiles_bytes(T);
  B.ctr = (unsigned long long *) p; p += 256;
  B.sort_tmp = p;
  B.sort_bytes = scratch_bytes - (int64_t) (p - (uint8_t *) d_scratch);
  /* the counters a gather would have left: originals at the region's front, reverse complements at its end */
  const unsigned long long h[4] = { (unsigned long long) n_orig, (unsigned long long) n_rc, 0, 0 };
  HM_CUDA(cudaMemcpyAsync(B.ctr,h,sizeof(h),cudaMemcpyHostToDevice,st));
  return hm_cond_settle(&B,n_out,st);
}

/* device bytes one rank's conditioning holds at most (each array rounded to 512 bytes, as torch's allocator
 * counts them); see the header                                                                              */
static int64_t a512(int64_t b) { return (b+511) & ~511ll; }

static int64_t ent(int64_t t, int two) { return a512(8*t)*(two ? 2 : 1) + a512(2*t); }

extern "C" int64_t hm_shard_condition_bytes(int kmer, int ibyte, int world, int64_t share, int64_t sent,
                                            int64_t received, int64_t rc_received, int64_t total_out, int do_symm)
{ if (kmer < 1 || kmer > HM_MAX_KMER || ibyte < 1 || ibyte > 3 || world < 1 || share < 0 || sent < 0 || received < 0 ||
      rc_received < 0 || total_out < 0)
    return -1;
  const int     two = kmer > 32;
  const int64_t np = (int64_t) 1 << hist_bits_of(kmer), pbyte = ((kmer+3)>>2) - ibyte + 2;
  const int64_t fixed = 2*a512(8*np) + a512(2*np) + a512(8*(2*world+2)) + a512(8*world) + (1ll << 20);
  const int64_t load  = ent(share,two) + a512(pbyte*share) + a512(8ll << (8*ibyte));
  const int64_t route = ent(share,two) + a512(hm_cond_tiles_bytes(share)) + ent(sent,two);
  const int64_t xchg  = ent(sent,two) + ent(received,two);
  const int64_t settle = do_symm ? 2*ent(received,two) + a512(hm_k_shard_settle_bytes(kmer,received,rc_received)) : 0;
  const int64_t gather = ent(received,two) + ent(total_out+world,two) + ent(total_out/world+1,two);
  int64_t most = load;
  if (route > most)  most = route;
  if (xchg > most)   most = xchg;
  if (settle > most) most = settle;
  if (gather > most) most = gather;
  return fixed + most;
}

/* ---- conditioning across the ranks into new table files (dist.condition_ktab, DESIGN.md §4f) ---------------
 * Memory model of one rank (arrays rounded to 512 bytes as torch's allocator rounds them; 1 MiB for small
 * tensors).  Resident for the whole call: the unpacked share (E = 10 / 18 bytes per entry at k <= 32 / > 32),
 * its tile counts, the two histograms, the destination map (int16 per prefix), the route counters and the
 * stub-bucket counts of one pass.  Beside it, at most one of: the load (the share's records and the stub index
 * on the device), or one pass -- route: the send buffer; exchange: send + receive; settle (symmetrising): the
 * received entries, the settled ones and the sort scratch; pack: the settled entries and their records.     */

static int64_t ent1(int64_t t, int two) { return ent(t > 1 ? t : 1,two); }

static int64_t rank_resident(int kmer, int ibyte, int world, int64_t share)
{ const int64_t np = (int64_t) 1 << hist_bits_of(kmer);
  return ent(share,kmer > 32) + a512(hm_cond_tiles_bytes(share)) + a512(16*np) + a512(2*np) + a512(8*(2*world+2)) +
         a512(8*world) + a512(8ll << (8*ibyte)) + (1ll << 20);
}

static int64_t rank_load(int kmer, int ibyte, int64_t share)
{ const int64_t pbyte = ((kmer+3)>>2) - ibyte + 2;
  return a512(pbyte*share) + a512(8ll << (8*ibyte));
}

static int64_t rank_pass(int kmer, int ibyte, int64_t sent, int64_t received, int64_t rc_received, int do_symm)
{ const int     two = kmer > 32;
  const int64_t pbyte = ((kmer+3)>>2) - ibyte + 2;
  const int64_t route = ent1(sent,two), xchg = ent1(sent,two) + ent1(received,two);
  const int64_t settle = do_symm ? 2*ent1(received,two) + a512(hm_k_shard_settle_bytes(kmer,received,rc_received)) : 0;
  const int64_t pack = ent1(received,two) + a512(pbyte*(received > 1 ? received : 1));
  int64_t most = route;
  if (xchg > most)   most = xchg;
  if (settle > most) most = settle;
  if (pack > most)   most = pack;
  return most;
}

extern "C" int64_t hm_rank_condition_bytes(int kmer, int ibyte, int world, int64_t share, int64_t sent,
                                           int64_t received, int64_t rc_received, int do_symm)
{ if (kmer < 1 || kmer > HM_MAX_KMER || ibyte < 1 || ibyte > 3 || world < 1 || share < 0 || sent < 0 || received < 0 ||
      rc_received < 0 || rc_received > received)
    return -1;
  const int64_t load = rank_load(kmer,ibyte,share), pass = rank_pass(kmer,ibyte,sent,received,rc_received,do_symm);
  return rank_resident(kmer,ibyte,world,share) + (load > pass ? load : pass);
}

/* a sub-range of t output entries, sized as if the rank sent and received t entries, all reverse complements */
static int64_t sub_range_bytes(int64_t t, int do_symm, int kmer, int ibyte)
{ return rank_pass(kmer,ibyte,t,t,do_symm ? t : 0,do_symm); }

extern "C" int hm_rank_condition_cut(int kmer, int ibyte, int world, int64_t share, int do_symm, int64_t budget,
                                     const int64_t *hist, int64_t np, int64_t *cuts, int64_t *n_sub)
{ if (kmer < 1 || kmer > HM_MAX_KMER || ibyte < 1 || ibyte > 3 || world < 1 || share < 0 || np < 0 ||
      (np > 0 && hist == NULL) || cuts == NULL || n_sub == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_condition_cut: bad arguments");
  *n_sub = 0;
  const int64_t resident = rank_resident(kmer,ibyte,world,share), load = rank_load(kmer,ibyte,share);
  const int64_t room = budget - resident;
  const int64_t limit = room > 0 ? hm_cond_range_limit(room,sub_range_bytes,do_symm,kmer,ibyte) : 0;
  int64_t cap = 0, big = 0;
  int r = 0;
  if (np > 0)
    r = hm_cond_cut(hist,np,limit,cuts,&cap,&big);
  else
    cuts[0] = 0;                                           /* an empty range: no sub-range */
  if ((np > 0 && r < 1) || load > room)
    return hm_set_error(HM_ENOMEM,"conditioning into files on a rank with a budget of %lld device bytes: its share of "
                        "%lld source entries holds %lld bytes resident and %lld more while it loads, and its largest "
                        "key prefix of %lld output entries needs %lld more in one pass; use more ranks, or "
                        "condition_kmer_table",(long long) budget,(long long) share,(long long) resident,
                        (long long) load,(long long) big,(long long) sub_range_bytes(big,do_symm,kmer,ibyte));
  *n_sub = r;
  return HM_OK;
}

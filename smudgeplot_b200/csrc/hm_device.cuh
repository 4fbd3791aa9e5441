/* hm_device.cuh -- device helpers shared by the kernel translation units (not installed) */
#ifndef HM_DEVICE_CUH
#define HM_DEVICE_CUH

#include <cuda_runtime.h>
#include <stdint.h>

template <typename IdxT> struct IdxNone { static constexpr IdxT value = (IdxT) ~(IdxT) 0; };

/* exact match of y inside its prefix bucket; -1 if absent.  KW = 64-bit words per key (k <= 32: 1,
 * k <= 64: 2, second word in the parallel array keys_lo); buckets are prefixes of the first word. */
template <typename IdxT, int KW>
__device__ __forceinline__ int64_t bucket_find(const uint64_t *__restrict__ keys,
                                               const uint64_t *__restrict__ keys_lo,
                                               const IdxT *__restrict__ bucket,
                                               int bshift, uint64_t y, uint64_t ylo)
{ uint64_t bk = y >> bshift;
  IdxT l = bucket[bk];
  IdxT r = bucket[bk+1];
  while (l < r)
    { IdxT     m = l + ((r-l)>>1);
      uint64_t v = __ldg(keys+m);
      if (KW == 1)
        { if (v == y)
            return (int64_t) m;
          if (v < y) l = m+1; else r = m;
        }
      else
        { if (v == y)
            { uint64_t w = __ldg(keys_lo+m);
              if (w == ylo)
                return (int64_t) m;
              if (w < ylo) l = m+1; else r = m;
            }
          else if (v < y) l = m+1; else r = m;
        }
    }
  return -1;
}

/* ---- mbarrier + TMA bulk copy (cp.async.bulk global -> shared; SASS: UBLKCP / SYNCS) ---- */

__device__ __forceinline__ uint32_t smem_u32(const void *p)
{ return (uint32_t) __cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count)
{ asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory"); }

__device__ __forceinline__ void fence_proxy_async_smem(void)
{ asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

__device__ __forceinline__ void mbar_arrive_expect_tx(uint64_t *bar, unsigned bytes)
{ asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;"
               :: "r"(smem_u32(bar)), "r"(bytes) : "memory"); }

__device__ __forceinline__ void bulk_copy_g2s(void *dst, const void *src, unsigned bytes, uint64_t *bar)
{ asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(__cvta_generic_to_global(src)), "r"(bytes), "r"(smem_u32(bar))
               : "memory"); }

__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity)
{ unsigned ok;
  do
    asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                 : "=r"(ok) : "r"(smem_u32(bar)), "r"(parity) : "memory");
  while (!ok);
}

/* ---- one thread per entry, CT entries per CTA (the conditioning kernels) ---- */

static constexpr int CT = 256;

static inline unsigned grid(int64_t n) { return (unsigned) ((n+CT-1)/CT > 0 ? (n+CT-1)/CT : 1); }

/* hist[key] += 1 for every lane with pred (lanes of a warp that share a key add once) */
template <typename K>
__device__ __forceinline__ void warp_count(unsigned long long *hist, bool pred, K key)
{ const unsigned act = __ballot_sync(0xffffffffu,pred);
  if (pred)
    { const unsigned peers = __match_any_sync(act,key);
      if ((threadIdx.x & 31) == (unsigned) (__ffs(peers)-1))
        atomicAdd(hist+key,(unsigned long long) __popc(peers));
    }
}

/* exclusive rank of this thread's pred among the CTA's (once per kernel: the shared counts are not reset) */
__device__ __forceinline__ int cta_rank(bool pred)
{ __shared__ int s_w[CT/32];
  const int      lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned b = __ballot_sync(0xffffffffu,pred);
  if (lane == 0) s_w[warp] = __popc(b);
  __syncthreads();
  int before = 0;
  for (int w = 0; w < warp; w++) before += s_w[w];
  return before + __popc(b & ((1u << lane)-1));
}

/* ---- packed k-mers: left aligned, base i in bits 63-2i..62-2i of word i/32 ---- */

#define HM_M5 0x5555555555555555ull

/* reverse complement of all 32 slots of one word */
__device__ __forceinline__ uint64_t revcomp_word(uint64_t x)
{ uint64_t r = __brevll(~x);                               /* slots reversed, bits inside a slot swapped */
  return ((r >> 1) & HM_M5) | ((r & HM_M5) << 1);
}

/* reverse complement of a left-aligned k-mer; KW = 1: k <= 32 (lo ignored), KW = 2: 32 < k <= 64 */
template <int KW>
__device__ __forceinline__ void revcomp_kmer(uint64_t hi, uint64_t lo, int k, uint64_t &rhi, uint64_t &rlo)
{ if (KW == 1)
    { uint64_t r = revcomp_word(hi);                       /* rc right aligned, complemented pad on top */
      rhi = (k < 32) ? (r << (64-2*k)) : r;
      rlo = 0;
    }
  else
    { uint64_t a = revcomp_word(lo), b = revcomp_word(hi);
      int      sh = 2*(64-k);
      if (sh == 0) { rhi = a; rlo = b; }
      else         { rhi = (a << sh) | (b >> (64-sh)); rlo = b << sh; }
    }
}

/* do x and z (distinct keys) differ in exactly one base?  pos = that base */
template <int KW>
__device__ __forceinline__ bool one_base_apart(uint64_t x, uint64_t xl, uint64_t z, uint64_t zl, int &pos)
{ uint64_t d = x ^ z;
  uint64_t u = (d | (d>>1)) & HM_M5;
  if (KW == 1)
    { pos = __clzll((long long) d) >> 1;
      return ((u & (u-1)) == 0);
    }
  uint64_t dl = xl ^ zl;
  uint64_t ul = (dl | (dl>>1)) & HM_M5;
  pos = (d != 0) ? (__clzll((long long) d) >> 1) : 32 + (__clzll((long long) dl) >> 1);
  return ((u & (u-1)) == 0) && ((ul & (ul-1)) == 0) && ((u == 0) != (ul == 0));
}

/* base (0..3) of a k-mer at position p, and the k-mer with that base replaced by c */
template <int KW>
__device__ __forceinline__ int base_at(uint64_t hi, uint64_t lo, int p)
{ return (int) (((KW == 1 || p < 32 ? hi : lo) >> (62-2*(p&31))) & 3); }

template <int KW>
__device__ __forceinline__ void set_base(uint64_t &hi, uint64_t &lo, int p, int c)
{ const int sh = 62-2*(p&31);
  if (KW == 1 || p < 32) hi = (hi & ~((uint64_t) 3 << sh)) | ((uint64_t) c << sh);
  else                   lo = (lo & ~((uint64_t) 3 << sh)) | ((uint64_t) c << sh);
}

#endif

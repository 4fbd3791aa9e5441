/*******************************************************************************************
 * hm_condition.cu -- table conditioning on the GPU: the two things the reference delegates to
 * external FastK executables before it scans (PloidyPlot.c:1381-1426):
 *
 *   trim        `Logex -T<t> '<tmp>.trim=A[<L>-]' <table>`   keep entries with count >= L
 *   symmetrise  `Symmex -T<t> -P<dir> <table> <tmp>.symx`     add the reverse complement of every
 *                                                             k-mer (same count), keep the table sorted
 *
 * FastK's tools are not part of the reference tree and are not pinned to a version (SURVEY.md
 * §8c), so this restates their documented effect, not their code: parity for THIS step is pinned
 * only against a numpy restatement in tests/ ("parity unpinned" against the real tools).  The
 * executable uses it by default and falls back to the reference's shell-outs with
 * HETMERS_EXTERNAL_CONDITIONING=1.
 *
 * Not a hot path (it runs once, before the scan): selection and sorting use CUB's device-wide
 * primitives (library code); the reverse-complement / duplicate-flag kernels are ours.
 * Duplicates (palindromes for even k, or an input that already held both strands) keep the
 * ORIGINAL entry: the concatenation puts originals first and the radix sort is stable.
 *******************************************************************************************/
#include <cub/cub.cuh>
#include <cuda_runtime.h>
#include <stdint.h>

#include "hetmers_b200.h"
#include "hm_internal.h"

__device__ __forceinline__ uint64_t rev2_64(uint64_t x)       /* reverse the 32 2-bit fields */
{ x = ((x >> 2)  & 0x3333333333333333ull) | ((x & 0x3333333333333333ull) << 2);
  x = ((x >> 4)  & 0x0F0F0F0F0F0F0F0Full) | ((x & 0x0F0F0F0F0F0F0F0Full) << 4);
  x = ((x >> 8)  & 0x00FF00FF00FF00FFull) | ((x & 0x00FF00FF00FF00FFull) << 8);
  x = ((x >> 16) & 0x0000FFFF0000FFFFull) | ((x & 0x0000FFFF0000FFFFull) << 16);
  return (x >> 32) | (x << 32);
}

__global__ void __launch_bounds__(256)
trim_flag_kernel(const uint16_t *__restrict__ cnt, int64_t n, int ethresh, uint8_t *__restrict__ flag)
{ int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    flag[i] = (cnt[i] >= ethresh);
}

/* out[0,n) = table, out[n,2n) = reverse complements with the same counts */
__global__ void __launch_bounds__(256)
append_revcomp_kernel(const uint64_t *__restrict__ hi, const uint64_t *__restrict__ lo,
                      const uint16_t *__restrict__ cnt, int64_t n, int kmer,
                      uint64_t *__restrict__ ohi, uint64_t *__restrict__ olo, uint16_t *__restrict__ ocnt)
{ int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n)
    return;
  uint64_t x = hi[i];
  uint16_t c = cnt[i];
  ohi[i] = x; ocnt[i] = c; ocnt[n+i] = c;
  if (lo == NULL)
    { uint64_t r = rev2_64(~x);
      if (kmer < 32)
        r = (r & (((uint64_t) 1 << (2*kmer))-1)) << (64-2*kmer);
      ohi[n+i] = r;
    }
  else
    { uint64_t w = lo[i];
      uint64_t a = rev2_64(~w), b = rev2_64(~x);          /* the two words swap */
      int      sh = 2*(64-kmer);
      olo[i] = w;
      if (sh == 0) { ohi[n+i] = a; olo[n+i] = b; }
      else         { ohi[n+i] = (a << sh) | (b >> (64-sh)); olo[n+i] = b << sh; }
    }
}

__global__ void __launch_bounds__(256)
iota_kernel(uint32_t *__restrict__ idx, int64_t n)
{ int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) idx[i] = (uint32_t) i;
}

template <typename T>
__global__ void __launch_bounds__(256)
gather_kernel(const T *__restrict__ src, const uint32_t *__restrict__ idx, int64_t n, T *__restrict__ dst)
{ int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] = src[idx[i]];
}

__global__ void __launch_bounds__(256)
first_of_run_kernel(const uint64_t *__restrict__ hi, const uint64_t *__restrict__ lo, int64_t n,
                    uint8_t *__restrict__ flag)
{ int64_t i = (int64_t) blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n)
    flag[i] = (i == 0) || hi[i] != hi[i-1] || (lo != NULL && lo[i] != lo[i-1]);
}

#define GRID(n) ((unsigned) (((n)+255)/256))

template <typename T>
static int select_flagged(const T *in, const uint8_t *flag, T *out, int64_t n, int64_t *d_nsel,
                          void **tmp, size_t *tmp_bytes, cudaStream_t st)
{ size_t need = 0;
  HM_CUDA(cub::DeviceSelect::Flagged(NULL,need,in,flag,out,d_nsel,n,st));
  if (need > *tmp_bytes)
    { if (*tmp) cudaFree(*tmp);
      *tmp = NULL; *tmp_bytes = 0;
      HM_CUDA(cudaMalloc(tmp,need));
      *tmp_bytes = need;
    }
  HM_CUDA(cub::DeviceSelect::Flagged(*tmp,need,in,flag,out,d_nsel,n,st));
  return HM_OK;
}

template <typename K, typename V>
static int sort_pairs(const K *kin, K *kout, const V *vin, V *vout, int64_t n, int begin_bit, int end_bit,
                      void **tmp, size_t *tmp_bytes, cudaStream_t st)
{ size_t need = 0;
  HM_CUDA(cub::DeviceRadixSort::SortPairs(NULL,need,kin,kout,vin,vout,n,begin_bit,end_bit,st));
  if (need > *tmp_bytes)
    { if (*tmp) cudaFree(*tmp);
      *tmp = NULL; *tmp_bytes = 0;
      HM_CUDA(cudaMalloc(tmp,need));
      *tmp_bytes = need;
    }
  HM_CUDA(cub::DeviceRadixSort::SortPairs(*tmp,need,kin,kout,vin,vout,n,begin_bit,end_bit,st));
  return HM_OK;
}

/* device allocations of one conditioning call: everything still registered is freed on return */
struct Scratch
  { void *p[32];
    int   n;
    Scratch() : n(0) {}
    ~Scratch() { for (int k = 0; k < n; k++) cudaFree(p[k]); }
    template <typename T> cudaError_t alloc(T **q, size_t bytes)
    { cudaError_t e = cudaMalloc((void **) q,bytes);
      if (e == cudaSuccess && n < 32) p[n++] = (void *) *q;
      return e;
    }
    void release(void *q)                      /* hand q to the caller (or it was freed by hand) */
    { for (int k = 0; k < n; k++)
        if (p[k] == q) { p[k] = p[--n]; return; }
    }
    void free_now(void *q) { if (q != NULL) { release(q); cudaFree(q); } }
  };

/* Replace (*pk, *pl, *pc, *pn) by the conditioned table: new cudaMalloc'ed arrays of *pcap entries
 * each (at least one spare: they are sized before the duplicates or the trimmed entries go).  *pl is
 * NULL for k <= 32.  The pointers are replaced only when the whole call has succeeded and produced a
 * new table; the caller's arrays are never freed here, and on any failure every temporary is
 * released.                                                                                      */
int hm_condition_arrays(int kmer, int ethresh, int do_trim, int do_symm,
                        uint64_t **pk, uint64_t **pl, uint16_t **pc, int64_t *pn, int64_t *pcap, cudaStream_t st)
{ int64_t   n = *pn;
  const int two = (*pl != NULL);
  Scratch   S;
  void     *tmp = NULL;                        /* CUB temporary storage (grown on demand) */
  size_t    tmp_bytes = 0;
  uint8_t  *flag = NULL;
  int64_t  *d_nsel = NULL, nsel = 0;
  int       rc = HM_OK;
  /* current table: the caller's arrays, or ours once a stage has produced new ones */
  uint64_t *ck = *pk, *cl = *pl;
  uint16_t *cc = *pc;
  int       own = 0;
  int64_t   cap = 0;                           /* entries each array of ours holds */

  if (do_symm && two && 2*n >= 0xFFFFFFF0ll)   /* before anything is allocated or touched */
    return hm_set_error(HM_EUNSUPPORTED,"symmetrising %lld entries of k=%d needs 64-bit sort indices",
                        (long long) n,kmer);
#define CK(call) do { cudaError_t _e = (call); if (_e != cudaSuccess) { if (tmp) cudaFree(tmp); return hm_cuda_fail(_e,#call); } } while (0)
#define RC(call) do { if ((rc = (call)) != HM_OK) { if (tmp) cudaFree(tmp); return rc; } } while (0)
  CK(S.alloc(&d_nsel,sizeof(int64_t)));

  if (do_trim && n > 0)
    { uint64_t *k2 = NULL, *l2 = NULL; uint16_t *c2 = NULL;
      CK(S.alloc(&flag,(size_t) n));
      CK(S.alloc(&k2,sizeof(uint64_t)*(size_t) (n+1)));
      CK(S.alloc(&c2,sizeof(uint16_t)*(size_t) (n+1)));
      if (two) CK(S.alloc(&l2,sizeof(uint64_t)*(size_t) (n+1)));
      trim_flag_kernel<<<GRID(n),256,0,st>>>(cc,n,ethresh,flag);
      RC(select_flagged(ck,flag,k2,n,d_nsel,&tmp,&tmp_bytes,st));
      if (two) RC(select_flagged(cl,flag,l2,n,d_nsel,&tmp,&tmp_bytes,st));
      RC(select_flagged(cc,flag,c2,n,d_nsel,&tmp,&tmp_bytes,st));
      CK(cudaMemcpyAsync(&nsel,d_nsel,sizeof(int64_t),cudaMemcpyDeviceToHost,st));
      CK(cudaStreamSynchronize(st));
      S.free_now(flag); flag = NULL;
      ck = k2; cc = c2; cl = l2; cap = n+1; n = nsel; own = 1;
    }

  if (do_symm && n > 0)
    { int64_t   m = 2*n;
      uint64_t *h0 = NULL, *l0 = NULL, *h1 = NULL, *l1 = NULL;
      uint16_t *c0 = NULL, *c1 = NULL;
      CK(S.alloc(&h0,sizeof(uint64_t)*(size_t) (m+1)));
      CK(S.alloc(&h1,sizeof(uint64_t)*(size_t) (m+1)));
      CK(S.alloc(&c0,sizeof(uint16_t)*(size_t) (m+1)));
      CK(S.alloc(&c1,sizeof(uint16_t)*(size_t) (m+1)));
      if (two)
        { CK(S.alloc(&l0,sizeof(uint64_t)*(size_t) (m+1)));
          CK(S.alloc(&l1,sizeof(uint64_t)*(size_t) (m+1)));
        }
      append_revcomp_kernel<<<GRID(n),256,0,st>>>(ck,cl,cc,n,kmer,h0,l0,c0);
      if (own)                                       /* the trimmed intermediate is ours: drop it now */
        { CK(cudaStreamSynchronize(st));
          S.free_now(ck); S.free_now(cc); S.free_now(cl);
          ck = NULL; cc = NULL; cl = NULL; own = 0;
        }
      if (!two)
        { int bb = kmer < 32 ? 64-2*kmer : 0;
          RC(sort_pairs(h0,h1,c0,c1,m,bb,64,&tmp,&tmp_bytes,st));
        }
      else
        { uint32_t *i0 = NULL, *i1 = NULL;
          CK(S.alloc(&i0,sizeof(uint32_t)*(size_t) m));
          CK(S.alloc(&i1,sizeof(uint32_t)*(size_t) m));
          iota_kernel<<<GRID(m),256,0,st>>>(i0,m);
          int bb = kmer < 64 ? 128-2*kmer : 0;
          /* least significant word first, then a stable sort on the most significant word */
          RC(sort_pairs(l0,l1,i0,i1,m,bb,64,&tmp,&tmp_bytes,st));
          gather_kernel<uint64_t><<<GRID(m),256,0,st>>>(h0,i1,m,h1);          /* hi in lo-order   */
          RC(sort_pairs(h1,l1,i1,i0,m,0,64,&tmp,&tmp_bytes,st));
          /* l1 = sorted hi, i0 = final permutation */
          gather_kernel<uint64_t><<<GRID(m),256,0,st>>>(l0,i0,m,h1);          /* h1 := lo sorted  */
          gather_kernel<uint16_t><<<GRID(m),256,0,st>>>(c0,i0,m,c1);
          /* arrange as (h1 = hi, l1 = lo) */
          uint64_t *t = h1; h1 = l1; l1 = t;
          CK(cudaStreamSynchronize(st));
          S.free_now(i0); S.free_now(i1);
        }
      /* unique (first of every run of equal keys wins) back into h0/l0/c0 */
      CK(S.alloc(&flag,(size_t) m));
      first_of_run_kernel<<<GRID(m),256,0,st>>>(h1,two ? l1 : NULL,m,flag);
      RC(select_flagged(h1,flag,h0,m,d_nsel,&tmp,&tmp_bytes,st));
      if (two) RC(select_flagged(l1,flag,l0,m,d_nsel,&tmp,&tmp_bytes,st));
      RC(select_flagged(c1,flag,c0,m,d_nsel,&tmp,&tmp_bytes,st));
      CK(cudaMemcpyAsync(&nsel,d_nsel,sizeof(int64_t),cudaMemcpyDeviceToHost,st));
      CK(cudaStreamSynchronize(st));
      ck = h0; cc = c0; cl = l0; cap = m+1; n = nsel; own = 1;
    }

  CK(cudaStreamSynchronize(st));
#undef CK
#undef RC
  if (tmp) cudaFree(tmp);
  if (own)                                           /* success: hand the new table over */
    { S.release(ck); S.release(cc); if (cl) S.release(cl);
      *pk = ck; *pc = cc; *pl = cl; *pcap = cap;
    }
  *pn = n;
  return HM_OK;
}

static int64_t sort_pairs_tmp(int64_t n)
{ size_t need = 0;
  cub::DeviceRadixSort::SortPairs(NULL,need,(const uint64_t *) NULL,(uint64_t *) NULL,(const uint64_t *) NULL,
                                  (uint64_t *) NULL,n,0,64);
  return (int64_t) need;
}

/* Device bytes a conditioning call borrows besides the caller's table of n entries: the larger of the
 * trim stage (flags + one n-entry copy) and the symmetrise stage (two 2n-entry tables, sort indices for
 * two-word keys, flags), plus CUB's temporary storage.  hm_scan_condition checks it against the budget
 * before it touches anything.                                                                        */
int64_t hm_condition_bytes(int kmer, int64_t n, int do_trim, int do_symm)
{ const int64_t ent = 8 + (kmer > 32 ? 8 : 0) + 2;
  int64_t trim = 0, symm = 0;
  if (do_trim)
    trim = n + ent*(n+1) + sort_pairs_tmp(n) + 8;
  if (do_symm)
    { int64_t m = 2*n;
      symm = 2*ent*(m+1) + m + sort_pairs_tmp(m) + 8;
      if (kmer > 32)
        symm += 2*4*m;
    }
  return trim > symm ? trim : symm;
}

/* scratch of hm_sort_keys for up to n keys: the other buffers of the radix sort + CUB's temporary storage */
int64_t hm_sort_keys_bytes(int64_t n, int kmer)
{ size_t need = 0;
  if (n < 1) n = 1;
  if (kmer <= 32)
    cub::DeviceRadixSort::SortKeys(NULL,need,(const uint64_t *) NULL,(uint64_t *) NULL,n,0,64);
  else
    need = (size_t) sort_pairs_tmp(n);
  return ((8*n+255) & ~255ll)*(kmer > 32 ? 2 : 1) + (int64_t) need + 256;
}

/* Sort n packed keys in place, in the caller's scratch (hm_sort_keys_bytes), enqueued on st: one radix sort
 * for one-word keys; for two-word keys the least significant word first, then a stable sort on the most
 * significant word (the order of hm_condition_arrays, the other word riding along as the value).       */
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

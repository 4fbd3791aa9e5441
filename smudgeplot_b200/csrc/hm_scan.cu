/*******************************************************************************************
 * hm_scan.cu -- layer B of include/hetmers_b200.h: the whole hetmers path from HOST buffers.
 *
 *   hm_scan_create   H2D of the raw FastK part payloads (double-buffered, copy stream ||
 *                    unpack stream), SoA unpack, bucket index          ("T_load", device part)
 *   hm_scan_examine  trimmed? / symmetric? decisions of examine_table (PloidyPlot.c:1167-1230)
 *   hm_scan_run      pass 1 -> (degree exchange when >1 GPU) -> pass 2 -> plot D2H  ("T_scan")
 *
 * Every device holds a full replica of the table (the symmetric scan needs ~13.4 B per k=31 entry, so
 * an 80 GB H100 holds ~6e9 entries with its work area); work is
 * sharded by contiguous index range [lo_g, hi_g).  With one GPU there is no exchange at all.
 * With several GPUs in this single process the loader gathers the shards over NVLink peer
 * copies and foreign degree bytes are reached through the owner's array (remote atomics / loads
 * fused into the two kernels; summed by a peer-memory kernel of hm_peer.cu if there are no
 * native NVLink atomics); the
 * one-process-per-GPU variant (torch.distributed / NCCL) lives in smudgeplot_b200/dist.py and
 * uses layer A directly; its streamed counterpart drives one rank's share through the hm_rank_scan_* calls
 * at the end of this file.
 * A table whose in-core footprint exceeds the device budget is not loaded here: every run streams it
 * in run-aligned chunks (run_stream, DESIGN.md §4c), through one GPU or, sharded, each GPU its own
 * run-aligned share of the table.
 *******************************************************************************************/
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>
#include <pthread.h>
#include <unistd.h>
#include <errno.h>
#include <sys/stat.h>
#include <fcntl.h>

#include "hetmers_b200.h"
#include "hm_internal.h"

#define HM_MAX_GPUS 16
#define LOAD_CHUNK  (16ll<<20)        /* records per H2D/unpack chunk */

typedef struct
  { int                 dev;
    cudaStream_t        st, st_copy;
    uint64_t           *keys;
    uint64_t           *keys_lo;      /* second key word, k > 32 only */
    uint16_t           *cnt;
    uint8_t            *deg;          /* n rounded up to 4 */
    void               *bucket;
    uint32_t           *filter;       /* prefix presence bitmap */
    void               *up;           /* hi-lo entries */
    void               *p2scratch;    /* pass 2 defer list (multi-GPU peer mode) */
    int64_t             p2scratch_bytes;
    unsigned long long *plot;
    int64_t             lo, hi;       /* this device's work range */
    void               *symm_work;    /* work area of the strand-symmetric scan (hm_symm.cu) */
    hm_symm_layout      symm_layout;
    int64_t             slo, shi;     /* its run-aligned range */
    uint64_t           *fp_acc;       /* device uint64[4]: symmetry fingerprint sums of the entries loaded here */
    cudaEvent_t         ev[4];        /* a run's pass 1 from ev[0] to ev[1], pass 2 from ev[2] to ev[3] */
    int                 pool;         /* allocations come from the device's stream-ordered pool */
    struct DevBlock    *blocks;       /* every device allocation held (dev_alloc) */
    int64_t             held, peak, chunks;   /* device bytes now / at most (streamed: since the last run began);
                                                 (streamed) chunks of the last run */
  } DevTable;

struct hm_scan
  { int      kmer, ibyte, bits, fpos, idx64, ngpu;
    int64_t  n;
    DevTable d[HM_MAX_GPUS];
    double   ms_load, ms_alloc, ms_records, ms_index;
    int      ran, peer_mode;              /* ran: the direct passes have filled deg/up (extract, download) */
    hm_shards sh[HM_MAX_GPUS];
    int64_t  launches;
    int      symmetric;                   /* fingerprint verdict: every rc(x) present with count(x)        */
    int      have_direct;                 /* deg / up / filter allocated and the filter built               */
    int      have_symm;                   /* symmetric-scan work areas allocated, cuts aligned              */
    int      symm_ready;                  /* they hold the candidates of a symmetric run with a clean status  */
                                          /*   (what hm_scan_extract lists the pairs from)                    */
    int      last_path;                   /* HM_PATH_DIRECT / HM_PATH_SYMM of the last run                  */
    int      invalid;                     /* a failed conditioning left the replicas inconsistent            */
    int      conditioned;                 /* hm_scan_condition changed the table: its files no longer describe it */
    const hm_host_table *src;             /* the table hm_scan_create was given (hm_scan_condition_files reads it) */
    hm_symm_shards ssh[HM_MAX_GPUS];
    uint64_t seed[2];
    /* residency (DESIGN.md §4c) */
    int64_t  budget;                      /* device bytes this scan may hold per GPU (streamed: per shard)    */
    int64_t  incore_bytes;                /* what the in-core scan allocates per GPU                          */
    int      streamed;                    /* nothing resident: every run streams the host table, each shard   */
                                          /*   its run-aligned range [d[r].lo, d[r].hi) through d[r].dev      */
    const hm_host_table *host;            /* (streamed) the caller's table, valid until hm_scan_destroy        */
    hm_stream_layout plan;                /* (streamed) per shard                                              */
    volatile int stop;                    /* (streamed) a shard failed: the others leave their chunk loops     */
    int      nshard, rank;                /* (streamed) shards of the table, and the one d[0] streams: n_gpus and 0  */
                                          /*   in one process, (world, rank) for one rank of a job (hm_rank_scan)  */
    hm_spill_stats spill;                 /* (streamed) what the last run did with its lists (hm_scan_spill_stats) */
    int64_t  list_cap;                    /* (streamed) the run's list host budget (0: the lists stay on the device) */
    int64_t  host_held;                   /* (streamed) host bytes the lists of every shard hold                     */
    const char *list_knob;                /* (streamed) what sets list_cap, for messages (NULL: the environment's)  */
  };

static double now_ms(void)
{ struct timespec ts;
  clock_gettime(CLOCK_MONOTONIC,&ts);
  return ts.tv_sec*1e3 + ts.tv_nsec*1e-6;
}

/* multi-GPU helpers (hm_peer.cu) */
int hm_peer_enable(const int *dev, int n);
int hm_peer_sum_deg(uint8_t **deg, const int64_t *lo, const int64_t *hi, const int *dev,
                    cudaStream_t *st, int n, int64_t nels);
int hm_peer_sum_plot(unsigned long long **plot, const int *dev, cudaStream_t *st, int n);

/* rc = the first failure of a sequence of CUDA calls (needs cudaError_t e and int rc in scope) */
#define TRY(call) do { if (rc == HM_OK && (e = (call)) != cudaSuccess) rc = hm_cuda_fail(e,#call); } while (0)

/* Every device allocation of a DevTable goes through dev_alloc / dev_free, which keep its size in D->held and
 * D->peak.  Allocations of a one-GPU scan come from the device's stream-ordered memory pool with a release
 * threshold of "never": a second hm_scan_create in the same process (bench e2e leg, a service handling many
 * tables) reuses the memory instead of paying cudaMalloc / cudaFree of several GB every call.  Multi-GPU scans
 * keep cudaMalloc: their arrays are mapped by the peers.  HETMERS_NO_POOL=1 disables the pool.               */
typedef struct DevBlock { void *p; int64_t bytes; int pooled; struct DevBlock *next; } DevBlock;

/* whether D's allocations may come from the pool */
static int pool_setup(int dev, int enable)
{ static int configured[64] = {0};
  if (!enable || dev < 0 || dev >= 64 || getenv("HETMERS_NO_POOL") != NULL)
    return 0;
  if (configured[dev] == 0)
    { cudaMemPool_t pool;
      unsigned long long never = ~0ull;
      configured[dev] = 1;
      if (cudaDeviceGetDefaultMemPool(&pool,dev) != cudaSuccess ||
          cudaMemPoolSetAttribute(pool,cudaMemPoolAttrReleaseThreshold,&never) != cudaSuccess)
        { cudaGetLastError(); configured[dev] = -1; }
    }
  return configured[dev] == 1;
}

static void dev_release(DevTable *D, void *p, int pooled)
{ if (pooled) cudaFreeAsync(p,D->st);
  else        cudaFree(p);
}

/* *pp = `bytes` of device memory on D's device (current), stream-ordered on D->st when pooled, counted in D->held */
static cudaError_t dev_alloc(DevTable *D, void *pp, int64_t bytes)
{ void      **p = (void **) pp;
  cudaError_t e = cudaErrorMemoryAllocation;
  int         pooled = 0;
  if (D->pool)
    { if ((e = cudaMallocAsync(p,(size_t) bytes,D->st)) == cudaSuccess) pooled = 1;
      else                                                               cudaGetLastError();
    }
  if (!pooled && (e = cudaMalloc(p,(size_t) bytes)) != cudaSuccess)
    return e;
  DevBlock *b = (DevBlock *) malloc(sizeof(DevBlock));
  if (b == NULL)                                           /* out of host memory: it cannot be counted */
    { dev_release(D,*p,pooled);
      *p = NULL;
      return cudaErrorMemoryAllocation;
    }
  b->p = *p; b->bytes = bytes; b->pooled = pooled; b->next = D->blocks;
  D->blocks = b;
  D->held += bytes;
  if (D->held > D->peak) D->peak = D->held;
  return cudaSuccess;
}

static void dev_unlink(DevTable *D, DevBlock **at)
{ DevBlock *b = *at;
  *at = b->next;
  dev_release(D,b->p,b->pooled);
  D->held -= b->bytes;
  free(b);
}

/* frees what dev_alloc gave; NULL is ignored */
static void dev_free(DevTable *D, void *p)
{ for (DevBlock **at = &D->blocks; p != NULL && *at != NULL; at = &(*at)->next)
    if ((*at)->p == p)
      { dev_unlink(D,at);
        return;
      }
}

/* the bytes of what dev_alloc gave as p; 0 for NULL */
static int64_t dev_bytes(const DevTable *D, const void *p)
{ for (const DevBlock *b = D->blocks; p != NULL && b != NULL; b = b->next)
    if (b->p == p)
      return b->bytes;
  return 0;
}

static void free_dev(DevTable *D)
{ cudaSetDevice(D->dev);
  while (D->blocks != NULL)
    dev_unlink(D,&D->blocks);
  if (D->st) cudaStreamSynchronize(D->st);
  if (D->st)      cudaStreamDestroy(D->st);
  if (D->st_copy) cudaStreamDestroy(D->st_copy);
  for (int k = 0; k < 4; k++)
    if (D->ev[k]) cudaEventDestroy(D->ev[k]);
  memset(D,0,sizeof(*D));
}

/* set each GPU's device and synchronise its stream; the first error */
static int sync_all(hm_scan *s, const char *what)
{ int rc = HM_OK;
  for (int g = 0; g < s->ngpu; g++)
    { cudaError_t e = cudaSetDevice(s->d[g].dev);
      if (e == cudaSuccess) e = cudaStreamSynchronize(s->d[g].st);
      if (e != cudaSuccess && rc == HM_OK) rc = hm_cuda_fail(e,what);
    }
  return rc;
}

/* the slowest GPU's time from its event a to its event b */
static float slowest_ms(hm_scan *s, int a, int b)
{ float worst = 0;
  for (int g = 0; g < s->ngpu; g++)
    { float ms = 0;
      cudaSetDevice(s->d[g].dev);
      if (cudaEventElapsedTime(&ms,s->d[g].ev[a],s->d[g].ev[b]) == cudaSuccess && ms > worst) worst = ms;
    }
  cudaGetLastError();
  return worst;
}

/* fn(s, g, arg) for every GPU g at once, a host thread each (the calling thread takes the last).  A failure sets
 * s->stop, which the shards of a streamed run watch; the first failing GPU's error wins, naming its shard when
 * there are several                                                                                            */
typedef int (*GpuFn)(hm_scan *s, int g, void *arg);
typedef struct { hm_scan *s; int g; GpuFn fn; void *arg; int rc; char msg[512]; } GpuJob;

static void *gpu_worker(void *p)
{ GpuJob *J = (GpuJob *) p;
  J->rc = J->fn(J->s,J->g,J->arg);
  if (J->rc != HM_OK)
    { J->s->stop = 1;
      strncpy(J->msg,hm_last_error(),sizeof(J->msg)-1); J->msg[sizeof(J->msg)-1] = 0;
    }
  return NULL;
}

static int on_every_gpu(hm_scan *s, GpuFn fn, void *arg)
{ int       G = s->ngpu, rc = HM_OK;
  GpuJob    job[HM_MAX_GPUS];
  pthread_t th[HM_MAX_GPUS];
  int       created[HM_MAX_GPUS];
  for (int g = 0; g < G; g++)
    { memset(job+g,0,sizeof(job[g]));
      job[g].s = s; job[g].g = g; job[g].fn = fn; job[g].arg = arg;
      created[g] = (g < G-1 && pthread_create(th+g,NULL,gpu_worker,job+g) == 0);
      if (!created[g])
        gpu_worker(job+g);
    }
  for (int g = 0; g < G; g++)
    { if (created[g]) pthread_join(th[g],NULL);
      if (job[g].rc != HM_OK && rc == HM_OK)
        rc = G == 1 ? hm_set_error(job[g].rc,"%s",job[g].msg)
                    : hm_set_error(job[g].rc,"shard %d of %d (GPU %d, entries %lld..%lld): %s",g,G,s->d[g].dev,
                                   (long long) s->d[g].lo,(long long) s->d[g].hi,job[g].msg);
    }
  return rc;
}

extern "C" void hm_scan_destroy(hm_scan *s)
{ if (s == NULL)
    return;
  for (int g = 0; g < s->ngpu; g++)
    { int had_symm = (s->d[g].symm_work != NULL);
      free_dev(s->d+g);
      if (had_symm)                              /* hand the L2 lines the Bloom window made persisting back */
        { cudaCtxResetPersistingL2Cache(); cudaGetLastError(); }
    }
  free(s);
}

/* ---- host-side staging for pageable sources (mmap'ed part files) -------------------------
 * cudaMemcpyAsync from pageable memory is staged by the driver on one thread.  The
 * executable's table lives in the page cache, so the loader copies each chunk into a pinned
 * buffer with a few host threads (this is what the reference's -T is for on the host side) while
 * the previous chunk is in flight to the GPU.                                                   */
static int g_io_threads = 0;

extern "C" void hm_set_io_threads(int n) { g_io_threads = n; }

typedef struct { uint8_t *dst; const uint8_t *src; size_t bytes; int fd; int64_t off; int err; } CopyJob;

static void *copy_worker(void *arg)
{ CopyJob *j = (CopyJob *) arg;
  j->err = 0;
  if (j->fd < 0)
    memcpy(j->dst,j->src,j->bytes);
  else
    { size_t got = 0;                                   /* page cache -> pinned buffer, no mapping */
      while (got < j->bytes)
        { ssize_t r = pread(j->fd,j->dst+got,j->bytes-got,j->off+(int64_t) got);
          if (r < 0 && errno == EINTR) continue;
          if (r <= 0) { j->err = (r < 0) ? errno : -1; break; }    /* -1: file shorter than its header says */
          got += (size_t) r;
        }
    }
  return NULL;
}

/* fill dst[0,bytes) from memory `src` (fd < 0) or from file `fd` at `off`, with the I/O threads;
 * 0, or the errno (-1 = short file) of the first slice that could not be read                  */
static int parallel_fill(uint8_t *dst, const uint8_t *src, int fd, int64_t foff, size_t bytes)
{ int nt = g_io_threads;
  if (nt <= 0)
    { long c = sysconf(_SC_NPROCESSORS_ONLN);
      nt = c > 16 ? 16 : (c < 1 ? 1 : (int) c);
    }
  if (nt > 64) nt = 64;
  if (bytes < ((size_t) 4<<20)) nt = 1;
  pthread_t th[64];
  CopyJob   job[64];
  int       created[64];
  size_t    per = ((bytes/nt)+4095) & ~(size_t) 4095;
  int       njob = 0, err = 0;
  for (int k = 0; k < nt; k++)
    { size_t off = per*k;
      if (off >= bytes) break;
      job[k].dst = dst+off; job[k].src = src ? src+off : NULL;
      job[k].fd = fd; job[k].off = foff+(int64_t) off;
      job[k].bytes = bytes-off < per ? bytes-off : per;
      created[k] = 0;
      njob = k+1;
      if (k == nt-1 || off+per >= bytes)
        { copy_worker(job+k); break; }                 /* the calling thread takes the last slice */
      if (pthread_create(th+k,NULL,copy_worker,job+k) != 0)
        copy_worker(job+k);                            /* no thread to be had: copy inline */
      else
        created[k] = 1;
    }
  for (int k = 0; k < njob; k++)
    { if (created[k])
        pthread_join(th[k],NULL);
      if (job[k].err != 0 && err == 0)
        err = job[k].err;
    }
  return err;
}

/* ---- background start-up (hm_prewarm) ---- */
#define PIN_CACHE_BYTES ((size_t) (LOAD_CHUNK/2) * 8)
static pthread_t g_warm_th;
static int       g_warm_state = 0;            /* 0 idle, 1 running, 2 joined */
static int       g_warm_ngpu = 1;
static uint8_t  *g_pin_cache[2] = { NULL, NULL };

static void *warm_one(void *arg)
{ int g = (int) (intptr_t) arg;
  if (cudaSetDevice(g) == cudaSuccess)
    cudaFree(0);                              /* creates the primary context */
  return NULL;
}

static void *warm_worker(void *)
{ int n = 0;
  if (cudaGetDeviceCount(&n) != cudaSuccess)
    { cudaGetLastError(); return NULL; }
  int use = (g_warm_ngpu <= 0 || g_warm_ngpu > n) ? n : g_warm_ngpu;
  if (use > HM_MAX_GPUS) use = HM_MAX_GPUS;
  pthread_t th[HM_MAX_GPUS];
  int       made[HM_MAX_GPUS];
  for (int g = 1; g < use; g++)               /* the contexts of several GPUs at once */
    made[g] = (pthread_create(th+g,NULL,warm_one,(void *) (intptr_t) g) == 0);
  warm_one((void *) (intptr_t) 0);
  for (int g = 1; g < use; g++)
    if (made[g]) pthread_join(th[g],NULL);
    else         warm_one((void *) (intptr_t) g);
  cudaSetDevice(0);
  for (int i = 0; i < 2; i++)
    if (cudaHostAlloc(&g_pin_cache[i],PIN_CACHE_BYTES,cudaHostAllocDefault) != cudaSuccess)
      { cudaGetLastError(); g_pin_cache[i] = NULL; }
  return NULL;
}

extern "C" void hm_prewarm(int n_gpus)
{ if (g_warm_state != 0)
    return;
  g_warm_ngpu = n_gpus;
  if (pthread_create(&g_warm_th,NULL,warm_worker,NULL) == 0)
    g_warm_state = 1;
}

static void prewarm_join(void)
{ if (g_warm_state == 1)
    { pthread_join(g_warm_th,NULL);
      g_warm_state = 2;
    }
}

static int is_pageable(const void *p)
{ cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a,p) != cudaSuccess)
    { cudaGetLastError(); return 1; }
  return (a.type == cudaMemoryTypeUnregistered);
}

/* Host -> device staging of table records: two device staging buffers (the copy of chunk c+1 overlaps the
 * unpack of chunk c) and, for pageable sources, two pinned host buffers filled by host threads.          */
typedef struct
  { uint8_t    *stage[2], *pin[2];
    int         pin_cached[2], staged, used[2], b;
    cudaEvent_t copied[2], unpacked[2];
    int64_t     chunk;                /* records per H2D copy */
  } Stager;

static int stager_open(hm_scan *s, DevTable *D, const hm_host_table *t, int64_t count, Stager *G)
{ int kbyte = (t->kmer+3)>>2;
  int pbyte = kbyte - t->ibyte + 2;
  memset(G,0,sizeof(*G));
  G->chunk = LOAD_CHUNK;
  for (int p = 0; p < t->nparts && !G->staged; p++)
    if (t->part_nels[p] > 0 &&
        ((t->part_fd != NULL && t->part_fd[p] >= 0) || is_pageable(t->part_rec[p])))
      G->staged = 1;
  if (G->staged)
    G->chunk = LOAD_CHUNK/2;
  if (G->chunk > count) G->chunk = count;
  for (int i = 0; i < 2; i++)
    { HM_CUDA(dev_alloc(D,&G->stage[i],G->chunk*pbyte));
      if (G->staged)
        { if (s->ngpu == 1 && g_pin_cache[i] != NULL && (size_t) G->chunk*pbyte <= PIN_CACHE_BYTES)
            { G->pin[i] = g_pin_cache[i]; g_pin_cache[i] = NULL; G->pin_cached[i] = 1; }   /* from hm_prewarm */
          else
            HM_CUDA(cudaHostAlloc(&G->pin[i],(size_t) G->chunk*pbyte,cudaHostAllocDefault));
        }
      HM_CUDA(cudaEventCreateWithFlags(&G->copied[i],cudaEventDisableTiming));
      HM_CUDA(cudaEventCreateWithFlags(&G->unpacked[i],cudaEventDisableTiming));
    }
  HM_CUDA(cudaStreamSynchronize(D->st));         /* (pool) allocations are used on both streams */
  return HM_OK;
}

static void stager_close(DevTable *D, Stager *G)
{ for (int i = 0; i < 2; i++)
    { dev_free(D,G->stage[i]);
      if (G->copied[i] != NULL)   cudaEventDestroy(G->copied[i]);
      if (G->unpacked[i] != NULL) cudaEventDestroy(G->unpacked[i]);
      if (G->pin[i] != NULL)
        { if (G->pin_cached[i]) g_pin_cache[i] = G->pin[i];        /* back into the cache for the next table */
          else                  cudaFreeHost(G->pin[i]);
        }
    }
  memset(G,0,sizeof(*G));
}

/* Load ordinals [first, first+count) of the table into keys/keys_lo/cnt (which receive ordinal `first`
 * at index 0).  Walks the parts, copies payload chunks H2D on st_copy into the stager's device buffers
 * and unpacks them on st.  extras: D's arrays hold the whole table -- build its bucket index chunk by chunk
 * (one GPU) and add the symmetry fingerprint of what is loaded.                                        */
static int load_into(hm_scan *s, DevTable *D, const hm_host_table *t, const int64_t *d_index,
                     int64_t first, int64_t count, uint64_t *keys, uint64_t *keys_lo, uint16_t *cnt,
                     int extras, Stager *G)
{ int      kbyte = (t->kmer+3)>>2;
  int      pbyte = kbyte - t->ibyte + 2;
  int64_t  chunk = G->chunk;
  int      rc = HM_OK;

  if (count <= 0)
    return HM_OK;
  /* one GPU: the whole table arrives here in order, so the bucket index is built chunk by chunk
   * right behind the unpack (hidden behind the next chunk's H2D); so is the symmetry fingerprint   */
  const int inc = extras && (s->ngpu == 1 && first == 0 && count == s->n);
  int64_t pstart = 0;                               /* ordinal of the part's first record */
  for (int p = 0; p < t->nparts && rc == HM_OK; p++)
    { int64_t pn   = t->part_nels[p];
      int64_t from = first > pstart ? first : pstart;
      int64_t to   = first+count < pstart+pn ? first+count : pstart+pn;
      for (int64_t o = from; o < to && rc == HM_OK; o += chunk)
        { int64_t        m   = to-o < chunk ? to-o : chunk;
          const uint8_t *src = t->part_rec[p] + (o-pstart)*pbyte;
          int            b   = G->b;
          if (G->staged)
            { if (G->used[b])
                cudaEventSynchronize(G->copied[b]);   /* pin[b] has left for the GPU */
              int ferr;
              if (t->part_fd != NULL && t->part_fd[p] >= 0)
                ferr = parallel_fill(G->pin[b],NULL,t->part_fd[p],t->part_fd_off[p]+(o-pstart)*pbyte,(size_t) m*pbyte);
              else
                ferr = parallel_fill(G->pin[b],src,-1,0,(size_t) m*pbyte);
              if (ferr != 0)
                { rc = hm_set_error(HM_EIO,"short read on part %d of the table (%s)",p+1,
                                    ferr > 0 ? strerror(ferr) : "file truncated");
                  break;
                }
              src = G->pin[b];
            }
          if (G->used[b])
            cudaStreamWaitEvent(D->st_copy,G->unpacked[b],0);
          cudaError_t e = cudaMemcpyAsync(G->stage[b],src,(size_t) m*pbyte,cudaMemcpyHostToDevice,D->st_copy);
          if (e != cudaSuccess) { rc = hm_cuda_fail(e,"cudaMemcpyAsync(H2D records)"); break; }
          cudaEventRecord(G->copied[b],D->st_copy);
          cudaStreamWaitEvent(D->st,G->copied[b],0);
          int64_t at = o-first;
          rc = hm_k_unpack_records(G->stage[b],m,o,d_index,t->ibyte,t->kmer,keys+at,
                                   keys_lo ? keys_lo+at : NULL,cnt+at,D->st);
          __sync_fetch_and_add(&s->launches,1);
          cudaEventRecord(G->unpacked[b],D->st);
          if (inc && rc == HM_OK)
            { rc = hm_build_bucket_index_range(D->keys,s->n,s->bits,D->bucket,s->idx64,o,o+m,D->st);
              __sync_fetch_and_add(&s->launches,1);
            }
          if (extras && rc == HM_OK && s->kmer >= HM_SYMM_MIN_KMER)   /* symmetry fingerprint of what this device loads */
            { rc = hm_k_symm_fingerprint(D->keys,D->keys_lo,D->cnt,o,o+m,s->kmer,s->seed,D->fp_acc,D->st);
              __sync_fetch_and_add(&s->launches,1);
            }
          G->used[b] = 1;
          G->b ^= 1;
        }
      pstart += pn;
    }
  cudaStreamSynchronize(D->st_copy);
  cudaError_t e = cudaStreamSynchronize(D->st);
  if (rc == HM_OK && e != cudaSuccess)
    rc = hm_cuda_fail(e,"unpack");
  return rc;
}

/* ordinals [first, first+count) into D's full-table arrays */
static int load_range(hm_scan *s, DevTable *D, const hm_host_table *t, const int64_t *d_index,
                      int64_t first, int64_t count)
{ Stager G;
  if (count <= 0)
    return HM_OK;
  int rc = stager_open(s,D,t,count,&G);
  if (rc == HM_OK)
    rc = load_into(s,D,t,d_index,first,count,D->keys+first,D->keys_lo ? D->keys_lo+first : NULL,
                   D->cnt+first,1,&G);
  stager_close(D,&G);
  return rc;
}

/* on_every_gpu: stub index upload + this device's shard of the records of table t */
static int load_shard(hm_scan *s, int g, void *t)
{ const hm_host_table *T = (const hm_host_table *) t;
  DevTable *D = s->d+g;
  int64_t  *d_index = NULL;
  int64_t   ixlen = (int64_t) 1 << (8*T->ibyte);
  cudaError_t e = cudaSetDevice(D->dev);
  if (e == cudaSuccess) e = dev_alloc(D,&d_index,sizeof(int64_t)*ixlen);
  if (e == cudaSuccess) e = cudaMemcpyAsync(d_index,T->index,sizeof(int64_t)*ixlen,cudaMemcpyHostToDevice,D->st);
  if (e == cudaSuccess) e = cudaMemsetAsync(D->fp_acc,0,4*sizeof(uint64_t),D->st);
  if (e == cudaSuccess) e = cudaStreamSynchronize(D->st);     /* pool memory is about to be used on the copy stream too */
  int rc = e != cudaSuccess ? hm_cuda_fail(e,"stub index upload") : load_range(s,D,T,d_index,D->lo,D->hi-D->lo);
  dev_free(D,d_index);
  return rc;
}

/* sum of the per-device fingerprint accumulators -> s->symmetric */
static int fingerprint_verdict(hm_scan *s)
{ uint64_t tot[4] = {0,0,0,0};
  if (s->kmer < HM_SYMM_MIN_KMER)
    { s->symmetric = 0; return HM_OK; }
  for (int g = 0; g < s->ngpu; g++)
    { uint64_t h[4];
      HM_CUDA(cudaSetDevice(s->d[g].dev));
      HM_CUDA(cudaMemcpyAsync(h,s->d[g].fp_acc,sizeof(h),cudaMemcpyDeviceToHost,s->d[g].st));
      HM_CUDA(cudaStreamSynchronize(s->d[g].st));
      for (int k = 0; k < 4; k++) tot[k] += h[k];
    }
  s->symmetric = (tot[0] == tot[2] && tot[1] == tot[3]);
  return HM_OK;
}

/* ---- device budget ---------------------------------------------------------------------------------- */
static int64_t g_budget = 0;

extern "C" void hm_set_device_budget(int64_t bytes) { g_budget = bytes > 0 ? bytes : 0; }

/* host bytes a streamed run's lists may take in host memory (0: they stay on the device or the run refuses) */
static int64_t g_list_host_budget = 0;

extern "C" void hm_set_list_host_budget(int64_t bytes) { g_list_host_budget = bytes > 0 ? bytes : 0; }

/* pass 2 of lists in host memory: device bytes of a slice of c candidates with its pending slots, queries and
 * their sort scratch, and of a partition of p S keys with its bucket index                                  */
static int64_t spill_slice_bytes(int64_t c, int KW)
{ return c*(8*KW+8) + 8*c + 2*c*(2*(8*KW+8)+1) + 2*c*HM_SPILL_SORT_Q + HM_SPILL_SORT_FIXED; }

static int64_t spill_part_bytes(int64_t p, int KW)
{ return p*8*KW + 4*((1ll << hm_pick_bucket_bits(p))+1); }

/* the largest x <= most with f(x) <= room (f increasing), 0 if none */
static int64_t spill_largest(int64_t most, int64_t room, int KW, int64_t (*f)(int64_t, int))
{ int64_t lo = 0, hi = most;
  while (lo < hi)
    { int64_t mid = lo + (hi-lo+1)/2;
      if (f(mid,KW) <= room) lo = mid; else hi = mid-1;
    }
  return lo;
}

extern "C" int hm_spill_plan(int64_t n_cand, int64_t n_s, int kmer, int64_t room, hm_spill_layout *out)
{ if (n_cand < 0 || n_s < 0 || kmer < 1 || kmer > HM_MAX_KMER || out == NULL)
    return hm_set_error(HM_EINVAL,"hm_spill_plan: bad arguments");
  int     KW = kmer > 32 ? 2 : 1;
  int64_t nc = n_cand > 1 ? n_cand : 1, np = n_s > 1 ? n_s : 1, slice, part;
  if (nc > HM_SPILL_MAX_SLICE) nc = HM_SPILL_MAX_SLICE;      /* query indices and slots are 32-bit        */
  if (np > HM_SPILL_MAX_PART)  np = HM_SPILL_MAX_PART;       /* a partition's bucket index is 32-bit      */
  if (spill_slice_bytes(nc,KW) + spill_part_bytes(np,KW) <= room)
    { slice = nc; part = np; }
  else
    { slice = spill_largest(nc,room/2,KW,spill_slice_bytes);
      part  = spill_largest(np,room-spill_slice_bytes(slice,KW),KW,spill_part_bytes);
      slice = spill_largest(nc,room-spill_part_bytes(part,KW),KW,spill_slice_bytes);
    }
  int64_t min_c = nc < HM_SPILL_MIN ? nc : HM_SPILL_MIN, min_p = np < HM_SPILL_MIN ? np : HM_SPILL_MIN;
  if (slice < min_c || part < min_p)
    return hm_set_error(HM_ENOMEM,"pass 2 of the streamed scan's lists in host memory has %lld bytes of device room, "
                        "and slices of %lld candidates (%lld bytes) beside partitions of %lld S keys (%lld bytes) need "
                        "%lld; give the scan a larger device budget (HETMERS_DEVICE_BUDGET)",(long long) room,
                        (long long) min_c,(long long) spill_slice_bytes(min_c,KW),(long long) min_p,
                        (long long) spill_part_bytes(min_p,KW),
                        (long long) (spill_slice_bytes(min_c,KW) + spill_part_bytes(min_p,KW)));
  memset(out,0,sizeof(*out));
  out->room = room;
  out->slice = slice; out->queries = 2*slice;
  out->part = part; out->part_bits = hm_pick_bucket_bits(part);
  out->slice_bytes = spill_slice_bytes(slice,KW); out->part_bytes = spill_part_bytes(part,KW);
  return HM_OK;
}

/* a rank's parked routed rounds (hm_rank_spill_plan): device bytes of the slice and receive sides of a slice of c
 * candidates, for `world` ranks, counting or listing                                                          */
static int64_t rank_spill_slice_bytes(int64_t c, int KW, int world, int listing)
{ int64_t send = c*(8*KW+8) + 8*c + 2*c*(8*KW+8) + 2*c*(8*KW+4) + 2*c;
  int64_t keep = listing ? c*8*KW + 2*c*(int64_t) sizeof(hm_pair_rec) : 0;
  int64_t recv = (int64_t) world*2*c*(2*8*KW + 8 + 2 + HM_SPILL_SORT_Q) + HM_SPILL_SORT_FIXED;
  return send + keep + recv + HM_RANK_SPILL_FIXED;
}

/* the largest c <= most whose slice side fits room, 0 if none */
static int64_t rank_spill_largest(int64_t most, int64_t room, int KW, int world, int listing)
{ int64_t lo = 0, hi = most;
  while (lo < hi)
    { int64_t mid = lo + (hi-lo+1)/2;
      if (rank_spill_slice_bytes(mid,KW,world,listing) <= room) lo = mid; else hi = mid-1;
    }
  return lo;
}

extern "C" int hm_rank_spill_plan(int64_t n_cand, int64_t n_s, int kmer, int world, int listing, int64_t room,
                                  hm_spill_layout *out)
{ if (n_cand < 0 || n_s < 0 || kmer < 1 || kmer > HM_MAX_KMER || world < 1 || world > HM_MAX_SHARDS || out == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_spill_plan: bad arguments");
  int     KW = kmer > 32 ? 2 : 1, L = listing != 0;
  int64_t nc = n_cand > 1 ? n_cand : 1, np = n_s > 1 ? n_s : 1, slice, part;
  if (nc > HM_SPILL_MAX_SLICE/world) nc = HM_SPILL_MAX_SLICE/world;    /* received keys are sorted with 32-bit indices */
  if (np > HM_SPILL_MAX_PART)        np = HM_SPILL_MAX_PART;           /* a partition's bucket index is 32-bit      */
  if (rank_spill_slice_bytes(nc,KW,world,L) + spill_part_bytes(np,KW) <= room)
    { slice = nc; part = np; }
  else
    { slice = rank_spill_largest(nc,room/2,KW,world,L);
      part  = spill_largest(np,room-rank_spill_slice_bytes(slice,KW,world,L),KW,spill_part_bytes);
      slice = rank_spill_largest(nc,room-spill_part_bytes(part,KW),KW,world,L);
    }
  int64_t min_c = nc < HM_SPILL_MIN ? nc : HM_SPILL_MIN, min_p = np < HM_SPILL_MIN ? np : HM_SPILL_MIN;
  if (slice < min_c || part < min_p)
    return hm_set_error(HM_ENOMEM,"pass 2 of a rank's lists in host memory has %lld bytes of device room, and %s slices "
                        "of %lld candidates with what %d ranks send for them (%lld bytes) beside partitions of %lld S "
                        "keys (%lld bytes) need %lld; give the rank a larger device budget",(long long) room,
                        L ? "listing" : "counting",(long long) min_c,world,
                        (long long) rank_spill_slice_bytes(min_c,KW,world,L),(long long) min_p,
                        (long long) spill_part_bytes(min_p,KW),
                        (long long) (rank_spill_slice_bytes(min_c,KW,world,L) + spill_part_bytes(min_p,KW)));
  memset(out,0,sizeof(*out));
  out->room = room;
  out->slice = slice; out->queries = 2*slice;
  out->part = part; out->part_bits = hm_pick_bucket_bits(part);
  out->slice_bytes = rank_spill_slice_bytes(slice,KW,world,L); out->part_bytes = spill_part_bytes(part,KW);
  return HM_OK;
}

/* the budget per GPU: the one set, or the smallest free memory of the devices (counting what an idle
 * stream-ordered pool keeps reserved for us) minus a reserve for the CUDA runtime and library code; a device
 * listed m times (shards of a streamed scan sharing it) gives each of them 1/m of that                  */
static int64_t device_budget(const int *dev, int n_gpus)
{ if (g_budget > 0)
    return g_budget;
  int64_t best = -1;
  for (int g = 0; g < n_gpus; g++)
    { int    d = dev ? dev[g] : g, m = 0;
      for (int h = 0; h < n_gpus; h++)
        m += ((dev ? dev[h] : h) == d);
      size_t fr = 0, tot = 0;
      if (cudaSetDevice(d) != cudaSuccess || cudaMemGetInfo(&fr,&tot) != cudaSuccess)
        { cudaGetLastError(); continue; }
      int64_t f = (int64_t) fr;
      cudaMemPool_t pool;
      unsigned long long res = 0, used = 0;
      if (cudaDeviceGetDefaultMemPool(&pool,d) == cudaSuccess &&
          cudaMemPoolGetAttribute(pool,cudaMemPoolAttrReservedMemCurrent,&res) == cudaSuccess &&
          cudaMemPoolGetAttribute(pool,cudaMemPoolAttrUsedMemCurrent,&used) == cudaSuccess && res > used)
        f += (int64_t) (res-used);
      cudaGetLastError();
      f = f > HM_BUDGET_RESERVE ? (f-HM_BUDGET_RESERVE)/m : 0;
      if (best < 0 || f < best) best = f;
    }
  return best < 0 ? 0 : best;
}

/* device bytes the in-core scan allocates per GPU: table arrays, bucket index, plot, fingerprint sums and the
 * symmetric scan's work area (the direct passes' buffers come on top only for tables that need them)     */
static int64_t incore_bytes(int64_t n, int kmer, int n_gpus, int bits, int idx64)
{ int64_t b = 8*(n+1) + (kmer > 32 ? 8*(n+1) : 0) + 2*(n+8) + (int64_t) (idx64 ? 8 : 4)*((1ll << bits)+1) +
              8*(int64_t) HM_PLOT_CELLS + 32;
  hm_symm_layout L;
  if (kmer >= HM_SYMM_MIN_KMER && hm_symm_plan(n,(n+n_gpus-1)/n_gpus < n ? (n+n_gpus-1)/n_gpus : n,kmer,n_gpus,&L) == HM_OK)
    b += L.bytes;
  return b;
}

/* ---- the streamed scan's plan --------------------------------------------------------------------- */
#define STREAM_MIN_CHUNK 256

/* work area of the streamed scan: header + the whole-table Bloom filter of hm_symm_plan (a segment per shard) */
static int stream_work_layout(int64_t n, int kmer, int n_seg, hm_symm_layout *L)
{ int rc = hm_symm_plan(n,0,kmer,n_seg,L);
  if (rc != HM_OK) return rc;
  L->bytes = (L->off_cand_key+255) & ~255ll;
  L->cand_cap = 0; L->runs_cap = 0;
  return HM_OK;
}

static int64_t stage_bytes(int64_t chunk, int kmer, int ibyte)
{ int64_t c = chunk < LOAD_CHUNK ? chunk : LOAD_CHUNK;
  return 2*c*(((kmer+3)>>2) - ibyte + 2);
}

/* two chunk buffers (keys, second words, counts), their bucket index, the run list, staging, and the
 * scratch that sorts a chunk's S keys                                                                 */
static int64_t chunk_bytes(int64_t c, int kmer, int ibyte)
{ int KW = kmer > 32 ? 2 : 1;
  return 2*(8*KW*(c+1) + 2*(c+8)) + 4*((1ll << hm_pick_bucket_bits(c))+1) + 8*(c/3+1024) + stage_bytes(c,kmer,ibyte) +
         hm_sort_keys_bytes(c+1024,kmer);
}

/* list room one chunk of c entries may take: a candidate record per two entries, an S key per entry */
static int64_t chunk_list_bytes(int64_t c, int kmer)
{ int KW = kmer > 32 ? 2 : 1;
  return (8*KW+8)*(c/2+1024) + 8*KW*(c+1024);
}

/* several shards: the room for each one's lists and chunks is planned from its share of n/G entries (chunks no
 * longer than the share); every shard holds the whole-table Bloom filter of G segments                  */
extern "C" int hm_stream_plan_shards(int64_t n, int kmer, int ibyte, int64_t budget, int n_shards, hm_stream_layout *out)
{ if (out == NULL || n < 0 || kmer < 1 || kmer > HM_MAX_KMER || ibyte < 1 || ibyte > 3 || budget < 0 ||
      n_shards < 1 || n_shards > HM_MAX_GPUS)
    return hm_set_error(HM_EINVAL,"hm_stream_plan_shards: bad arguments");
  hm_symm_layout L;
  int rc = stream_work_layout(n,kmer,n_shards,&L);
  if (rc != HM_OK) return rc;
  memset(out,0,sizeof(*out));
  out->budget = budget;
  out->fixed_bytes = 8*(1ll << (8*ibyte)) + 8*(int64_t) HM_PLOT_CELLS + 32 + L.bytes;
  /* the largest chunk whose buffers + list room take at most a quarter of what is left: the rest is for
   * the candidate records and S keys of the chunks before it (a few B per entry of the share) and
   * for growing those lists, which holds the old and the new array at once                             */
  int64_t share = (n+n_shards-1)/n_shards;
  int64_t avail = budget - out->fixed_bytes, lo = 0, hi = share < (1ll << 31) ? share : (1ll << 31);
  if (avail > 0)
    while (lo < hi)
      { int64_t mid = lo + (hi-lo+1)/2;
        if (chunk_bytes(mid,kmer,ibyte) + chunk_list_bytes(mid,kmer) <= avail/4) lo = mid;
        else                                                                   hi = mid-1;
      }
  int64_t need = share < STREAM_MIN_CHUNK ? share : STREAM_MIN_CHUNK;
  if (avail <= 0 || lo < need || lo < 1)
    return hm_set_error(HM_ENOMEM,"a device budget of %lld bytes cannot hold one chunk of the streamed scan: "
                        "%lld bytes are fixed (stub index, plot, Bloom filter of %lld entries) and a chunk of "
                        "%lld entries needs %lld more",(long long) budget,(long long) out->fixed_bytes,(long long) n,
                        (long long) need,(long long) (chunk_bytes(need,kmer,ibyte)+chunk_list_bytes(need,kmer)));
  out->chunk = lo;
  out->chunk_bytes = chunk_bytes(lo,kmer,ibyte);
  out->chunk_list_bytes = chunk_list_bytes(lo,kmer);
  out->list_bytes = budget - out->fixed_bytes - out->chunk_bytes;
  return HM_OK;
}

extern "C" int hm_stream_plan(int64_t n, int kmer, int ibyte, int64_t budget, hm_stream_layout *out)
{ if (out == NULL || n < 0 || kmer < 1 || kmer > HM_MAX_KMER || ibyte < 1 || ibyte > 3 || budget < 0)
    return hm_set_error(HM_EINVAL,"hm_stream_plan: bad arguments");
  return hm_stream_plan_shards(n,kmer,ibyte,budget,1,out);
}

/* streamed: the largest peak of a shard, the chunks of all shards */
extern "C" int hm_scan_residency(const hm_scan *s, int64_t *device_bytes, int64_t *chunks)
{ int64_t peak = 0, nch = 0;
  for (int g = 0; g < s->ngpu; g++)
    { if (s->d[g].peak > peak) peak = s->d[g].peak;
      nch += s->d[g].chunks;
    }
  if (device_bytes) *device_bytes = s->streamed ? peak : s->incore_bytes;
  if (chunks)       *chunks = s->streamed ? nch : 0;
  return s->streamed;
}

/* A window of `cap` entries onto the host table of a streamed scan, on the first GPU: keys, second words, counts,
 * the stub index and a Stager.  Between runs: it leaves the peak the last run reported as it was.           */
typedef struct { uint64_t *keys, *klo; uint16_t *cnt; int64_t *d_index; Stager G; int64_t peak; } Window;

static void window_close(hm_scan *s, Window *W)
{ DevTable *D = s->d;
  stager_close(D,&W->G);
  dev_free(D,W->keys); dev_free(D,W->klo); dev_free(D,W->cnt); dev_free(D,W->d_index);
  D->peak = W->peak;
}

static int window_open(hm_scan *s, int64_t cap, Window *W)
{ DevTable *D = s->d;
  int64_t   ixlen = (int64_t) 1 << (8*s->ibyte);
  int       rc = HM_OK;
  cudaError_t e;
  memset(W,0,sizeof(*W));
  W->peak = D->peak;
  TRY(cudaSetDevice(D->dev));
  TRY(dev_alloc(D,&W->keys,8*(cap+1)));
  if (s->kmer > 32) TRY(dev_alloc(D,&W->klo,8*(cap+1)));
  TRY(dev_alloc(D,&W->cnt,2*(cap+8)));
  TRY(dev_alloc(D,&W->d_index,8*ixlen));
  TRY(cudaMemcpyAsync(W->d_index,s->host->index,8*(size_t) ixlen,cudaMemcpyHostToDevice,D->st));
  if (rc == HM_OK)
    rc = stager_open(s,D,s->host,cap,&W->G);
  if (rc != HM_OK)
    window_close(s,W);
  return rc;
}

/* ordinals [first, first+count) into the window */
static int window_load(hm_scan *s, Window *W, int64_t first, int64_t count)
{ return load_into(s,s->d,s->host,W->d_index,first,count,W->keys,W->klo,W->cnt,0,&W->G); }

/* Shard cuts of a streamed scan over G = s->nshard shards, from the host table: c_r is the first run start (a run =
 * the entries sharing their first k/2 bases) at or after n*r/G -- hm_symm_align_cut's rule -- found by loading
 * a few records at a time around each nominal cut on the first device.  Sets the range and descriptor
 * (first_key[r] = word 0 of entry c_r) of the shards this process streams (shard s->rank + g on d[g]) and how
 * many shards own keys: those up to the last non-empty one (a run longer than a share can leave shards empty,
 * in the middle or at the end).                                                                          */
static int stream_cuts(hm_scan *s)
{ int      G = s->nshard, rc;
  int64_t  n = s->n, cut[HM_MAX_GPUS+1];
  uint64_t first[HM_MAX_GPUS];
  const int64_t W = 4096;
  const int psh = 64-2*(s->kmer>>1);
  uint64_t buf[4096];
  Window   win;
  cudaError_t e;
  if ((rc = window_open(s,W,&win)) != HM_OK)
    return rc;
  cut[0] = 0; cut[G] = n; first[0] = 0;
  for (int r = 1; r < G && rc == HM_OK; r++)
    { int64_t  c = n*r/G;
      uint64_t prev;
      if (c <= cut[r-1])                                   /* the run before reaches past this share's start */
        { cut[r] = cut[r-1]; first[r] = first[r-1]; continue; }
      if ((rc = window_load(s,&win,c-1,1)) != HM_OK) break;
      if ((e = cudaMemcpy(&prev,win.keys,8,cudaMemcpyDeviceToHost)) != cudaSuccess) { rc = hm_cuda_fail(e,"cut key"); break; }
      cut[r] = n; first[r] = ~0ull;
      for (int64_t o = c; o < n && rc == HM_OK; o += W)
        { int64_t m = n-o < W ? n-o : W, i;
          if ((rc = window_load(s,&win,o,m)) != HM_OK) break;
          if ((e = cudaMemcpy(buf,win.keys,8*(size_t) m,cudaMemcpyDeviceToHost)) != cudaSuccess)
            { rc = hm_cuda_fail(e,"cut keys"); break; }
          for (i = 0; i < m && ((buf[i] ^ prev) >> psh) == 0; i++)
            ;
          if (i < m)
            { cut[r] = o+i; first[r] = buf[i]; break; }
        }
    }
  window_close(s,&win);
  if (rc != HM_OK)
    return rc;
  int live = 1;                                            /* shards up to the last non-empty one */
  for (int r = 1; r < G; r++)
    if (cut[r] < n) live = r+1;
  for (int g = 0; g < s->ngpu; g++)
    { hm_symm_shards *sh = s->ssh+g;
      memset(sh,0,sizeof(*sh));
      sh->n_seg = live; sh->self = s->rank+g;
      for (int r = 0; r <= G; r++) sh->off[r] = cut[r];
      for (int r = 0; r < G; r++)  sh->first_key[r] = first[r];
      s->d[g].lo = cut[s->rank+g]; s->d[g].hi = cut[s->rank+g+1];
    }
  return HM_OK;
}

/* streamed: the plan of each of s->nshard shards under s->budget (HETMERS_STREAM_CHUNK: smaller chunks) */
static int stream_setup(hm_scan *s, const hm_host_table *t)
{ int rc = hm_stream_plan_shards(s->n,t->kmer,t->ibyte,s->budget,s->nshard,&s->plan);
  if (rc != HM_OK)
    return rc;
  const char *cc = getenv("HETMERS_STREAM_CHUNK");         /* smaller chunks than the budget allows */
  if (cc != NULL && atoll(cc) >= 1 && atoll(cc) < s->plan.chunk)
    { s->plan.chunk = atoll(cc);
      s->plan.chunk_bytes = chunk_bytes(s->plan.chunk,t->kmer,t->ibyte);
      s->plan.chunk_list_bytes = chunk_list_bytes(s->plan.chunk,t->kmer);
      s->plan.list_bytes = s->budget - s->plan.fixed_bytes - s->plan.chunk_bytes;
    }
  s->streamed = 1; s->host = t;
  return HM_OK;
}

/* a device's streams and timing events; its allocations come from the pool if `pool` */
static int open_device(DevTable *D, int dev, int pool)
{ int rc = HM_OK;
  cudaError_t e;
  D->dev = dev;
  TRY(cudaSetDevice(D->dev));
  D->pool = pool_setup(D->dev,pool);
  TRY(cudaStreamCreateWithFlags(&D->st,cudaStreamNonBlocking));
  TRY(cudaStreamCreateWithFlags(&D->st_copy,cudaStreamNonBlocking));
  for (int k = 0; k < 4; k++)
    TRY(cudaEventCreate(&D->ev[k]));
  return rc;
}

/* stream: 1 streams the scan whatever its size */
static int scan_create(const hm_host_table *t, const int *dev, int n_gpus, int stream, hm_scan **out)
{ double t0 = now_ms();
  if (t == NULL || out == NULL || n_gpus < 1 || n_gpus > HM_MAX_GPUS)
    return hm_set_error(HM_EINVAL,"hm_scan_create: bad arguments");
  if (t->kmer < 1 || t->kmer > HM_MAX_KMER)
    return hm_set_error(HM_EUNSUPPORTED,"k-mer length %d not supported by this build (1..%d)",
                        t->kmer,HM_MAX_KMER);
  int kbyte = (t->kmer+3)>>2;
  if (t->ibyte < 1 || t->ibyte > 3 || t->ibyte > kbyte)
    return hm_set_error(HM_EFORMAT,"table has ibyte=%d with k=%d",t->ibyte,t->kmer);
  prewarm_join();
  if (hm_device_count() < 1)
    return hm_set_error(HM_ECUDA,"no CUDA device visible (this build has no CPU fallback)");

  hm_scan *s = (hm_scan *) calloc(1,sizeof(hm_scan));
  if (s == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory");
  s->kmer = t->kmer; s->ibyte = t->ibyte; s->n = t->nels; s->ngpu = n_gpus; s->nshard = n_gpus; s->src = t;
  s->bits  = hm_pick_bucket_bits(s->n);
  s->fpos  = hm_pick_filter_bits(s->n);
  s->idx64 = (s->n >= 0xFFFFFFF0ll);
  hm_symm_seeds(s->seed);
  int64_t n  = s->n;
  size_t  ib = s->idx64 ? 8 : 4;
  int     rc = HM_OK;

  s->budget = device_budget(dev,n_gpus);
  s->incore_bytes = incore_bytes(n,t->kmer,n_gpus,s->bits,s->idx64);
  if (s->incore_bytes > s->budget || stream)
    { /* streamed: only the plot and the fingerprint sums are allocated now; the table stays on the host.
       * Several GPUs: shard r streams its run-aligned share [c_r, c_r+1) through dev[r] (DESIGN.md §4c) */
      if ((rc = stream_setup(s,t)) != HM_OK)
        { free(s); return rc; }
    }
  else
    for (int g = 0; g < n_gpus; g++)
      for (int h = 0; h < g; h++)
        if ((dev ? dev[g] : g) == (dev ? dev[h] : h))
          { free(s);
            return hm_set_error(HM_EINVAL,"GPU %d is listed twice: only a streamed scan can run several shards on one "
                                "device",dev ? dev[g] : g);
          }
  /* several GPUs: the peers map the table arrays (in core) or read the owners' S lists (streamed) */
  if (n_gpus > 1 && (rc = hm_peer_enable(dev,n_gpus)) != HM_OK)
    { free(s); return rc; }

  /* in core: table arrays + bucket index; the work buffers of either scan path are allocated by the path
   * that runs (ensure_direct / ensure_symm)                                                              */
  for (int g = 0; g < n_gpus && rc == HM_OK; g++)
    { DevTable *D = s->d+g;
      cudaError_t e;
      D->lo  = s->streamed ? 0 : n*g/n_gpus;
      D->hi  = s->streamed ? n : n*(g+1)/n_gpus;
      rc = open_device(D,dev ? dev[g] : g,n_gpus == 1);
      if (!s->streamed)
        { TRY(dev_alloc(D,&D->keys,sizeof(uint64_t)*(n+1)));
          if (t->kmer > 32)
            TRY(dev_alloc(D,&D->keys_lo,sizeof(uint64_t)*(n+1)));
          TRY(dev_alloc(D,&D->cnt,sizeof(uint16_t)*(n+8)));
          TRY(dev_alloc(D,&D->bucket,(int64_t) ib*((1ll << s->bits)+1)));
        }
      TRY(dev_alloc(D,&D->plot,sizeof(unsigned long long)*HM_PLOT_CELLS));
      TRY(dev_alloc(D,&D->fp_acc,4*sizeof(uint64_t)));
    }
  if (s->streamed)
    { if (rc == HM_OK && n_gpus > 1 && t->kmer >= HM_SYMM_MIN_KMER)   /* (smaller k: refused by the run) */
        rc = stream_cuts(s);
      if (rc != HM_OK)
        { hm_scan_destroy(s); return rc; }
      s->ms_load = now_ms()-t0;
      *out = s;
      return HM_OK;
    }

  double t_alloc = now_ms();
  /* each device unpacks its own shard from the host -- all devices at once, one host thread each --
   * then the shards are exchanged over peer copies so that every device ends with the full table */
  if (rc == HM_OK)
    rc = on_every_gpu(s,load_shard,(void *) t);
  double t_rec = now_ms();
  if (n_gpus > 1 && rc == HM_OK)
    { for (int g = 0; g < n_gpus && rc == HM_OK; g++)        /* all-gather by peer copies */
        for (int h = 0; h < n_gpus && rc == HM_OK; h++)
          if (h != g)
            { DevTable *S = s->d+h, *D = s->d+g;
              int64_t m = S->hi-S->lo;
              if (m <= 0) continue;
              cudaSetDevice(D->dev);
              cudaError_t e = cudaMemcpyPeerAsync(D->keys+S->lo,D->dev,S->keys+S->lo,S->dev,
                                                  sizeof(uint64_t)*(size_t) m,D->st);
              if (e == cudaSuccess && D->keys_lo != NULL)
                e = cudaMemcpyPeerAsync(D->keys_lo+S->lo,D->dev,S->keys_lo+S->lo,S->dev,
                                        sizeof(uint64_t)*(size_t) m,D->st);
              if (e == cudaSuccess)
                e = cudaMemcpyPeerAsync(D->cnt+S->lo,D->dev,S->cnt+S->lo,S->dev,
                                        sizeof(uint16_t)*(size_t) m,D->st);
              if (e != cudaSuccess) rc = hm_cuda_fail(e,"cudaMemcpyPeerAsync(table shard)");
            }
      int rc2 = sync_all(s,"table shards");
      if (rc == HM_OK) rc = rc2;
    }
  for (int g = 0; g < n_gpus && rc == HM_OK && n_gpus > 1; g++)     /* (one GPU: done chunk-wise) */
    { DevTable *D = s->d+g;
      cudaSetDevice(D->dev);
      rc = hm_k_build_bucket_index(D->keys,n,s->bits,D->bucket,s->idx64,D->st);
      s->launches += 1;
    }
  int rc2 = sync_all(s,"table load");
  if (rc == HM_OK) rc = rc2;
  if (rc == HM_OK)
    rc = fingerprint_verdict(s);
  if (rc != HM_OK)
    { hm_scan_destroy(s); return rc; }
  s->ms_load = now_ms()-t0;
  s->ms_alloc = t_alloc-t0; s->ms_records = t_rec-t_alloc; s->ms_index = now_ms()-t_rec;
  *out = s;
  return HM_OK;
}

extern "C" int hm_scan_create(const hm_host_table *t, const int *dev, int n_gpus, hm_scan **out)
{ const char *force = getenv("HETMERS_STREAM");            /* =1: stream whatever the budget (tests, capping) */
  return scan_create(t,dev,n_gpus,force != NULL && strcmp(force,"1") == 0,out);
}

extern "C" int hm_scan_create_streamed(const hm_host_table *t, const int *dev, int n_gpus, hm_scan **out)
{ return scan_create(t,dev,n_gpus,1,out);
}

/* work buffers of the direct passes (hm_kernels.cu): incidence array, recorded partners, prefix filter */
static int ensure_direct(hm_scan *s)
{ if (s->have_direct)
    return HM_OK;
  int64_t n  = s->n;
  size_t  ib = s->idx64 ? 8 : 4;
  int     rc = HM_OK;
  for (int g = 0; g < s->ngpu && rc == HM_OK; g++)
    { DevTable *D = s->d+g;
      cudaError_t e;
      TRY(cudaSetDevice(D->dev));
      if (D->deg == NULL)    TRY(dev_alloc(D,&D->deg,(n+4)&~3ll));
      if (D->up == NULL)     TRY(dev_alloc(D,&D->up,(int64_t) ib*(D->hi-D->lo+1)));
      if (D->filter == NULL) TRY(dev_alloc(D,&D->filter,sizeof(uint32_t)*hm_filter_words(s->fpos)));
      if (rc == HM_OK)
        rc = hm_k_build_filter(D->keys,n,s->fpos,D->filter,D->st);
      s->launches += 1;
    }
  int rc2 = sync_all(s,"prefix filter");
  if (rc == HM_OK) rc = rc2;
  if (rc == HM_OK)
    s->have_direct = 1;
  return rc;
}

/* work areas of the strand-symmetric scan (hm_symm.cu); several GPUs: cuts on run boundaries */
static int ensure_symm(hm_scan *s)
{ if (s->have_symm)
    return HM_OK;
  int     G = s->ngpu;
  int64_t n = s->n, cut[HM_MAX_GPUS+1];
  cut[0] = 0; cut[G] = n;
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  for (int g = 1; g < G; g++)
    { int rc = hm_symm_align_cut(s->d[0].keys,n,s->kmer,n*g/G,&cut[g]);
      if (rc != HM_OK) return rc;
      if (cut[g] < cut[g-1]) cut[g] = cut[g-1];
    }
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      hm_symm_shards *sh = s->ssh+g;
      memset(sh,0,sizeof(*sh));
      sh->n_seg = G; sh->self = g;
      for (int r = 0; r <= G; r++) sh->off[r] = cut[r];
      HM_CUDA(cudaSetDevice(D->dev));
      for (int r = 1; r < G; r++)
        if (cut[r] < n)
          HM_CUDA(cudaMemcpy(&sh->first_key[r],D->keys+cut[r],sizeof(uint64_t),cudaMemcpyDeviceToHost));
        else
          sh->first_key[r] = ~0ull;
      D->slo = cut[g]; D->shi = cut[g+1];
      int rc = hm_symm_plan(n,D->shi-D->slo,s->kmer,G,&D->symm_layout);
      if (rc != HM_OK) return rc;
      dev_free(D,D->symm_work);
      D->symm_work = NULL;
      HM_CUDA(dev_alloc(D,&D->symm_work,D->symm_layout.bytes));
    }
  s->have_symm = 1; s->symm_ready = 0;
  return HM_OK;
}

/* ---- conditioning (DESIGN.md §4d; kernels, settle step and plan in hm_condition.cu) --------------------------
 * One range loop, two ends.  Pass 0 histograms the output by key prefix over the source; the plan cuts the
 * prefixes into key ranges; each range is then gathered over the source's chunks and settled (sort + merge).
 * Source: the host table through the loader, a chunk at a time (hm_scan_condition_files), or the resident
 * table as one chunk (hm_scan_condition).  Sink: FastK records handed to a writer thread, or the new table's
 * device arrays at the range's offset.                                                                     */

static int cond_hist_bits(int kmer) { return 2*kmer < HM_COND_HIST_BITS ? 2*kmer : HM_COND_HIST_BITS; }

typedef struct
  { hm_scan             *s;
    DevTable            *D;
    const hm_host_table *t;                /* the host table, or NULL: the resident arrays below are the source */
    const int64_t       *d_index;          /* (host table) its stub index on the device, and the loader        */
    Stager              *G;
    uint64_t            *keys, *klo;       /* the chunk buffers (host table) or the resident table            */
    uint16_t            *cnt;
    int64_t              n, chunk;         /* source entries; entries per chunk                               */
  } CondSrc;

/* ordinals [o, o+m) of the source: loaded into the chunk buffers, or where they lie in the resident arrays */
static int cond_fetch(const CondSrc *S, int64_t o, int64_t m, const uint64_t **k, const uint64_t **l, const uint16_t **c)
{ if (S->t == NULL)
    { *k = S->keys+o; *l = S->klo ? S->klo+o : NULL; *c = S->cnt+o;
      return HM_OK;
    }
  *k = S->keys; *l = S->klo; *c = S->cnt;
  return load_into(S->s,S->D,S->t,S->d_index,o,m,S->keys,S->klo,S->cnt,0,S->G);
}

/* pass 0 over source ordinals [first, end): kept originals (+ their reverse complements) per key prefix -> hist
 * (host, 2^hb entries)                                                                                        */
static int cond_histogram(const CondSrc *S, int64_t first, int64_t end, int ethr, int do_symm, int hb,
                          unsigned long long *d_hist, int64_t *hist)
{ cudaStream_t  st = S->D->st;
  const int64_t np = (int64_t) 1 << hb;
  int           rc = HM_OK;
  HM_CUDA(cudaMemsetAsync(d_hist,0,8*(size_t) np,st));
  for (int64_t o = first; o < end && rc == HM_OK; o += S->chunk)
    { const int64_t   m = end-o < S->chunk ? end-o : S->chunk;
      const uint64_t *k, *l;
      const uint16_t *c;
      rc = cond_fetch(S,o,m,&k,&l,&c);
      if (rc == HM_OK) rc = hm_cond_hist(k,l,c,m,S->s->kmer,ethr,do_symm,hb,d_hist,st);
    }
  if (rc != HM_OK)
    return rc;
  HM_CUDA(cudaMemcpyAsync(hist,d_hist,8*(size_t) np,cudaMemcpyDeviceToHost,st));
  HM_CUDA(cudaStreamSynchronize(st));
  return HM_OK;
}

/* the range [p0, p1) of key prefixes gathered over the source's chunks into B and settled; *n_r: its entries */
static int cond_range(const CondSrc *S, const hm_cond_bufs *B, uint64_t p0, uint64_t p1, unsigned long long *tiles,
                      int64_t *n_r)
{ cudaStream_t st = S->D->st;
  int          rc = HM_OK;
  HM_CUDA(cudaMemsetAsync(B->ctr,0,256,st));
  for (int64_t o = 0; o < S->n && rc == HM_OK; o += S->chunk)
    { const int64_t   m = S->n-o < S->chunk ? S->n-o : S->chunk;
      const uint64_t *k, *l;
      const uint16_t *c;
      rc = cond_fetch(S,o,m,&k,&l,&c);
      if (rc == HM_OK) rc = hm_cond_gather(k,l,c,m,B,p0,p1,tiles,st);
    }
  return rc != HM_OK ? rc : hm_cond_settle(B,n_r,st);
}

/* ---- in place --------------------------------------------------------------------------------------------- */

/* device bytes of the in-place conditioning of a range of t output entries: the region its originals and
 * reverse complements are gathered into and, when symmetrising, the sort's other buffers (+ the uint32
 * permutation pair at k > 32), CUB's scratch bound and the merge's tile counts.  The range settles straight
 * into the new table's arrays: no records, no merged copy.                                                 */
static int64_t in_place_range_bytes(int64_t t, int do_symm, int kmer, int ibyte)
{ const int64_t E = kmer > 32 ? 18 : 10;
  (void) ibyte;
  if (t < 1) t = 1;
  return E*t + (do_symm ? E*t + (kmer > 32 ? 8*t : 0) + hm_cond_sort_room(t) + 2*hm_cond_tiles_bytes(t) : 0);
}

typedef struct
  { int      ethr, do_symm, hb, n_ranges;
    int64_t *cuts;                         /* key-prefix bounds of the ranges                              */
    int64_t  out_cap;                      /* entries of each new array: the histogram's total (an upper   */
                                           /*   bound: duplicates go) or, trimming only, n; plus one       */
    int64_t  range_cap;                    /* entries of the largest range                                 */
  } InPlace;

/* one GPU's replica conditioned into new arrays of P->out_cap entries, which replace D's only when every range
 * has settled; every allocation goes through dev_alloc, and the temporaries are gone on return             */
static int condition_replica(hm_scan *s, DevTable *D, const InPlace *P, int64_t *n_out)
{ const int     two = s->kmer > 32;
  const int64_t cap = P->out_cap, T = P->do_symm ? (P->range_cap > 0 ? P->range_cap : 1) : cap;
  CondSrc S;
  memset(&S,0,sizeof(S));
  S.s = s; S.D = D; S.keys = D->keys; S.klo = D->keys_lo; S.cnt = D->cnt;
  S.n = s->n; S.chunk = s->n > 0 ? s->n : 1;
  hm_cond_bufs B;
  memset(&B,0,sizeof(B));
  B.kmer = s->kmer; B.ibyte = s->ibyte; B.hb = P->hb; B.ethresh = P->ethr; B.do_symm = P->do_symm; B.cap = T;
  uint64_t *nk = NULL, *nl = NULL;
  uint16_t *nc = NULL;
  unsigned long long *tiles = NULL;
  int       rc = HM_OK;
  cudaError_t e;
  TRY(dev_alloc(D,&nk,8*cap));
  if (two) TRY(dev_alloc(D,&nl,8*cap));
  TRY(dev_alloc(D,&nc,2*cap));
  TRY(dev_alloc(D,&B.ctr,256));
  TRY(dev_alloc(D,&tiles,hm_cond_tiles_bytes(S.n)));
  if (!P->do_symm)                                         /* the kept originals are the new table */
    { B.key = nk; B.lo = nl; B.cnt = nc; }
  else
    { TRY(dev_alloc(D,&B.key,8*T));
      if (two) TRY(dev_alloc(D,&B.lo,8*T));
      TRY(dev_alloc(D,&B.cnt,2*T));
      TRY(dev_alloc(D,&B.alt_key,8*T));
      TRY(dev_alloc(D,&B.alt_cnt,2*T));
      if (two)
        { TRY(dev_alloc(D,&B.alt_lo,8*T));
          TRY(dev_alloc(D,&B.idx[0],4*T));
          TRY(dev_alloc(D,&B.idx[1],4*T));
        }
      TRY(dev_alloc(D,&B.mtiles,2*hm_cond_tiles_bytes(T)));
      B.sort_bytes = hm_cond_sort_room(T);
      TRY(dev_alloc(D,&B.sort_tmp,B.sort_bytes));
    }
  int64_t out = 0;
  for (int r = 0; r < P->n_ranges && rc == HM_OK; r++)
    { int64_t n_r = 0;
      if (P->do_symm)                                      /* the range's place in the new table */
        { B.m_key = nk+out; B.m_lo = two ? nl+out : NULL; B.m_cnt = nc+out; }
      rc = cond_range(&S,&B,(uint64_t) P->cuts[r],(uint64_t) P->cuts[r+1],tiles,&n_r);
      s->launches += 3 + (P->do_symm ? 6 : 0);
      out += n_r;
    }
  void *tmp[] = { B.ctr, tiles, B.alt_key, B.alt_cnt, B.alt_lo, B.idx[0], B.idx[1], B.mtiles, B.sort_tmp,
                  P->do_symm ? B.key : NULL, P->do_symm ? B.lo : NULL, P->do_symm ? B.cnt : NULL };
  for (size_t k = 0; k < sizeof(tmp)/sizeof(tmp[0]); k++)
    dev_free(D,tmp[k]);
  void *drop[3] = { nk, nl, nc };
  if (rc == HM_OK)                                         /* the new table replaces the old one */
    { drop[0] = D->keys; drop[1] = D->keys_lo; drop[2] = D->cnt;
      D->keys = nk; D->keys_lo = nl; D->cnt = nc;
    }
  for (int a = 0; a < 3; a++)
    dev_free(D,drop[a]);
  *n_out = out;
  return rc;
}

/* Trim (count >= ethresh) and / or symmetrise (add reverse complements) the device-resident table in place:
 * what the reference gets from `Logex` and `Symmex` (PloidyPlot.c:1381-1426), without leaving the GPU.  The
 * replicas are identical, so GPU 0 histograms the output and the plan is every GPU's; each GPU then conditions
 * its own replica through the range passes, and the index structures and work buffers are rebuilt for the
 * new size.  The plan is checked against the budget before anything is touched.                          */
extern "C" int hm_scan_condition(hm_scan *s, int ethresh, int do_trim, int do_symm, int64_t *nels_out)
{ int     G = s->ngpu, rc = HM_OK;
  int64_t n_new = -1;
  if (s->invalid)
    return hm_set_error(HM_EINVAL,"this scan was left unusable by an earlier failed conditioning");
  if (!do_trim && !do_symm)
    { if (nels_out) *nels_out = s->n;
      return HM_OK;
    }
  if (s->streamed)
    return hm_set_error(HM_EUNSUPPORTED,"conditioning on the GPU needs the table resident; this one does not fit in "
                                        "device memory (budget %lld bytes)",(long long) s->budget);
  InPlace P;
  memset(&P,0,sizeof(P));
  P.ethr = do_trim ? ethresh : 0; P.do_symm = do_symm; P.hb = cond_hist_bits(s->kmer);
  const int64_t np = (int64_t) 1 << P.hb;
  int64_t whole[2] = { 0, np }, *hist = NULL, big = 0, total = s->n;
  P.cuts = whole; P.n_ranges = 1; P.range_cap = s->n;
  if (do_symm)                                             /* pass 0 on GPU 0: the output histogram */
    { DevTable *D = s->d;
      unsigned long long *d_hist = NULL;
      cudaError_t e;
      hist = (int64_t *) malloc(sizeof(int64_t)*(size_t) np);
      P.cuts = (int64_t *) malloc(sizeof(int64_t)*(size_t) (np+1));
      if (hist == NULL || P.cuts == NULL)
        { free(hist); free(P.cuts); return hm_set_error(HM_ENOMEM,"out of host memory"); }
      CondSrc S;
      memset(&S,0,sizeof(S));
      S.s = s; S.D = D; S.keys = D->keys; S.klo = D->keys_lo; S.cnt = D->cnt; S.n = s->n; S.chunk = s->n > 0 ? s->n : 1;
      TRY(cudaSetDevice(D->dev));
      TRY(dev_alloc(D,&d_hist,8*np));
      if (rc == HM_OK) rc = cond_histogram(&S,0,s->n,P.ethr,1,P.hb,d_hist,hist);
      dev_free(D,d_hist);
      s->launches += 1;
      total = 0;
      for (int64_t p = 0; p < np; p++) total += hist[p];
    }
  P.out_cap = total + 1;
  /* what each GPU holds meanwhile: its table and what stays of the scan (the index and work buffers go), the
   * new arrays, the counters and the chunk's tile counts, and the working set of the largest range          */
  int64_t held = 0;
  for (int g = 0; g < G; g++)
    { const DevTable *D = s->d+g;
      int64_t h = D->held - dev_bytes(D,D->deg) - dev_bytes(D,D->up) - dev_bytes(D,D->bucket) -
                  dev_bytes(D,D->filter) - dev_bytes(D,D->symm_work);
      if (h > held) held = h;
    }
  const int64_t fixed = held + (s->kmer > 32 ? 18 : 10)*P.out_cap + 256 + hm_cond_tiles_bytes(s->n);
  int64_t need = fixed, one = fixed;
  if (rc == HM_OK && do_symm)
    { const int64_t limit = hm_cond_range_limit(s->budget-fixed,in_place_range_bytes,1,s->kmer,s->ibyte);
      P.n_ranges = hm_cond_cut(hist,np,limit,P.cuts,&P.range_cap,&big);
      need += in_place_range_bytes(big,1,s->kmer,s->ibyte);
      one  += in_place_range_bytes(total,1,s->kmer,s->ibyte);
    }
  free(hist);
  if (rc == HM_OK && (P.n_ranges < 1 || need > s->budget))
    rc = hm_set_error(HM_ENOMEM,"conditioning %lld entries on the GPU needs %lld device bytes (%lld in one range), more "
                      "than the budget of %lld",(long long) s->n,(long long) need,(long long) one,(long long) s->budget);
  if (rc != HM_OK)
    { if (P.cuts != whole) free(P.cuts);
      return rc;
    }

  /* everything derived from the old table goes first: work buffers of both paths, the index */
  s->conditioned = 1;
  s->ran = 0; s->have_direct = 0; s->have_symm = 0; s->symm_ready = 0;
  if ((rc = sync_all(s,"conditioning")) != HM_OK)
    { if (P.cuts != whole) free(P.cuts);
      return rc;
    }
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      cudaSetDevice(D->dev);
      dev_free(D,D->deg);    D->deg = NULL;
      dev_free(D,D->up);     D->up = NULL;
      dev_free(D,D->bucket); D->bucket = NULL;
      dev_free(D,D->filter); D->filter = NULL;
      dev_free(D,D->symm_work); D->symm_work = NULL;
    }
  for (int g = 0; g < G && rc == HM_OK; g++)
    { DevTable *D = s->d+g;
      int64_t   n = 0;
      cudaError_t e;
      TRY(cudaSetDevice(D->dev));
      if (rc == HM_OK)
        rc = condition_replica(s,D,&P,&n);
      if (rc == HM_OK && n_new >= 0 && n != n_new)
        rc = hm_set_error(HM_ECUDA,"conditioning gave %lld entries on GPU %d but %lld on GPU 0",
                          (long long) n,D->dev,(long long) n_new);
      if (rc != HM_OK && g > 0)
        s->invalid = 1;                        /* the replicas no longer agree */
      n_new = n;
    }
  if (P.cuts != whole) free(P.cuts);
  if (rc == HM_OK)
    { s->n     = n_new;
      s->bits  = hm_pick_bucket_bits(s->n);
      s->fpos  = hm_pick_filter_bits(s->n);
      s->idx64 = (s->n >= 0xFFFFFFF0ll);
    }
  /* index (also after a failure on GPU 0: the old table is intact and stays usable) */
  size_t ib = s->idx64 ? 8 : 4;
  int    rc_cond = rc;
  rc = HM_OK;
  for (int g = 0; g < G && rc == HM_OK && !s->invalid; g++)
    { DevTable *D = s->d+g;
      int64_t   n = s->n;
      cudaError_t e;
      D->lo = n*g/G;
      D->hi = n*(g+1)/G;
      TRY(cudaSetDevice(D->dev));
      TRY(dev_alloc(D,&D->bucket,(int64_t) ib*((1ll << s->bits)+1)));
      TRY(cudaMemsetAsync(D->fp_acc,0,4*sizeof(uint64_t),D->st));
      if (rc == HM_OK)
        rc = hm_k_build_bucket_index(D->keys,n,s->bits,D->bucket,s->idx64,D->st);
      if (rc == HM_OK && s->kmer >= HM_SYMM_MIN_KMER)
        rc = hm_k_symm_fingerprint(D->keys,D->keys_lo,D->cnt,D->lo,D->hi,s->kmer,s->seed,D->fp_acc,D->st);
      s->launches += 2;
    }
  int rc_sync = sync_all(s,"re-index after conditioning");
  if (rc == HM_OK) rc = rc_sync;
  if (rc == HM_OK && !s->invalid)
    rc = fingerprint_verdict(s);
  if (rc != HM_OK)
    s->invalid = 1;
  if (nels_out) *nels_out = s->n;
  return rc_cond != HM_OK ? rc_cond : rc;
}

/* ---- into table files ------------------------------------------------------------------------------------ */

/* 1 if the table `dst` would be written over holds one of the source's part files */
static int names_source(const hm_host_table *t, const char *dst)
{ hm_table *d = NULL;
  int       same = 0;
  if (t->part_fd == NULL || hm_table_open(dst,&d) != HM_OK)
    return 0;
  const hm_host_table *v = hm_table_view(d);
  for (int p = 0; p < v->nparts && !same; p++)
    for (int q = 0; q < t->nparts && !same; q++)
      { struct stat a, b;
        if (v->part_fd[p] >= 0 && t->part_fd[q] >= 0 && fstat(v->part_fd[p],&a) == 0 && fstat(t->part_fd[q],&b) == 0)
          same = (a.st_dev == b.st_dev && a.st_ino == b.st_ino);
      }
  hm_table_close(d);
  return same;
}

/* one range's records, from the device to the table files on a host thread: pinned pieces, the copy of the next
 * piece overlapping the write of this one.  Appended (one GPU: the thread announces the buckets first), or
 * written at the ordinal the range was placed at (several GPUs)                                             */
typedef struct
  { int             dev, pbyte, rc, positional;
    hm_table_writer *w;
    const uint8_t  *d_rec;
    int64_t         n, b0, nb, *counts, pin_bytes, first;
    uint8_t        *pin[2];
    cudaStream_t    st;
    double          ms;
    char            msg[512];
  } WriteJob;

static void *write_worker(void *p)
{ WriteJob *J = (WriteJob *) p;
  double    t0 = now_ms();
  int64_t   per = J->pin_bytes/J->pbyte;
  cudaError_t e = cudaSetDevice(J->dev);
  J->rc = e != cudaSuccess ? hm_cuda_fail(e,"writer thread")
                           : J->positional ? HM_OK : hm_table_write_buckets(J->w,J->b0,J->nb,J->counts);
  if (J->rc == HM_OK && J->n > 0)
    { e = cudaMemcpyAsync(J->pin[0],J->d_rec,(size_t) ((J->n < per ? J->n : per)*J->pbyte),cudaMemcpyDeviceToHost,J->st);
      for (int64_t o = 0, i = 0; o < J->n && J->rc == HM_OK; o += per, i++)
        { int64_t m = J->n-o < per ? J->n-o : per;
          if (e == cudaSuccess) e = cudaStreamSynchronize(J->st);
          if (e == cudaSuccess && o+per < J->n)
            { int64_t m2 = J->n-o-per < per ? J->n-o-per : per;
              e = cudaMemcpyAsync(J->pin[(i+1)&1],J->d_rec+(o+per)*J->pbyte,(size_t) (m2*J->pbyte),cudaMemcpyDeviceToHost,J->st);
            }
          if (e != cudaSuccess) { J->rc = hm_cuda_fail(e,"records to the host"); break; }
          J->rc = J->positional ? hm_table_write_at(J->w,J->first+o,J->pin[i&1],m)
                                : hm_table_write_append(J->w,J->pin[i&1],m);
        }
      cudaStreamSynchronize(J->st);
    }
  if (J->rc != HM_OK)
    { strncpy(J->msg,hm_last_error(),sizeof(J->msg)-1); J->msg[sizeof(J->msg)-1] = 0; }
  J->ms += now_ms()-t0;
  return NULL;
}

static int g_cond_gpus = 1;

extern "C" int hm_set_condition_gpus(int n)
{ const int was = g_cond_gpus;
  g_cond_gpus = n > 1 ? n : 1;
  return was;
}

/* what one GPU of hm_scan_condition_files holds: its source (the host table through its own loader, or its
 * resident replica), the fixed part and the range buffers, and its writer thread                           */
typedef struct
  { DevTable           *D;
    CondSrc             src;
    hm_cond_bufs        B;
    int64_t            *d_index;
    uint64_t           *ck, *cl;
    uint16_t           *cc;
    unsigned long long *d_hist, *tiles;
    Stager              G;
    WriteJob            J;
    pthread_t           th;
    int                 writing;
    int64_t            *hist, *hcnt;      /* host: this GPU's share of the histogram; a range's bucket counts */
    int64_t             held0, peak0, out, ranges;
    int                 rc;
    char                msg[512];
  } CondGpu;

typedef struct
  { CondGpu        *gpu;
    int             n_gpus, ethr, do_symm, hb, ibyte;
    int64_t         n, n_ranges, *cuts;
    hm_table_writer *w;
    pthread_mutex_t mu;                    /* (several GPUs) ranges are placed in order: `next` is due       */
    pthread_cond_t  cv;
    int64_t         next;
    volatile int    stop;                  /* a GPU failed: the others leave at their next range             */
  } CondRun;

/* GPU g's share of the source: the fixed part (stub index, bucket counts, histogram, counters) and the chunk
 * buffers + loader, or (resident) tile counts for chunks of its replica                                      */
static int cond_gpu_open(hm_scan *s, CondGpu *C, DevTable *D, const hm_host_table *t, int resident, int64_t chunk,
                         int np_bits, int ethr, int do_symm)
{ const int64_t ixlen = (int64_t) 1 << (8*t->ibyte), np = (int64_t) 1 << np_bits;
  int rc = HM_OK;
  cudaError_t e;
  C->D = D;
  HM_CUDA(cudaSetDevice(D->dev));
  C->held0 = D->held; C->peak0 = D->peak;
  D->peak = D->held;
  C->B.kmer = s->kmer; C->B.ibyte = t->ibyte; C->B.hb = np_bits; C->B.ethresh = ethr; C->B.do_symm = do_symm;
  C->hist = (int64_t *) calloc((size_t) np,sizeof(int64_t));
  C->hcnt = (int64_t *) malloc(sizeof(int64_t)*(size_t) ixlen);
  if (C->hist == NULL || C->hcnt == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory");
  if (!resident) TRY(dev_alloc(D,&C->d_index,8*ixlen));
  TRY(dev_alloc(D,&C->B.bcount,8*ixlen));
  TRY(dev_alloc(D,&C->d_hist,8*np));
  TRY(dev_alloc(D,&C->B.ctr,256));
  if (!resident)
    { TRY(dev_alloc(D,&C->ck,8*(chunk+1)));
      if (s->kmer > 32) TRY(dev_alloc(D,&C->cl,8*(chunk+1)));
      TRY(dev_alloc(D,&C->cc,2*(chunk+8)));
    }
  TRY(dev_alloc(D,&C->tiles,hm_cond_tiles_bytes(chunk)));
  if (!resident)
    { TRY(cudaMemcpyAsync(C->d_index,t->index,8*(size_t) ixlen,cudaMemcpyHostToDevice,D->st));
      if (rc == HM_OK)
        rc = stager_open(s,D,t,chunk,&C->G);
      C->src.t = t; C->src.d_index = C->d_index; C->src.G = &C->G;
      C->src.keys = C->ck; C->src.klo = C->cl; C->src.cnt = C->cc;
    }
  else
    { C->src.keys = D->keys; C->src.klo = D->keys_lo; C->src.cnt = D->cnt; }
  C->src.s = s; C->src.D = D; C->src.n = t->nels; C->src.chunk = chunk;
  return rc;
}

/* the range buffers, sized for the largest range */
static int cond_gpu_range_bufs(CondGpu *C, int64_t T, int pbyte)
{ DevTable *D = C->D;
  hm_cond_bufs *B = &C->B;
  const int two = B->kmer > 32;
  int rc = HM_OK;
  cudaError_t e;
  B->cap = T;
  TRY(cudaSetDevice(D->dev));
  TRY(dev_alloc(D,&B->key,8*T));
  if (two) TRY(dev_alloc(D,&B->lo,8*T));
  TRY(dev_alloc(D,&B->cnt,2*T));
  TRY(dev_alloc(D,&B->rec,pbyte*T));
  if (B->do_symm)
    { TRY(dev_alloc(D,&B->alt_key,8*T));
      TRY(dev_alloc(D,&B->alt_cnt,2*T));
      TRY(dev_alloc(D,&B->m_key,8*T));
      TRY(dev_alloc(D,&B->m_cnt,2*T));
      if (two)
        { TRY(dev_alloc(D,&B->alt_lo,8*T));
          TRY(dev_alloc(D,&B->m_lo,8*T));
          TRY(dev_alloc(D,&B->idx[0],4*T));
          TRY(dev_alloc(D,&B->idx[1],4*T));
        }
      TRY(dev_alloc(D,&B->mtiles,2*hm_cond_tiles_bytes(T)));
      B->sort_bytes = hm_cond_sort_room(T);
      TRY(dev_alloc(D,&B->sort_tmp,B->sort_bytes));
    }
  if (rc == HM_OK)
    { C->J.dev = D->dev; C->J.pbyte = pbyte; C->J.d_rec = B->rec;
      C->J.pin_bytes = (int64_t) pbyte*((64ll << 20)/pbyte);
      TRY(cudaStreamCreateWithFlags(&C->J.st,cudaStreamNonBlocking));
      TRY(cudaHostAlloc(&C->J.pin[0],(size_t) C->J.pin_bytes,cudaHostAllocDefault));
      TRY(cudaHostAlloc(&C->J.pin[1],(size_t) C->J.pin_bytes,cudaHostAllocDefault));
    }
  return rc;
}

/* everything GPU C allocated goes; the scan's own residency report is left as it was */
static void cond_gpu_close(CondGpu *C)
{ DevTable *D = C->D;
  hm_cond_bufs *B = &C->B;
  if (D == NULL)
    return;
  cudaSetDevice(D->dev);
  stager_close(D,&C->G);
  cudaStreamSynchronize(D->st);
  void *mine[] = { C->d_index, B->bcount, C->d_hist, B->ctr, C->ck, C->cl, C->cc, C->tiles, B->key, B->lo, B->cnt,
                   B->rec, B->alt_key, B->alt_cnt, B->m_key, B->m_cnt, B->alt_lo, B->m_lo, B->idx[0], B->idx[1],
                   B->mtiles, B->sort_tmp };
  for (size_t k = 0; k < sizeof(mine)/sizeof(mine[0]); k++)
    dev_free(D,mine[k]);
  cudaStreamSynchronize(D->st);
  if (C->J.st) cudaStreamDestroy(C->J.st);
  if (C->J.pin[0]) cudaFreeHost(C->J.pin[0]);
  if (C->J.pin[1]) cudaFreeHost(C->J.pin[1]);
  D->peak = C->peak0 > D->held ? C->peak0 : D->held;
  free(C->hist); free(C->hcnt);
}

/* pass 0 on GPU g: its contiguous slice of the source ordinals */
static int cond_gpu_hist(CondRun *R, int g)
{ CondGpu *C = R->gpu+g;
  HM_CUDA(cudaSetDevice(C->D->dev));
  return cond_histogram(&C->src,R->n*g/R->n_gpus,R->n*(g+1)/R->n_gpus,R->ethr,R->do_symm,R->hb,C->d_hist,C->hist);
}

static int writer_join(CondGpu *C)
{ if (!C->writing)
    return HM_OK;
  pthread_join(C->th,NULL);
  C->writing = 0;
  return C->J.rc != HM_OK ? hm_set_error(C->J.rc,"%s",C->J.msg) : HM_OK;
}

/* the other GPUs stop at their next range; those waiting to place theirs are let go */
static void cond_stop(CondRun *R)
{ pthread_mutex_lock(&R->mu);
  R->stop = 1;
  pthread_cond_broadcast(&R->cv);
  pthread_mutex_unlock(&R->mu);
}

/* passes 1..R on GPU g: ranges g, g + G, ...  One GPU appends; several place each range once every earlier one is
 * placed (placing waits only for the placing of the range before, never for a write), then write it at its
 * offsets                                                                                                     */
static int cond_gpu_ranges(CondRun *R, int g)
{ CondGpu      *C = R->gpu+g;
  DevTable     *D = C->D;
  const int     hb = R->hb, ibyte = R->ibyte, several = R->n_gpus > 1;
  int           rc = HM_OK;
  cudaError_t   e;
  TRY(cudaSetDevice(D->dev));
  for (int64_t r = g; r < R->n_ranges && rc == HM_OK && !R->stop; r += R->n_gpus)
    { const uint64_t p0 = (uint64_t) R->cuts[r], p1 = (uint64_t) R->cuts[r+1];
      int64_t n_r = 0;
      rc = cond_range(&C->src,&C->B,p0,p1,C->tiles,&n_r);
      /* the stub buckets the range's keys fall in */
      const uint64_t b0 = 8*ibyte >= hb ? p0 << (8*ibyte-hb) : p0 >> (hb-8*ibyte);
      const uint64_t b1 = 8*ibyte >= hb ? p1 << (8*ibyte-hb) : ((p1-1) >> (hb-8*ibyte)) + 1;
      const int rw = writer_join(C);                            /* the last range's records have left B.rec */
      if (rc == HM_OK) rc = rw;
      if (rc == HM_OK) rc = hm_cond_pack(&C->B,n_r,b0,(int64_t) (b1-b0),D->st);
      TRY(cudaMemcpyAsync(C->hcnt,C->B.bcount,8*(size_t) (b1-b0),cudaMemcpyDeviceToHost,D->st));
      TRY(cudaStreamSynchronize(D->st));
      C->J.n = n_r; C->J.b0 = (int64_t) b0; C->J.nb = (int64_t) (b1-b0); C->J.counts = C->hcnt;
      if (rc == HM_OK && several)
        { pthread_mutex_lock(&R->mu);
          while (R->next != r && !R->stop)
            pthread_cond_wait(&R->cv,&R->mu);
          if (!R->stop)
            { rc = hm_table_write_place(R->w,C->J.b0,C->J.nb,C->hcnt,&C->J.first);
              R->next = r+1;
            }
          pthread_cond_broadcast(&R->cv);
          pthread_mutex_unlock(&R->mu);
          if (R->stop && rc == HM_OK)
            break;
        }
      if (rc == HM_OK)
        { C->J.positional = several;
          C->out += n_r;
          if (pthread_create(&C->th,NULL,write_worker,&C->J) == 0) C->writing = 1;
          else                                                  write_worker(&C->J);
          if (!C->writing && C->J.rc != HM_OK) rc = hm_set_error(C->J.rc,"%s",C->J.msg);
        }
      C->ranges++;
    }
  if (rc != HM_OK && several)
    cond_stop(R);
  const int rw = writer_join(C);
  return rc != HM_OK ? rc : rw;
}

typedef int (*CondFn)(CondRun *R, int g);
typedef struct { CondRun *R; CondFn fn; int g; } CondTask;

static void *cond_worker(void *p)
{ CondTask *T = (CondTask *) p;
  CondGpu  *C = T->R->gpu+T->g;
  C->rc = T->fn(T->R,T->g);
  if (C->rc != HM_OK)
    { strncpy(C->msg,hm_last_error(),sizeof(C->msg)-1); C->msg[sizeof(C->msg)-1] = 0; }
  return NULL;
}

/* fn on every GPU of the call at once, a host thread each (the calling thread takes the last); the first
 * failing GPU's error, naming it when there are several.  The GPUs wait for each other (ranges are placed in
 * order), so one cannot run after another: a thread that cannot be started stops the call.                  */
static int cond_on_gpus(CondRun *R, CondFn fn)
{ const int G = R->n_gpus;
  CondTask  task[HM_MAX_GPUS];
  pthread_t th[HM_MAX_GPUS];
  int       made = 0, rc = HM_OK;
  if (G == 1)
    return fn(R,0);
  for (int g = 0; g < G; g++)
    { task[g].R = R; task[g].fn = fn; task[g].g = g;
      R->gpu[g].rc = HM_OK;
    }
  while (made < G-1 && pthread_create(th+made,NULL,cond_worker,task+made) == 0)
    made++;
  if (made == G-1)
    cond_worker(task+G-1);
  else
    { cond_stop(R);
      rc = hm_set_error(HM_ENOMEM,"conditioning on %d GPUs: cannot start the host thread of GPU %d",G,made);
    }
  for (int g = 0; g < made; g++)
    pthread_join(th[g],NULL);
  for (int g = 0; g < G && rc == HM_OK; g++)
    if (R->gpu[g].rc != HM_OK)
      rc = hm_set_error(R->gpu[g].rc,"conditioning on GPU %d (%d of %d): %s",R->gpu[g].D->dev,g,G,R->gpu[g].msg);
  return rc;
}

/* hm_scan_condition_files (dst) and hm_scan_condition_host (out, dst NULL): one plan and one set of range passes,
 * the writer's target the only difference                                                                      */
static int condition_into(hm_scan *s, int ethresh, int do_trim, int do_symm, const char *dst, int64_t host_budget,
                          hm_host_table **out, hm_condition_stats *st)
{ double t0 = now_ms();
  const char *who = dst != NULL ? "hm_scan_condition_files" : "hm_scan_condition_host";
  if (s == NULL || (dst == NULL && out == NULL))
    return hm_set_error(HM_EINVAL,"%s: NULL argument",who);
  if (out != NULL)
    *out = NULL;
  if (s->conditioned || s->invalid)
    return hm_set_error(HM_EINVAL,"this scan's table was conditioned in place: the files it was created from no longer "
                        "describe it");
  if (!do_trim && !do_symm)
    return hm_set_error(HM_EINVAL,"%s: neither trimming nor symmetrising was asked for",who);
  const hm_host_table *t = s->src;
  if (dst != NULL && names_source(t,dst))
    return hm_set_error(HM_EINVAL,"%s names the source table: conditioning writes a new table",dst);

  const int G = g_cond_gpus < s->ngpu ? g_cond_gpus : s->ngpu;
  const int resident = G > 1 && !s->streamed;     /* several GPUs of an in-core scan read their replicas */
  const int kmer = s->kmer, ibyte = t->ibyte;
  const int pbyte = ((kmer+3)>>2) - ibyte + 2;
  const int hb = cond_hist_bits(kmer);
  const int64_t n = t->nels, np = (int64_t) 1 << hb, ixlen = (int64_t) 1 << (8*ibyte);
  const int ethr = do_trim ? ethresh : 0;
  int       rc = HM_OK;
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  /* what the call may hold on each GPU: an explicit budget covers the scan too (as hm_scan_condition counts its
   * table), so the scan's resident arrays come off it; the default one is free memory, which already excludes
   * them.  The plan takes the smallest.                                                                      */
  int dev[HM_MAX_GPUS] = { 0 };
  for (int g = 0; g < G; g++) dev[g] = s->d[g].dev;
  int64_t budget = g_budget > 0 ? g_budget - s->d[0].held : device_budget(dev,G);
  for (int g = 1; g < G && g_budget > 0; g++)
    if (g_budget - s->d[g].held < budget) budget = g_budget - s->d[g].held;

  hm_condition_stats S;
  memset(&S,0,sizeof(S));
  S.nels_in = n;
  S.budget_bytes = budget;
  S.gpus = G;
  hm_condition_layout lay;
  int64_t *hist = (int64_t *) calloc((size_t) np,sizeof(int64_t));
  int64_t *cuts = (int64_t *) malloc(sizeof(int64_t)*(size_t) (np+1));
  CondGpu *gpu  = (CondGpu *) calloc((size_t) G,sizeof(CondGpu));
  if (hist == NULL || cuts == NULL || gpu == NULL)
    { free(hist); free(cuts); free(gpu); return hm_set_error(HM_ENOMEM,"out of host memory"); }
  /* the fixed part and a chunk must fit before the source is read (an empty histogram asks nothing more) */
  if ((rc = hm_condition_plan(n,kmer,ibyte,budget,do_symm,hist,hb,cuts,&lay)) != HM_OK)
    { free(hist); free(cuts); free(gpu); return rc; }

  CondRun R;
  memset(&R,0,sizeof(R));
  R.gpu = gpu; R.n_gpus = G; R.ethr = ethr; R.do_symm = do_symm; R.hb = hb; R.ibyte = ibyte; R.n = n;
  R.cuts = cuts;
  pthread_mutex_init(&R.mu,NULL);
  pthread_cond_init(&R.cv,NULL);
  for (int g = 0; g < G && rc == HM_OK; g++)
    rc = cond_gpu_open(s,gpu+g,s->d+g,t,resident,lay.chunk,hb,ethr,do_symm);

  /* pass 0: the output histogram, a slice of the source per GPU */
  if (rc == HM_OK)
    rc = cond_on_gpus(&R,cond_gpu_hist);
  for (int g = 0; g < G && rc == HM_OK; g++)
    for (int64_t p = 0; p < np; p++) hist[p] += gpu[g].hist[p];
  S.ms_hist = now_ms()-t0;
  if (rc == HM_OK)
    rc = hm_condition_plan(n,kmer,ibyte,budget,do_symm,hist,hb,cuts,&lay);
  int64_t hint = 0;
  for (int64_t p = 0; p < np; p++) hint += hist[p];

  /* into host memory: the histogram bounds the records (settling merges an original with an equal reverse
   * complement, a palindrome with itself), and the buffer is checked and allocated before the first range pass */
  const int64_t host_need = hint*pbyte + 8*ixlen;
  if (rc == HM_OK && dst == NULL && host_budget >= 0 && host_need > host_budget)
    rc = hm_set_error(HM_ENOMEM,"conditioning into host memory needs %lld host bytes (%lld records of %d bytes and a "
                      "stub index of %lld), beyond the host budget of %lld",(long long) host_need,(long long) hint,
                      pbyte,(long long) (8*ixlen),(long long) host_budget);
  const int minval = do_trim && ethresh > t->minval ? ethresh : t->minval;
  if (rc == HM_OK && dst == NULL)
    rc = hm_table_write_open_host(kmer,ibyte,minval,hint,&R.w);
  const int64_t T = lay.range_cap > 0 ? lay.range_cap : 1;
  for (int g = 0; g < G && rc == HM_OK; g++)
    rc = cond_gpu_range_bufs(gpu+g,T,pbyte);
  if (rc == HM_OK && dst != NULL)
    rc = hm_table_write_open(dst,kmer,ibyte,minval,t->nparts > 0 ? t->nparts : 1,hint,&R.w);
  for (int g = 0; g < G; g++)
    gpu[g].J.w = R.w;

  /* passes 1..R: a key range each */
  double t_ranges = now_ms();
  R.n_ranges = lay.n_ranges;
  if (rc == HM_OK)
    rc = cond_on_gpus(&R,cond_gpu_ranges);
  S.ms_ranges = now_ms()-t_ranges;
  if (R.w != NULL)
    { int rw = rc != HM_OK ? (hm_table_write_abort(R.w), HM_OK)
             : dst != NULL ? hm_table_write_close(R.w) : hm_table_write_close_host(R.w,out);
      if (rc == HM_OK) rc = rw;
    }

  for (int g = 0; g < G; g++)
    { CondGpu *C = gpu+g;
      if (C->D != NULL)
        { const int64_t peak = C->D->peak - C->held0;
          if (peak > S.peak_bytes) S.peak_bytes = peak;
          if (g < HM_COND_MAX_GPUS) S.gpu_peak_bytes[g] = peak;
        }
      S.nels_out += C->out;
      S.ranges += (int32_t) C->ranges;
      S.ms_write += C->J.ms;
      if (C->J.ms > S.ms_write_max) S.ms_write_max = C->J.ms;
      cond_gpu_close(C);
    }
  pthread_mutex_destroy(&R.mu);
  pthread_cond_destroy(&R.cv);
  free(hist); free(cuts); free(gpu);
  S.passes = S.ranges+1;
  S.bytes_read = resident ? 0 : (int64_t) S.passes*n*pbyte;
  S.bytes_written = dst != NULL ? 16 + 8*ixlen + 12ll*(t->nparts > 0 ? t->nparts : 1) + S.nels_out*pbyte
                                 : rc == HM_OK ? 8*ixlen + S.nels_out*pbyte : 0;   /* host bytes held */
  S.ms_total = now_ms()-t0;
  if (st != NULL) *st = S;
  return rc;
}

extern "C" int hm_scan_condition_files(hm_scan *s, int ethresh, int do_trim, int do_symm, const char *dst,
                                       hm_condition_stats *st)
{ if (dst == NULL)
    return hm_set_error(HM_EINVAL,"hm_scan_condition_files: NULL argument");
  return condition_into(s,ethresh,do_trim,do_symm,dst,-1,NULL,st);
}

extern "C" int hm_scan_condition_host(hm_scan *s, int ethresh, int do_trim, int do_symm, int64_t host_budget,
                                      hm_host_table **out, hm_condition_stats *st)
{ if (out == NULL)
    return hm_set_error(HM_EINVAL,"hm_scan_condition_host: NULL argument");
  return condition_into(s,ethresh,do_trim,do_symm,NULL,host_budget,out,st);
}

/* reverse complement of a left-aligned packed k-mer (k <= 32) */
static uint64_t revcomp64(uint64_t x, int k)
{ x = ~x;
  x = ((x >> 2)  & 0x3333333333333333ull) | ((x & 0x3333333333333333ull) << 2);
  x = ((x >> 4)  & 0x0F0F0F0F0F0F0F0Full) | ((x & 0x0F0F0F0F0F0F0F0Full) << 4);
  x = ((x >> 8)  & 0x00FF00FF00FF00FFull) | ((x & 0x00FF00FF00FF00FFull) << 8);
  x = ((x >> 16) & 0x0000FFFF0000FFFFull) | ((x & 0x0000FFFF0000FFFFull) << 16);
  x = (x >> 32) | (x << 32);
  if (k < 32)
    x = (x & (((uint64_t) 1 << (2*k))-1)) << (64-2*k);
  return x;
}

/* reverse complement of a left-aligned packed k-mer of 33..64 bases held in two words */
static void revcomp128(uint64_t hi, uint64_t lo, int k, uint64_t *rhi, uint64_t *rlo)
{ /* reversing all 64 slots swaps the words; the k real bases end up right-aligned over 128 bits */
  uint64_t a = revcomp64(lo,32), b = revcomp64(hi,32);      /* full-word reverse complements */
  int      sh = 2*(64-k);                                    /* pad slots now sit on top: shift them out */
  if (sh == 0) { *rhi = a; *rlo = b; }
  else         { *rhi = (a << sh) | (b >> (64-sh)); *rlo = b << sh; }
}

/* examine_table (PloidyPlot.c:1167-1230).  trim: smallest non-zero count among the middle <=1e8
 * entries >= ethresh.  symm: reverse complement of entry 1 (moving on past palindromes, where
 * the reference's loop would never terminate) is present.                                      */
static int examine_streamed(hm_scan *s, int ethresh, int *trim, int *symm);

extern "C" int hm_scan_examine(hm_scan *s, int ethresh, int *trim, int *symm)
{ if (s->streamed)
    return examine_streamed(s,ethresh,trim,symm);
  DevTable *D = s->d;
  int64_t   n = s->n, frst, last;
  int       h_min = 0x8000, *d_min = NULL, rc = HM_OK;
  uint64_t *d_q = NULL;
  int64_t  *d_pos = NULL;
  int       two = (D->keys_lo != NULL);
  cudaError_t e;

  if (n+3 < 100000000) { frst = 0; last = n; }
  else { frst = n/2-50000000; last = n/2+50000000; }
  TRY(cudaSetDevice(D->dev));
  TRY(dev_alloc(D,&d_min,sizeof(int)));
  TRY(dev_alloc(D,&d_q,2*sizeof(uint64_t)));
  TRY(dev_alloc(D,&d_pos,sizeof(int64_t)));
  TRY(cudaMemcpyAsync(d_min,&h_min,sizeof(int),cudaMemcpyHostToDevice,D->st));
  if (rc == HM_OK)
    { rc = hm_k_min_count(D->cnt,frst,last,d_min,D->st);
      s->launches += 1;
    }
  if (rc == HM_OK)
    { e = cudaMemcpyAsync(&h_min,d_min,sizeof(int),cudaMemcpyDeviceToHost,D->st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(D->st);
      if (e != cudaSuccess) rc = hm_cuda_fail(e,"min_count");
    }
  if (rc == HM_OK)
    { *trim = (h_min >= ethresh);
      *symm = 1;
    }
  for (int64_t sidx = 1; sidx < n && rc == HM_OK; sidx++)
    { uint64_t x, xw = 0, q[2];
      int64_t  pos;
      e = cudaMemcpyAsync(&x,D->keys+sidx,sizeof(uint64_t),cudaMemcpyDeviceToHost,D->st);
      if (e == cudaSuccess && two)
        e = cudaMemcpyAsync(&xw,D->keys_lo+sidx,sizeof(uint64_t),cudaMemcpyDeviceToHost,D->st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(D->st);
      if (e != cudaSuccess) { rc = hm_cuda_fail(e,"examine: key fetch"); break; }
      if (two) revcomp128(x,xw,s->kmer,q,q+1);
      else     { q[0] = revcomp64(x,s->kmer); q[1] = 0; }
      cudaMemcpyAsync(d_q,q,2*sizeof(uint64_t),cudaMemcpyHostToDevice,D->st);
      rc = hm_k_find_keys(D->keys,D->keys_lo,n,D->bucket,s->bits,s->idx64,d_q,two ? d_q+1 : NULL,1,d_pos,D->st);
      s->launches += 1;
      if (rc != HM_OK) break;
      e = cudaMemcpyAsync(&pos,d_pos,sizeof(int64_t),cudaMemcpyDeviceToHost,D->st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(D->st);
      if (e != cudaSuccess) { rc = hm_cuda_fail(e,"examine: lookup"); break; }
      if (pos < 0) { *symm = 0; break; }
      if (pos != sidx) { *symm = 1; break; }
    }
  dev_free(D,d_min); dev_free(D,d_q); dev_free(D,d_pos);
  return rc;
}

/* several GPUs: their plots summed into GPU 0's; then GPU 0's plot to the host (queued on its stream) */
static int plot_to_host(hm_scan *s, int64_t *plot)
{ int G = s->ngpu;
  if (G > 1)
    { unsigned long long *pl[HM_MAX_GPUS]; int dev[HM_MAX_GPUS]; cudaStream_t st[HM_MAX_GPUS];
      for (int g = 0; g < G; g++)
        { pl[g] = s->d[g].plot; dev[g] = s->d[g].dev; st[g] = s->d[g].st; }
      int rc = hm_peer_sum_plot(pl,dev,st,G);
      if (rc != HM_OK) return rc;
      s->launches += 1;
    }
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  HM_CUDA(cudaMemcpyAsync(plot,s->d[0].plot,sizeof(int64_t)*HM_PLOT_CELLS,cudaMemcpyDeviceToHost,s->d[0].st));
  return HM_OK;
}

/* every GPU g pulls the Bloom segments the other GPUs filled (segment h: GPU h) into its work area work[g], on
 * st[g]; skip_empty: not from shards without entries.  One layout L serves every GPU: hm_symm_plan places the
 * segments (off_bloom, seg_words) by n and the segment count alone, not by a GPU's range.                   */
static int gather_bloom(hm_scan *s, void *const *work, const hm_symm_layout *L, const cudaStream_t *st, int skip_empty)
{ size_t segb = sizeof(uint32_t)*(size_t) L->seg_words;
  for (int g = 0; g < s->ngpu; g++)
    { HM_CUDA(cudaSetDevice(s->d[g].dev));
      for (int h = 0; h < s->ngpu; h++)
        if (h != g && !(skip_empty && s->d[h].hi <= s->d[h].lo))
          HM_CUDA(cudaMemcpyPeerAsync((uint8_t *) work[g] + L->off_bloom + segb*h,s->d[g].dev,
                                      (uint8_t *) work[h] + L->off_bloom + segb*h,s->d[h].dev,segb,st[g]));
    }
  return HM_OK;
}

/* a run's stats: what differs by path comes as arguments; ms_run is the run's wall clock */
static void fill_stats(const hm_scan *s, hm_scan_stats *st, int path, int bucket_bits, int filter_bits, double ms_h2d,
                       float ms1, float ms2, double ms_scan, double ms_run, double ms_records, double ms_index)
{ if (st == NULL)
    return;
  st->nels = s->n; st->n_gpus = s->ngpu; st->bucket_bits = bucket_bits;
  st->filter_bits = filter_bits; st->path = path;
  st->ms_h2d_unpack = ms_h2d;
  st->ms_pass1 = ms1; st->ms_pass2 = ms2;
  st->ms_scan = ms_scan;
  st->ms_total = s->ms_load + ms_run;
  st->kernel_launches = s->launches;
  st->ms_alloc = s->ms_alloc; st->ms_records = ms_records; st->ms_index = ms_index;
}

/* the direct passes of hm_kernels.cu: any table */
static int run_direct(hm_scan *s, int64_t *plot, hm_scan_stats *stats)
{ int         G = s->ngpu, rc = HM_OK;
  int64_t     n = s->n;
  if ((rc = ensure_direct(s)) != HM_OK)
    return rc;
  double      t0 = now_ms();

  /* several GPUs: foreign incidence bytes are reached through the owner's array (remote atomics
   * in pass 1, remote loads in pass 2) when every pair of GPUs has native NVLink atomics; otherwise
   * the partial arrays are summed by the peer-memory kernel of hm_peer.cu                        */
  int        peer_mode = (G > 1);
  hm_shards *sh = s->sh;
  for (int a = 0; a < G && peer_mode; a++)
    for (int b = a+1; b < G && peer_mode; b++)
      if (!hm_p2p_native_atomics(s->d[a].dev,s->d[b].dev))
        peer_mode = 0;
  if (getenv("HETMERS_DENSE_EXCHANGE") != NULL)
    peer_mode = 0;
  if (peer_mode)
    for (int g = 0; g < G; g++)
      { memset(&sh[g],0,sizeof(hm_shards));
        sh[g].n_shards = G; sh[g].self = g;
        for (int r = 0; r < G; r++)
          { sh[g].off[r] = s->d[r].lo; sh[g].deg[r] = s->d[r].deg; }
        sh[g].off[G] = n;
        DevTable *D = s->d+g;
        int64_t need = hm_pass2_scratch_bytes(D->hi-D->lo,s->idx64);
        if (D->p2scratch == NULL || D->p2scratch_bytes < need)
          { HM_CUDA(cudaSetDevice(D->dev));
            dev_free(D,D->p2scratch);
            D->p2scratch = NULL;
            HM_CUDA(dev_alloc(D,&D->p2scratch,need));
            D->p2scratch_bytes = need;
          }
        sh[g].scratch = D->p2scratch; sh[g].scratch_bytes = D->p2scratch_bytes;
      }

  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      HM_CUDA(cudaSetDevice(D->dev));
      HM_CUDA(cudaEventRecord(D->ev[0],D->st));
      HM_CUDA(cudaMemsetAsync(D->deg,0,(size_t) ((n+4)&~3ll),D->st));
      HM_CUDA(cudaMemsetAsync(D->plot,0,sizeof(unsigned long long)*HM_PLOT_CELLS,D->st));
    }
  if (peer_mode && (rc = sync_all(s,"zero the incidence arrays")) != HM_OK)   /* nobody adds to a peer before it has been zeroed */
    return rc;
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      HM_CUDA(cudaSetDevice(D->dev));
      rc = hm_k_pass1_degree(D->keys,D->keys_lo,D->cnt,n,D->bucket,s->bits,s->idx64,D->filter,s->fpos,s->kmer,
                             D->lo,D->hi,D->deg,D->up,peer_mode ? &sh[g] : NULL,D->st);
      if (rc != HM_OK) return rc;
      s->launches += (D->hi > D->lo);
      HM_CUDA(cudaEventRecord(D->ev[1],D->st));
    }
  if (G > 1 && !peer_mode)
    { uint8_t *deg[HM_MAX_GPUS]; int64_t lo[HM_MAX_GPUS], hi[HM_MAX_GPUS];
      int dev[HM_MAX_GPUS]; cudaStream_t st[HM_MAX_GPUS];
      for (int g = 0; g < G; g++)
        { deg[g] = s->d[g].deg; lo[g] = s->d[g].lo; hi[g] = s->d[g].hi;
          dev[g] = s->d[g].dev; st[g] = s->d[g].st;
        }
      rc = hm_peer_sum_deg(deg,lo,hi,dev,st,G,n);
      if (rc != HM_OK) return rc;
      s->launches += G;
    }
  if (peer_mode && (rc = sync_all(s,"pass 1")) != HM_OK)   /* every pass 1 (and its remote atomics) has landed */
    return rc;
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      HM_CUDA(cudaSetDevice(D->dev));
      HM_CUDA(cudaEventRecord(D->ev[2],D->st));
      rc = hm_k_pass2_plot(D->cnt,D->deg,D->up,s->idx64,D->lo,D->hi,D->plot,
                           peer_mode ? &sh[g] : NULL,D->st);
      if (rc != HM_OK) return rc;
      s->launches += (D->hi > D->lo);
      HM_CUDA(cudaEventRecord(D->ev[3],D->st));
    }
  if ((rc = plot_to_host(s,plot)) != HM_OK || (rc = sync_all(s,"direct passes")) != HM_OK)
    return rc;
  double t1 = now_ms();
  s->ran = 1; s->peer_mode = peer_mode; s->last_path = HM_PATH_DIRECT;
  fill_stats(s,stats,HM_PATH_DIRECT,s->bits,s->fpos,s->ms_load,slowest_ms(s,0,1),slowest_ms(s,2,3),
             G > 1 ? t1-t0 : slowest_ms(s,0,3),t1-t0,s->ms_records,s->ms_index);
  return HM_OK;
}

/* the strand-symmetric scan of hm_symm.cu: run scan -> (Bloom segments all-gathered over peer
 * copies when >1 GPU) -> resolve -> plot reduce.  *status = the OR of the devices' status words:
 * non-zero means the table was not symmetric after all and the plot must not be used.           */
static int run_symm(hm_scan *s, int64_t *plot, hm_scan_stats *stats, uint64_t *status)
{ int         G = s->ngpu, rc = HM_OK;
  int64_t     n = s->n;
  if ((rc = ensure_symm(s)) != HM_OK)
    return rc;
  s->symm_ready = 0;
  double      t0 = now_ms();
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      HM_CUDA(cudaSetDevice(D->dev));
      HM_CUDA(cudaEventRecord(D->ev[0],D->st));
      HM_CUDA(cudaMemsetAsync(D->plot,0,sizeof(unsigned long long)*HM_PLOT_CELLS,D->st));
      rc = hm_k_symm_runscan(D->keys,D->keys_lo,D->cnt,n,D->bucket,s->bits,s->idx64,s->kmer,D->slo,D->shi,
                             D->symm_work,&D->symm_layout,G > 1 ? &s->ssh[g] : NULL,D->st);
      if (rc == HM_OK)
        rc = hm_k_symm_runs(D->keys,D->keys_lo,D->cnt,n,D->bucket,s->bits,s->idx64,s->kmer,D->slo,D->shi,
                            D->symm_work,&D->symm_layout,G > 1 ? &s->ssh[g] : NULL,D->st);
      if (rc != HM_OK) return rc;
      s->launches += 2*(D->shi > D->slo);
      HM_CUDA(cudaEventRecord(D->ev[1],D->st));
    }
  if (G > 1)                                    /* every device pulls the other devices' Bloom segments */
    { void *work[HM_MAX_GPUS]; cudaStream_t st[HM_MAX_GPUS];
      for (int g = 0; g < G; g++)
        { work[g] = s->d[g].symm_work; st[g] = s->d[g].st; }
      if ((rc = sync_all(s,"symmetric pass 1")) != HM_OK ||
          (rc = gather_bloom(s,work,&s->d[0].symm_layout,st,0)) != HM_OK)
        return rc;
    }
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      HM_CUDA(cudaSetDevice(D->dev));
      HM_CUDA(cudaEventRecord(D->ev[2],D->st));
      rc = hm_k_symm_resolve(D->keys,D->keys_lo,D->cnt,n,D->bucket,s->bits,s->idx64,s->kmer,
                             D->symm_work,&D->symm_layout,G > 1 ? &s->ssh[g] : NULL,D->plot,D->st);
      if (rc != HM_OK) return rc;
      s->launches += 1;
      HM_CUDA(cudaEventRecord(D->ev[3],D->st));
    }
  if ((rc = plot_to_host(s,plot)) != HM_OK)
    return rc;
  uint64_t hdr[HM_MAX_GPUS][2];
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      HM_CUDA(cudaSetDevice(D->dev));
      HM_CUDA(cudaMemcpyAsync(hdr[g],(uint8_t *) D->symm_work + D->symm_layout.off_header,2*sizeof(uint64_t),
                              cudaMemcpyDeviceToHost,D->st));
    }
  if ((rc = sync_all(s,"symmetric scan")) != HM_OK)
    return rc;
  double t1 = now_ms();
  *status = 0;
  for (int g = 0; g < G; g++)
    *status |= hdr[g][1];
  s->last_path = HM_PATH_SYMM;
  s->symm_ready = (*status == 0);
  fill_stats(s,stats,HM_PATH_SYMM,s->bits,0,s->ms_load,slowest_ms(s,0,1),slowest_ms(s,2,3),
             G > 1 ? t1-t0 : slowest_ms(s,0,3),t1-t0,s->ms_records,s->ms_index);
  return HM_OK;
}

/* ---- the streamed symmetric scan (DESIGN.md §4c) ------------------------------------------------------ */

/* largest i in [1,m) where a run (entries sharing their first k/2 bases) starts; 0 if all m share one */
static int last_run_start(const uint64_t *d_keys, int64_t m, int kmer, int64_t *out)
{ const int psh = 64-2*(kmer>>1);
  uint64_t  buf[4096];
  int64_t   end = m;
  while (end > 1)
    { int64_t from = end > 4096 ? end-4096 : 0;
      HM_CUDA(cudaMemcpy(buf,d_keys+from,sizeof(uint64_t)*(size_t) (end-from),cudaMemcpyDeviceToHost));
      for (int64_t i = end-1; i > from; i--)
        if (((buf[i-from] ^ buf[i-1-from]) >> psh) != 0)
          { *out = i; return HM_OK; }
      end = from+1;
    }
  *out = 0;
  return HM_OK;
}

/* lists in host memory: blocks of pageable host memory, each one flush's entries -- nw arrays of n words one after
 * another (candidates: key, meta and at k > 32 lo; S: key and at k > 32 lo).  They move to and from the device
 * through a shard's two pinned staging halves (stage_copy), so the pinned memory stays 2 SPILL_STAGE_BYTES per
 * shard whatever the lists' size.                                                                             */
typedef struct { uint64_t *w; int64_t n; } HostBlock;
typedef struct { HostBlock *b; int nb, cap; } HostList;

/* a new block of n entries of nw words at the end of L (*out: its words) */
static int host_list_add(HostList *L, int64_t n, int nw, uint64_t **out)
{ if (L->nb == L->cap)
    { int        cap = L->cap ? 2*L->cap : 16;
      HostBlock *b = (HostBlock *) realloc(L->b,sizeof(HostBlock)*(size_t) cap);
      if (b == NULL) return hm_set_error(HM_ENOMEM,"out of host memory");
      L->b = b; L->cap = cap;
    }
  void *p = malloc(8*(size_t) n*(size_t) nw);
  if (p == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory for the streamed scan's host lists (%lld bytes)",
                        (long long) (8*n*nw));
  L->b[L->nb].w = (uint64_t *) p; L->b[L->nb].n = n;
  L->nb += 1;
  *out = (uint64_t *) p;
  return HM_OK;
}

static int64_t host_list_entries(const HostList *L)
{ int64_t n = 0;
  for (int i = 0; i < L->nb; i++) n += L->b[i].n;
  return n;
}

static void host_list_free(HostList *L)
{ for (int i = 0; i < L->nb; i++) free(L->b[i].w);
  free(L->b);
  memset(L,0,sizeof(*L));
}

/* everything one streamed run allocates */
typedef struct
  { int64_t   cap;                                     /* entries per chunk buffer */
    uint64_t *keys[2], *klo[2];
    uint16_t *cnt[2];
    void     *bucket;
    int       bits;
    int64_t  *d_index;
    void     *work;
    hm_symm_layout L;
    hm_stream_lists R;
    Stager    G;
    void     *s_bucket;
    void     *sort_tmp;                                /* sorts the S keys of one chunk */
    int64_t   sort_bytes;
    cudaStream_t sc;                                   /* the chunks' kernels: overlap the next chunk's load */
    hm_stream_sview *views;                            /* several shards: every shard's S view, on this device */
    double    ms_loop;                                 /* the chunk loop, wall clock */
    int       spill, spilled;                          /* the lists may go to host memory; they have        */
    int64_t   list_room;                               /* (tests) HETMERS_LIST_ROOM: flush above this many list bytes */
    HostList  hc, hs;                                  /* there: the candidate records, the S list          */
    uint8_t  *stage[2];                                /* pinned staging halves (stage_copy)                */
    cudaEvent_t stage_ev[2];
    int64_t   flushes, d2h_bytes, rounds, h2d_bytes, first_key_queries;
    double    ms_flush, ms_pass2;
  } StreamRun;

static void stream_free_chunks(DevTable *D, StreamRun *R)
{ if (R->sc) cudaStreamSynchronize(R->sc);
  for (int b = 0; b < 2; b++)
    { dev_free(D,R->keys[b]); dev_free(D,R->klo[b]); dev_free(D,R->cnt[b]);
      R->keys[b] = NULL; R->klo[b] = NULL; R->cnt[b] = NULL;
    }
  dev_free(D,R->bucket);   R->bucket = NULL;
  dev_free(D,R->R.runs);   R->R.runs = NULL;
  dev_free(D,R->sort_tmp); R->sort_tmp = NULL;
  stager_close(D,&R->G);
}

/* chunk buffers for `cap` entries (+ bucket index, run list, staging), within the budget */
static int stream_alloc_chunks(hm_scan *s, DevTable *D, StreamRun *R, int64_t cap)
{ int KW = s->kmer > 32 ? 2 : 1;
  int64_t need = chunk_bytes(cap,s->kmer,s->ibyte);
  if (D->held + need > s->budget)
    return HM_ENOMEM;
  cudaError_t e = cudaSuccess;
  R->cap = cap;
  R->bits = hm_pick_bucket_bits(cap);
  for (int b = 0; b < 2 && e == cudaSuccess; b++)
    { e = dev_alloc(D,&R->keys[b],8*(cap+1));
      if (e == cudaSuccess && KW == 2) e = dev_alloc(D,&R->klo[b],8*(cap+1));
      if (e == cudaSuccess) e = dev_alloc(D,&R->cnt[b],2*(cap+8));
    }
  if (e == cudaSuccess) e = dev_alloc(D,&R->bucket,4*((1ll << R->bits)+1));
  R->R.runs_cap = cap/3+1024;
  if (e == cudaSuccess) e = dev_alloc(D,&R->R.runs,8*R->R.runs_cap);
  R->sort_bytes = hm_sort_keys_bytes(cap+1024,s->kmer);
  if (e == cudaSuccess) e = dev_alloc(D,&R->sort_tmp,R->sort_bytes);
  if (e != cudaSuccess)
    return hm_cuda_fail(e,"streamed scan: chunk buffers");
  return stager_open(s,D,s->host,cap,&R->G);
}

/* grow a group of resident arrays (same capacity, 8-byte elements) to hold `need` entries: doubling, but
 * no further than the final size projected from the `used` entries the first `done` of the shard's `total`
 * entries gave                                                                                           */
static int stream_grow(hm_scan *s, DevTable *D, cudaStream_t st, uint64_t **arr[], int narr, int64_t *cap,
                       int64_t used, int64_t need, int64_t done, int64_t total, const char *what)
{ if (need <= *cap)
    return HM_OK;
  int64_t nc = 2 * *cap;
  if (done > 0)
    { int64_t proj = need + (int64_t) ((double) used / (double) done * (double) (total - done) * 1.02);
      if (nc > proj) nc = proj;
    }
  if (nc < need) nc = need;
  int64_t room = (s->budget - D->held) / (8*narr);        /* the old arrays are held until the copy is done */
  if (nc > room) nc = room;
  if (nc < need)
    return hm_set_error(HM_ENOMEM,"the streamed scan's %s list needs %lld entries (%lld bytes) but the device budget "
                        "of %lld bytes has room for %lld more while %lld bytes are held; give the scan a larger "
                        "budget (HETMERS_DEVICE_BUDGET)%s",what,(long long) need,(long long) (8*narr*need),
                        (long long) s->budget,(long long) (room > 0 ? room : 0),(long long) D->held,
                        s->nshard > 1 ? "" : " or more GPUs (HETMERS_GPUS)");
  for (int a = 0; a < narr; a++)
    { uint64_t *p = NULL;
      cudaError_t e = dev_alloc(D,&p,8*nc);
      if (e != cudaSuccess) return hm_cuda_fail(e,"streamed scan: resident lists");
      if (used > 0 && *arr[a] != NULL)
        HM_CUDA(cudaMemcpyAsync(p,*arr[a],8*(size_t) used,cudaMemcpyDeviceToDevice,st));
      HM_CUDA(cudaStreamSynchronize(st));
      dev_free(D,*arr[a]);
      *arr[a] = p;
    }
  *cap = nc;
  return HM_OK;
}

#define SPILL_STAGE_BYTES (16ll << 20)            /* one pinned staging half */

/* the shard's staging halves and their events, once per run (freed by stream_release) */
static int stage_open(StreamRun *R)
{ if (R->stage[0] != NULL)
    return HM_OK;
  for (int i = 0; i < 2; i++)
    { HM_CUDA(cudaHostAlloc((void **) &R->stage[i],(size_t) SPILL_STAGE_BYTES,cudaHostAllocPortable));
      HM_CUDA(cudaEventCreateWithFlags(&R->stage_ev[i],cudaEventDisableTiming));
    }
  return HM_OK;
}

static void stage_close(StreamRun *R)
{ for (int i = 0; i < 2; i++)
    { if (R->stage_ev[i]) { cudaEventSynchronize(R->stage_ev[i]); cudaEventDestroy(R->stage_ev[i]); }
      if (R->stage[i]) cudaFreeHost(R->stage[i]);
      R->stage[i] = NULL; R->stage_ev[i] = NULL;
    }
}

/* `bytes` from device memory to a pageable host array (to_host) or back, on R->sc, a staging half per piece: the
 * DMA of one piece overlaps the host copy of the other.  Returns with the host array written (to_host), or with
 * the host array read and the copies to the device enqueued on R->sc (the halves are waited for before reuse). */
static int stage_copy(StreamRun *R, void *dst, const void *src, int64_t bytes, int to_host)
{ const int64_t P = SPILL_STAGE_BYTES, n = (bytes+P-1)/P;
  int rc;
  if ((rc = stage_open(R)) != HM_OK)
    return rc;
  for (int64_t i = 0; i <= n; i++)
    { const int h = (int) (i & 1);
      const int64_t off = i*P, len = i < n ? (bytes-off < P ? bytes-off : P) : 0;
      if (to_host)
        { if (i < n)
            { HM_CUDA(cudaMemcpyAsync(R->stage[h],(const uint8_t *) src+off,(size_t) len,cudaMemcpyDeviceToHost,R->sc));
              HM_CUDA(cudaEventRecord(R->stage_ev[h],R->sc));
            }
          if (i >= 1)
            { const int64_t o1 = off-P, l1 = bytes-o1 < P ? bytes-o1 : P;
              HM_CUDA(cudaEventSynchronize(R->stage_ev[h^1]));
              memcpy((uint8_t *) dst+o1,R->stage[h^1],(size_t) l1);
            }
        }
      else if (i < n)
        { HM_CUDA(cudaEventSynchronize(R->stage_ev[h]));        /* the half's previous piece has left it */
          memcpy(R->stage[h],(const uint8_t *) src+off,(size_t) len);
          HM_CUDA(cudaMemcpyAsync((uint8_t *) dst+off,R->stage[h],(size_t) len,cudaMemcpyHostToDevice,R->sc));
          HM_CUDA(cudaEventRecord(R->stage_ev[h],R->sc));
        }
    }
  return HM_OK;
}

/* The nc candidate records and ns S keys on the device (the S keys sorted) appended to the host lists, the list
 * counts reset and the device lists freed: the next chunk grows them again from nothing.  HM_ENOMEM when the
 * host lists of every shard would pass the list host budget.                                                */
static int stream_flush(hm_scan *s, DevTable *D, StreamRun *R, uint64_t nc, uint64_t ns)
{ int     KW = s->kmer > 32 ? 2 : 1, rc = HM_OK;
  double  t0 = now_ms();
  int64_t bytes = (int64_t) nc*(8*KW+8) + (int64_t) ns*8*KW;
  int64_t held = __sync_add_and_fetch(&s->host_held,bytes), pk;
  if (held > s->list_cap)
    return hm_set_error(HM_ENOMEM,"the streamed scan's lists need %lld bytes of host memory (%lld of them in this flush) "
                        "but the list host budget is %lld bytes; give the scan a larger one (%s)",
                        (long long) held,(long long) bytes,(long long) s->list_cap,
                        s->list_knob ? s->list_knob : "HETMERS_LIST_HOST_BUDGET");
  while ((pk = s->spill.host_peak_bytes) < held && !__sync_bool_compare_and_swap(&s->spill.host_peak_bytes,pk,held))
    ;
  uint64_t *h = NULL;
  if (nc > 0 && (rc = host_list_add(&R->hc,(int64_t) nc,KW+1,&h)) == HM_OK)
    { rc = stage_copy(R,h,R->R.cand_key,8*(int64_t) nc,1);
      if (rc == HM_OK) rc = stage_copy(R,h+nc,R->R.cand_meta,8*(int64_t) nc,1);
      if (rc == HM_OK && KW == 2) rc = stage_copy(R,h+2*nc,R->R.cand_lo,8*(int64_t) nc,1);
    }
  if (rc == HM_OK && ns > 0 && (rc = host_list_add(&R->hs,(int64_t) ns,KW,&h)) == HM_OK)
    { rc = stage_copy(R,h,R->R.s_key,8*(int64_t) ns,1);
      if (rc == HM_OK && KW == 2) rc = stage_copy(R,h+ns,R->R.s_lo,8*(int64_t) ns,1);
    }
  if (rc == HM_OK) rc = hm_symm_stream_reset_lists(R->work,&R->L,R->sc);
  if (rc != HM_OK) return rc;
  HM_CUDA(cudaStreamSynchronize(R->sc));
  dev_free(D,R->R.cand_key); dev_free(D,R->R.cand_meta); dev_free(D,R->R.cand_lo);
  dev_free(D,R->R.s_key);    dev_free(D,R->R.s_lo);
  R->R.cand_key = R->R.cand_meta = R->R.cand_lo = R->R.s_key = R->R.s_lo = NULL;
  R->R.cand_cap = R->R.s_cap = 0;
  R->spilled = 1;
  R->flushes += 1;
  R->d2h_bytes += bytes;
  R->ms_flush += now_ms()-t0;
  return HM_OK;
}

/* pass 1 of one shard: its range [D->lo, D->hi) chunk by chunk (leaves early, with HM_OK, once s->stop is set) */
static int stream_pass(hm_scan *s, DevTable *D, StreamRun *R, const hm_symm_shards *sh)
{ const hm_host_table *t = s->host;
  int      KW = s->kmer > 32 ? 2 : 1, rc = HM_OK;
  int64_t  lo = D->lo, hi = D->hi, c0 = lo, chunks = 0;
  int64_t  from = lo;                                /* where the lists on the device began: lo, or the last flush */
  int      b = 0;
  uint64_t nc = 0, status = 0, ns = 0, ns0 = 0;     /* ns0: S keys before the chunk in flight */
  HM_CUDA(cudaEventRecord(D->ev[0],R->sc));
  while (c0 < hi && rc == HM_OK && !s->stop)
    { int64_t m = hi-c0 < R->cap ? hi-c0 : R->cap;
      /* the copy + unpack of this chunk overlaps the kernels of the previous one (on R->sc) */
      rc = load_into(s,D,t,R->d_index,c0,m,R->keys[b],KW == 2 ? R->klo[b] : NULL,R->cnt[b],0,&R->G);
      if (rc != HM_OK) break;
      int64_t cut = m;
      if (c0+m < hi && (rc = last_run_start(R->keys[b],m,s->kmer,&cut)) != HM_OK)
        break;
      if (cut == 0)
        { /* one run fills the whole chunk: larger buffers, and load it again */
          int64_t cap = 2*R->cap;
          stream_free_chunks(D,R);
          rc = stream_alloc_chunks(s,D,R,cap);
          if (rc == HM_ENOMEM)
            rc = hm_set_error(HM_ENOMEM,"a run of more than %lld entries (k-mers sharing their first %d bases) does "
                              "not fit in one chunk of the streamed scan under the device budget of %lld bytes",
                              (long long) m,s->kmer>>1,(long long) s->budget);
          b = 0;
          continue;
        }
      if ((rc = hm_symm_stream_counts(R->work,&R->L,&nc,&status,&ns,R->sc)) != HM_OK)   /* previous chunk done */
        break;
      /* its S keys, sorted in place: chunks come in key order, so the list stays sorted as a whole */
      if ((rc = hm_sort_keys(R->R.s_key+ns0,KW == 2 ? R->R.s_lo+ns0 : NULL,(int64_t) (ns-ns0),s->kmer,
                             R->sort_tmp,R->sort_bytes,R->sc)) != HM_OK)
        break;
      ns0 = ns;
      for (int flushed = 0; ; flushed = 1)        /* no room left: with a list host budget, flush and grow again */
        { uint64_t **ca[3] = { &R->R.cand_key, &R->R.cand_meta, &R->R.cand_lo };
          uint64_t **sa[2] = { &R->R.s_key, &R->R.s_lo };
          int64_t    want = ((int64_t) nc + cut/2 + 1024)*(8*KW+8) + ((int64_t) ns + cut + 1024)*8*KW;
          if (R->spill && R->list_room > 0 && !flushed && want > R->list_room)
            rc = HM_ENOMEM;
          else
            { rc = stream_grow(s,D,R->sc,ca,KW == 2 ? 3 : 2,&R->R.cand_cap,(int64_t) nc,(int64_t) nc + cut/2 + 1024,
                               c0-from,hi-from,"candidate");
              if (rc == HM_OK)
                rc = stream_grow(s,D,R->sc,sa,KW,&R->R.s_cap,(int64_t) ns,(int64_t) ns + cut + 1024,c0-from,hi-from,"S");
            }
          if (rc != HM_ENOMEM || !R->spill || flushed)
            break;
          if ((rc = stream_flush(s,D,R,nc,ns)) != HM_OK)
            break;
          nc = ns = ns0 = 0;
          from = c0;
        }
      if (rc != HM_OK) break;
      rc = hm_k_build_bucket_index(R->keys[b],m,R->bits,R->bucket,0,R->sc);
      if (rc == HM_OK)
        rc = hm_k_symm_fingerprint(R->keys[b],KW == 2 ? R->klo[b] : NULL,R->cnt[b],0,cut,s->kmer,s->seed,D->fp_acc,R->sc);
      if (rc == HM_OK)
        rc = hm_symm_stream_chunk(R->keys[b],KW == 2 ? R->klo[b] : NULL,R->cnt[b],m,R->bucket,R->bits,s->kmer,cut,
                                  R->work,&R->L,&R->R,sh,R->sc);
      __sync_fetch_and_add(&s->launches,4);
      c0 += cut;
      chunks += 1;
      b ^= 1;
    }
  if (rc == HM_OK && (rc = hm_symm_stream_counts(R->work,&R->L,&nc,&status,&ns,R->sc)) == HM_OK)
    rc = hm_sort_keys(R->R.s_key+ns0,KW == 2 ? R->R.s_lo+ns0 : NULL,(int64_t) (ns-ns0),s->kmer,
                      R->sort_tmp,R->sort_bytes,R->sc);
  cudaEventRecord(D->ev[1],R->sc);
  cudaError_t e = cudaStreamSynchronize(R->sc);
  if (rc == HM_OK && e != cudaSuccess) rc = hm_cuda_fail(e,"streamed scan: pass 1");
  D->chunks = chunks;
  return rc;
}

/* on_every_gpu: shard g's pass 1 on its own device (arg: the runs of every shard): stub index, work area (the
 * whole-table Bloom filter), chunk buffers, the chunk loop                                                  */
static int shard_pass1(hm_scan *s, int g, void *arg)
{ DevTable  *D = s->d+g;
  StreamRun *R = (StreamRun *) arg + g;
  const hm_symm_shards *sh = s->nshard > 1 ? s->ssh+g : NULL;
  int64_t ixlen = (int64_t) 1 << (8*s->ibyte);
  int     rc;
  cudaError_t e;
  HM_CUDA(cudaSetDevice(D->dev));
  HM_CUDA(cudaStreamCreateWithFlags(&R->sc,cudaStreamNonBlocking));
  if ((rc = stream_work_layout(s->n,s->kmer,s->nshard,&R->L)) != HM_OK) return rc;
  if ((e = dev_alloc(D,&R->d_index,8*ixlen)) != cudaSuccess ||
      (e = dev_alloc(D,&R->work,R->L.bytes)) != cudaSuccess)
    return hm_cuda_fail(e,"streamed scan: work area");
  HM_CUDA(cudaMemcpyAsync(R->d_index,s->host->index,8*(size_t) ixlen,cudaMemcpyHostToDevice,R->sc));
  HM_CUDA(cudaMemsetAsync(D->fp_acc,0,4*sizeof(uint64_t),R->sc));
  HM_CUDA(cudaMemsetAsync(D->plot,0,8*(size_t) HM_PLOT_CELLS,R->sc));
  if ((rc = hm_symm_stream_begin(R->work,&R->L,R->sc)) != HM_OK) return rc;
  HM_CUDA(cudaStreamSynchronize(R->sc));
  if ((rc = stream_alloc_chunks(s,D,R,s->plan.chunk)) != HM_OK)
    return rc == HM_ENOMEM ? hm_set_error(HM_ENOMEM,"the streamed scan's chunk buffers do not fit the device budget") : rc;
  double t0 = now_ms();
  if ((rc = stream_pass(s,D,R,sh)) != HM_OK)
    return rc;
  R->ms_loop = now_ms()-t0;
  uint64_t nc = 0, status = 0, ns = 0;
  if ((rc = hm_symm_stream_counts(R->work,&R->L,&nc,&status,&ns,R->sc)) != HM_OK) return rc;
  if (status != 0)
    return hm_set_error(HM_ECUDA,"streamed scan: list overflow in pass 1 (status %llu)",(unsigned long long) status);
  if (R->spilled)                               /* the rest of the lists joins what went to host memory */
    return stream_flush(s,D,R,nc,ns);
  return HM_OK;
}

static int refuse_asymmetric(const hm_scan *s)
{ return hm_set_error(HM_EUNSUPPORTED,"the table of %lld entries does not fit in device memory (budget %lld bytes) and "
                      "is not strand-symmetric; the direct passes need it resident",(long long) s->n,(long long) s->budget);
}

/* after pass 1: the chunk buffers and stub index of shard g freed, and its S list (sorted chunk by chunk) given a
 * bucket index in the room they leave: as fine as hm_pick_bucket_bits asks, coarser if the budget says so
 * (look-ups then bisect longer buckets).  zero: clear the index first (an empty S list: all offsets 0).      */
static int stream_s_index(hm_scan *s, int g, StreamRun *R, uint64_t ns, int sidx64, int zero, int *sbits)
{ DevTable *D = s->d+g;
  cudaError_t e;
  HM_CUDA(cudaSetDevice(D->dev));
  stream_free_chunks(D,R);
  dev_free(D,R->d_index); R->d_index = NULL;
  int bits = hm_pick_bucket_bits((int64_t) ns);
  while (bits > 1 && D->held + (int64_t) (sidx64 ? 8 : 4)*((1ll << bits)+1) > s->budget)
    bits -= 1;
  int64_t s_bucket_bytes = (int64_t) (sidx64 ? 8 : 4)*((1ll << bits)+1);
  if ((e = dev_alloc(D,&R->s_bucket,s_bucket_bytes)) != cudaSuccess)
    return hm_cuda_fail(e,"streamed scan: S index");
  if (zero)
    HM_CUDA(cudaMemsetAsync(R->s_bucket,0,(size_t) s_bucket_bytes,R->sc));
  *sbits = bits;
  if (!zero || ns > 0)
    return hm_k_build_bucket_index(R->R.s_key,(int64_t) ns,bits,R->s_bucket,sidx64,R->sc);
  return HM_OK;
}

/* everything a streamed run allocated on shard g (its thread has been joined) */
static void stream_release(hm_scan *s, int g, StreamRun *R)
{ DevTable *D = s->d+g;
  cudaSetDevice(D->dev);
  stream_free_chunks(D,R);
  dev_free(D,R->d_index);  dev_free(D,R->work);
  dev_free(D,R->s_bucket); dev_free(D,R->views);
  dev_free(D,R->R.cand_key); dev_free(D,R->R.cand_meta); dev_free(D,R->R.cand_lo);
  dev_free(D,R->R.s_key);    dev_free(D,R->R.s_lo);
  if (D->st) cudaStreamSynchronize(D->st);
  if (R->sc) cudaStreamSynchronize(R->sc);
  host_list_free(&R->hc); host_list_free(&R->hs);
  stage_close(R);
  if (R->sc) cudaStreamDestroy(R->sc);
  cudaCtxResetPersistingL2Cache();
  cudaGetLastError();
  memset(R,0,sizeof(*R));
}

/* ---- pass 2 of lists in host memory (DESIGN.md §4c, *Lists in host memory*) ---- */

/* one S partition: n keys (and at k > 32 their second words) in a host block; partitions cut the concatenated S
 * lists of the shards -- the whole table's S, sorted -- into pieces of at most plan.part keys                   */
typedef struct { const uint64_t *key, *lo; int64_t n; } SpillPart;

typedef struct
  { StreamRun      *RR;
    hm_spill_layout P;
    SpillPart      *parts;
    int64_t         nparts;
  } SpillRun;

/* the first index in [lo, hi) of the sorted queries q (KW words each) whose key is >= (kh, kl) */
static int64_t query_lower_bound(const uint64_t *q, int KW, int64_t lo, int64_t hi, uint64_t kh, uint64_t kl)
{ while (lo < hi)
    { int64_t  m = lo + (hi-lo)/2;
      uint64_t h = q[KW*m], l = KW == 2 ? q[KW*m+1] : 0;
      if (h < kh || (h == kh && l < kl)) lo = m+1; else hi = m;
    }
  return lo;
}

/* the S partitions of the host S list hs (blocks in key order), cut into pieces of at most `part` keys:
 * spill_part_count how many, spill_cut_parts appends them at parts + *n                                   */
static int64_t spill_part_count(const HostList *hs, int64_t part)
{ int64_t np = 0;
  for (int b = 0; b < hs->nb; b++)
    np += (hs->b[b].n + part-1)/part;
  return np;
}

static void spill_cut_parts(const HostList *hs, int64_t part, int KW, SpillPart *parts, int64_t *n)
{ for (int b = 0; b < hs->nb; b++)
    { const HostBlock *hb = hs->b+b;
      for (int64_t o = 0; o < hb->n; o += part)
        { SpillPart *P = parts + (*n)++;
          P->key = hb->w+o; P->lo = KW == 2 ? hb->w+hb->n+o : NULL;
          P->n = hb->n-o < part ? hb->n-o : part;
        }
    }
}

/* n sorted keys (hq on the host, d_q on the device, KW words each) answered against the partitions in key order:
 * the keys falling in partition p are the contiguous range between the lower bounds of its first key and the
 * next partition's; a partition no key falls in is not uploaded, the others are uploaded into pkey / plo,
 * indexed into pbucket (`bits`) and answer their range into ans (zeroed by the caller)                       */
static int spill_answer_parts(hm_scan *s, StreamRun *R, const SpillPart *parts, int64_t nparts, int bits,
                              const uint64_t *hq, const uint64_t *d_q, int64_t n, uint64_t *pkey, uint64_t *plo,
                              void *pbucket, uint8_t *ans)
{ const int KW = s->kmer > 32 ? 2 : 1;
  int       rc = HM_OK;
  int64_t   lo = 0;
  for (int64_t p = 0; p < nparts && lo < n && rc == HM_OK; p++)
    { const SpillPart *P = parts+p;
      int64_t hi = n;
      if (p+1 < nparts)
        hi = query_lower_bound(hq,KW,lo,n,P[1].key[0],KW == 2 ? P[1].lo[0] : 0);
      if (hi == lo)
        continue;                               /* no key falls in this partition: nothing uploaded */
      R->first_key_queries += (hq[KW*lo] == P->key[0] && (KW == 1 || hq[KW*lo+1] == P->lo[0]));
      rc = stage_copy(R,pkey,P->key,8*P->n,0);
      if (rc == HM_OK && KW == 2) rc = stage_copy(R,plo,P->lo,8*P->n,0);
      if (rc == HM_OK) rc = hm_k_build_bucket_index(pkey,P->n,bits,pbucket,0,R->sc);
      if (rc == HM_OK)
        rc = hm_symm_route_answer(pkey,plo,pbucket,bits,0,s->kmer,d_q+KW*lo,hi-lo,ans+lo,R->sc);
      R->h2d_bytes += 8*KW*P->n;
      __sync_fetch_and_add(&s->launches,2);
      lo = hi;
    }
  return rc;
}

/* the device buffers of one shard's pass 2 over host lists */
typedef struct
  { hm_stream_lists L;                            /* cand_key / cand_meta / cand_lo: one slice */
    hm_route_bufs   B;
    uint32_t       *perm[2];
    uint8_t        *ans;
    void           *tmp;
    int64_t         tmp_bytes;
    uint64_t       *pkey, *plo;                   /* one partition and its bucket index */
    void           *pbucket;
    uint64_t       *hq;                           /* (host) the round's sorted queries */
  } SpillBufs;

static void spill_free(DevTable *D, StreamRun *R, SpillBufs *X)
{ if (R->sc) cudaStreamSynchronize(R->sc);
  dev_free(D,X->L.cand_key); dev_free(D,X->L.cand_meta); dev_free(D,X->L.cand_lo);
  dev_free(D,X->B.pend); dev_free(D,X->B.q_key); dev_free(D,X->B.q_lo); dev_free(D,X->B.q_tag); dev_free(D,X->B.send);
  dev_free(D,X->perm[0]); dev_free(D,X->perm[1]); dev_free(D,X->ans); dev_free(D,X->tmp);
  dev_free(D,X->pkey); dev_free(D,X->plo); dev_free(D,X->pbucket);
  free(X->hq);
  memset(X,0,sizeof(*X));
}

/* the round's parked candidates settled: its queries sorted by key, each S partition some query falls in uploaded
 * and indexed, the queries in it answered; then every parked candidate none of whose queries was found counted */
static int spill_settle(hm_scan *s, int g, const SpillRun *S, StreamRun *R, SpillBufs *X, int64_t n_pend, int64_t n_q)
{ DevTable *D = s->d+g;
  const int KW = s->kmer > 32 ? 2 : 1, bits = S->P.part_bits;
  int rc;
  if ((rc = hm_symm_park_sort(s->kmer,&X->B,n_q,X->perm[0],X->perm[1],X->tmp,X->tmp_bytes,R->sc)) != HM_OK)
    return rc;
  if (n_q > 0)
    { HM_CUDA(cudaMemcpyAsync(X->hq,X->B.send,8*(size_t) KW*(size_t) n_q,cudaMemcpyDeviceToHost,R->sc));
      HM_CUDA(cudaMemsetAsync(X->ans,0,(size_t) n_q,R->sc));
      HM_CUDA(cudaStreamSynchronize(R->sc));
    }
  rc = spill_answer_parts(s,R,S->parts,S->nparts,bits,X->hq,X->B.send,n_q,X->pkey,X->plo,X->pbucket,X->ans);
  if (rc == HM_OK)
    rc = hm_symm_route_settle(s->kmer,&X->B,X->ans,n_q,n_pend,D->plot,R->sc);
  __sync_fetch_and_add(&s->launches,2);
  R->rounds += 1;
  return rc;
}

/* on_every_gpu: shard g's pass 2 over its candidates in host memory, in rounds of slices (arg: the SpillRun) */
static int shard_spill_pass2(hm_scan *s, int g, void *arg)
{ const SpillRun *S = (const SpillRun *) arg;
  DevTable  *D = s->d+g;
  StreamRun *R = S->RR+g;
  const hm_symm_shards *sh = s->nshard > 1 ? s->ssh+g : NULL;
  const int  KW = s->kmer > 32 ? 2 : 1;
  const int64_t C = S->P.slice, Q = S->P.queries;
  SpillBufs  X;
  int        rc = HM_OK;
  cudaError_t e;
  memset(&X,0,sizeof(X));
  X.L = R->R;
  X.L.cand_cap = C;
  X.tmp_bytes = hm_sort_perm_bytes(Q);
  TRY(cudaSetDevice(D->dev));
  TRY(dev_alloc(D,&X.L.cand_key,8*C));
  TRY(dev_alloc(D,&X.L.cand_meta,8*C));
  X.L.cand_lo = NULL;
  if (KW == 2) TRY(dev_alloc(D,&X.L.cand_lo,8*C));
  TRY(dev_alloc(D,&X.B.pend,8*C));
  TRY(dev_alloc(D,&X.B.q_key,8*Q));
  if (KW == 2) TRY(dev_alloc(D,&X.B.q_lo,8*Q));
  TRY(dev_alloc(D,&X.B.q_tag,8*Q));
  TRY(dev_alloc(D,&X.B.send,8*KW*Q));
  TRY(dev_alloc(D,&X.perm[0],4*Q));
  TRY(dev_alloc(D,&X.perm[1],4*Q));
  TRY(dev_alloc(D,&X.ans,Q));
  TRY(dev_alloc(D,&X.tmp,X.tmp_bytes));
  TRY(dev_alloc(D,&X.pkey,8*S->P.part));
  if (KW == 2) TRY(dev_alloc(D,&X.plo,8*S->P.part));
  TRY(dev_alloc(D,&X.pbucket,4*((1ll << S->P.part_bits)+1)));
  X.B.pend_cap = C; X.B.q_cap = Q;
  if (rc == HM_OK && D->held > s->budget)
    rc = hm_set_error(HM_ENOMEM,"pass 2 of the streamed scan's lists in host memory holds %lld device bytes, more than "
                      "the budget of %lld (the plan counted %lld)",(long long) D->held,(long long) s->budget,
                      (long long) (S->P.slice_bytes+S->P.part_bytes));
  if (rc == HM_OK && (X.hq = (uint64_t *) malloc(8*(size_t) KW*(size_t) Q)) == NULL)
    rc = hm_set_error(HM_ENOMEM,"out of host memory");
  double  t0 = now_ms();
  int64_t in_round = 0, n_pend = 0, n_q = 0;
  uint64_t status = 0;
  if (rc == HM_OK) cudaEventRecord(D->ev[2],R->sc);
  for (int b = 0; b < R->hc.nb && rc == HM_OK && !s->stop; b++)
    { const HostBlock *hb = R->hc.b+b;
      for (int64_t c = 0; c < hb->n && rc == HM_OK; c += C)
        { int64_t m = hb->n-c < C ? hb->n-c : C;
          if (in_round > 0 && n_pend + m > C)           /* the next slice might not find a pending slot for each hit */
            { rc = spill_settle(s,g,S,R,&X,n_pend,n_q);
              in_round = 0;
              if (rc != HM_OK) break;
            }
          rc = stage_copy(R,X.L.cand_key,hb->w+c,8*m,0);
          if (rc == HM_OK) rc = stage_copy(R,X.L.cand_meta,hb->w+hb->n+c,8*m,0);
          if (rc == HM_OK && KW == 2) rc = stage_copy(R,X.L.cand_lo,hb->w+2*hb->n+c,8*m,0);
          R->h2d_bytes += m*(8*KW+8);
          if (rc == HM_OK)
            rc = hm_symm_park_resolve(s->kmer,m,in_round == 0,R->work,&R->L,&X.L,sh,&X.B,D->plot,R->sc);
          __sync_fetch_and_add(&s->launches,1);
          if (rc == HM_OK)
            rc = hm_symm_park_counts(R->work,&R->L,&n_pend,&n_q,&status,R->sc);
          if (rc == HM_OK && (status != 0 || n_pend > C || n_q > Q))   /* the round rule keeps both within the buffers */
            rc = hm_set_error(HM_ECUDA,"streamed scan: pass 2 of the host lists overflowed (status %llu, %lld parked "
                              "of %lld slots, %lld queries of %lld)",(unsigned long long) status,(long long) n_pend,
                              (long long) C,(long long) n_q,(long long) Q);
          in_round += 1;
        }
    }
  if (rc == HM_OK && in_round > 0)
    rc = spill_settle(s,g,S,R,&X,n_pend,n_q);
  cudaEventRecord(D->ev[3],R->sc);
  R->ms_pass2 = now_ms()-t0;
  spill_free(D,R,&X);
  return rc;
}

/* pass 2 of every shard whose lists went to host memory: the chunk buffers and stub index freed, one plan for the
 * room that leaves on every shard, the S partitions cut, the rounds of every shard at once                   */
static int spill_pass2(hm_scan *s, StreamRun *RR)
{ int      G = s->ngpu, KW = s->kmer > 32 ? 2 : 1, rc;
  int64_t  ncmax = 0, ns = 0, room = -1;
  SpillRun S;
  memset(&S,0,sizeof(S));
  S.RR = RR;
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      HM_CUDA(cudaSetDevice(D->dev));
      stream_free_chunks(D,RR+g);
      dev_free(D,RR[g].d_index); RR[g].d_index = NULL;
      int64_t nc = host_list_entries(&RR[g].hc);
      if (nc > ncmax) ncmax = nc;
      ns += host_list_entries(&RR[g].hs);
      if (room < 0 || s->budget - D->held < room) room = s->budget - D->held;
    }
  const char *e = getenv("HETMERS_SPILL_ROOM");              /* smaller slices and partitions than the room allows */
  if (e != NULL && atoll(e) > 0 && atoll(e) < room)
    room = atoll(e);
  if ((rc = hm_spill_plan(ncmax,ns,s->kmer,room,&S.P)) != HM_OK)
    return rc;
  if ((e = getenv("HETMERS_SPILL_PART")) != NULL && atoll(e) > 0 && atoll(e) < S.P.part)   /* smaller partitions */
    { S.P.part = atoll(e);
      S.P.part_bits = hm_pick_bucket_bits(S.P.part);
    }
  int64_t np = 0;
  for (int g = 0; g < G; g++)
    np += spill_part_count(&RR[g].hs,S.P.part);
  if ((S.parts = (SpillPart *) malloc(sizeof(SpillPart)*(size_t) (np > 0 ? np : 1))) == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory");
  for (int g = 0; g < G; g++)                                  /* shards in key order, blocks in key order */
    spill_cut_parts(&RR[g].hs,S.P.part,KW,S.parts,&S.nparts);
  rc = on_every_gpu(s,shard_spill_pass2,&S);
  free(S.parts);
  s->spill.partitions = S.nparts;
  s->spill.slice = S.P.slice; s->spill.part = S.P.part;
  return rc;
}

/* pass 2 of every shard with its lists on the device: the chunk buffers and stub index freed, to make room for
 * each shard's S index; the exact checks look keys up in the S list of their owner (peer memory)            */
static int stream_lists_pass2(hm_scan *s, StreamRun *RR, const uint64_t *ns, int *sbits, int sidx64)
{ int G = s->ngpu, KW = s->kmer > 32 ? 2 : 1, rc = HM_OK;
  cudaError_t e;
  for (int g = 0; g < G; g++)
    if ((rc = stream_s_index(s,g,RR+g,ns[g],sidx64,G > 1,&sbits[g])) != HM_OK)
      return rc;
  if (G > 1)                                    /* each shard's pass 2 reads every shard's S view */
    { hm_stream_sview V[HM_MAX_GPUS];
      memset(V,0,sizeof(V));
      for (int h = 0; h < G; h++)
        { V[h].s_key = RR[h].R.s_key; V[h].s_lo = KW == 2 ? RR[h].R.s_lo : NULL;
          V[h].s_bucket = RR[h].s_bucket; V[h].n_s = (int64_t) ns[h]; V[h].bits = sbits[h];
        }
      for (int g = 0; g < G; g++)
        { DevTable *D = s->d+g;
          HM_CUDA(cudaSetDevice(D->dev));
          if ((e = dev_alloc(D,&RR[g].views,sizeof(V))) != cudaSuccess)
            return hm_cuda_fail(e,"streamed scan: S views");
          HM_CUDA(cudaMemcpyAsync(RR[g].views,V,sizeof(V),cudaMemcpyHostToDevice,RR[g].sc));
        }
      for (int g = 0; g < G; g++)               /* every S index and Bloom segment is in place */
        { HM_CUDA(cudaSetDevice(s->d[g].dev)); HM_CUDA(cudaStreamSynchronize(RR[g].sc)); }
    }

  for (int g = 0; g < G; g++)
    { DevTable  *D = s->d+g;
      StreamRun *R = RR+g;
      HM_CUDA(cudaSetDevice(D->dev));
      cudaEventRecord(D->ev[2],R->sc);
      rc = hm_symm_stream_resolve(R->R.s_key,KW == 2 ? R->R.s_lo : NULL,(int64_t) ns[g],R->s_bucket,sbits[g],sidx64,
                                  s->kmer,G == 1 ? s->n : D->hi-D->lo,R->work,&R->L,&R->R,G > 1 ? s->ssh+g : NULL,
                                  R->views,D->plot,R->sc);
      cudaEventRecord(D->ev[3],R->sc);
      __sync_fetch_and_add(&s->launches,3);
      if (rc != HM_OK) return rc;
    }
  return HM_OK;
}

/* Pass 1 of every shard at once; the verdict over all shards' fingerprints; the Bloom segments all-gathered; the
 * chunk buffers and stub index freed, to make room for each shard's S index; pass 2 of every shard, whose exact
 * checks look keys up in the S list of their owner (peer memory); the plots summed on the host.              */
static int run_stream_body(hm_scan *s, StreamRun *RR, int64_t *plot, hm_scan_stats *stats)
{ int       G = s->ngpu, KW = s->kmer > 32 ? 2 : 1, rc = HM_OK;
  double    t0 = now_ms();
  double    ms_loop = 0;
  cudaError_t e;
  s->stop = 0;
  if ((rc = on_every_gpu(s,shard_pass1,RR)) != HM_OK)
    return rc;
  for (int g = 0; g < G; g++)
    if (RR[g].ms_loop > ms_loop) ms_loop = RR[g].ms_loop;
  float  ms1 = slowest_ms(s,0,1);
  double t_pass1 = now_ms();
  if ((rc = fingerprint_verdict(s)) != HM_OK) return rc;
  if (!s->symmetric)
    return refuse_asymmetric(s);
  int spilled = 0;
  for (int g = 0; g < G; g++)
    spilled |= RR[g].spilled;
  for (int g = 0; g < G && spilled; g++)        /* one pass 2 for every shard: every shard's lists to host memory */
    if (!RR[g].spilled)
      { uint64_t nc = 0, status = 0, nsg = 0;
        HM_CUDA(cudaSetDevice(s->d[g].dev));
        if ((rc = hm_symm_stream_counts(RR[g].work,&RR[g].L,&nc,&status,&nsg,RR[g].sc)) != HM_OK ||
            (rc = stream_flush(s,s->d+g,RR+g,nc,nsg)) != HM_OK)
          return rc;
      }

  uint64_t ns[HM_MAX_GPUS];
  int      sbits[HM_MAX_GPUS], sidx64 = 0;
  for (int g = 0; g < G; g++)
    { uint64_t nc = 0, status = 0;
      HM_CUDA(cudaSetDevice(s->d[g].dev));
      if ((rc = hm_symm_stream_counts(RR[g].work,&RR[g].L,&nc,&status,&ns[g],RR[g].sc)) != HM_OK) return rc;
      if ((int64_t) ns[g] >= 0xFFFFFFF0ll) sidx64 = 1;    /* one offset width for every shard's index */
    }
  if (G > 1)                                    /* every shard pulls the other shards' Bloom segments */
    { void *work[HM_MAX_GPUS]; cudaStream_t st[HM_MAX_GPUS];
      for (int g = 0; g < G; g++)
        { work[g] = RR[g].work; st[g] = RR[g].sc; }
      if ((rc = gather_bloom(s,work,&RR[0].L,st,1)) != HM_OK)
        return rc;
    }
  if (spilled)
    { if ((rc = spill_pass2(s,RR)) != HM_OK)
        return rc;
    }
  else if ((rc = stream_lists_pass2(s,RR,ns,sbits,sidx64)) != HM_OK)
    return rc;
  int64_t *tmp = NULL;
  if (G > 1)
    { if ((tmp = (int64_t *) malloc(sizeof(int64_t)*HM_PLOT_CELLS)) == NULL)
        return hm_set_error(HM_ENOMEM,"out of host memory");
      memset(plot,0,sizeof(int64_t)*HM_PLOT_CELLS);
    }
  for (int g = 0; g < G && rc == HM_OK; g++)
    { DevTable  *D = s->d+g;
      StreamRun *R = RR+g;
      uint64_t   nc = 0, status = 0, nsx = 0;
      cudaSetDevice(D->dev);
      if ((e = cudaMemcpyAsync(G == 1 ? plot : tmp,D->plot,sizeof(int64_t)*HM_PLOT_CELLS,
                               cudaMemcpyDeviceToHost,R->sc)) != cudaSuccess)
        rc = hm_cuda_fail(e,"plot D2H");
      if (rc == HM_OK)
        rc = hm_symm_stream_counts(R->work,&R->L,&nc,&status,&nsx,R->sc);      /* (synchronises) */
      if (rc == HM_OK && status != 0)
        rc = hm_set_error(HM_ECUDA,"streamed scan: pass 2 status %llu%s",(unsigned long long) status,G > 1 ? " on a shard" : "");
      if (rc == HM_OK && G > 1)
        for (int64_t i = 0; i < HM_PLOT_CELLS; i++)
          plot[i] += tmp[i];
    }
  free(tmp);
  if (rc != HM_OK)
    return rc;
  double t1 = now_ms();
  s->last_path = HM_PATH_SYMM;
  fill_stats(s,stats,HM_PATH_SYMM,RR[0].bits,0,s->ms_load+ms_loop,              /* the loads, with pass 1 behind them */
             ms1,slowest_ms(s,2,3),t1-t0,t1-t0,ms_loop,t1-t_pass1);              /* (the slowest shard's passes)       */
  return HM_OK;
}

static int run_stream(hm_scan *s, int64_t *plot, hm_scan_stats *stats)
{ int       G = s->ngpu;
  StreamRun R[HM_MAX_GPUS];
  if (s->kmer < HM_SYMM_MIN_KMER)
    return hm_set_error(HM_EUNSUPPORTED,"the table does not fit in device memory and k = %d has no strand-symmetric "
                        "scan; the direct passes need it resident",s->kmer);
  memset(R,0,sizeof(R));
  memset(&s->spill,0,sizeof(s->spill));
  s->list_cap = g_list_host_budget;
  s->host_held = 0;
  for (int g = 0; g < G; g++)
    { s->d[g].peak = s->d[g].held;
      s->d[g].chunks = 0;
      R[g].spill = (s->list_cap > 0);
      if (R[g].spill && getenv("HETMERS_LIST_ROOM") != NULL)    /* smaller device lists than the budget allows */
        R[g].list_room = atoll(getenv("HETMERS_LIST_ROOM"));
    }
  int rc = run_stream_body(s,R,plot,stats);
  hm_spill_stats *X = &s->spill;
  for (int g = 0; g < G; g++)
    { X->spilled |= R[g].spilled;
      X->flushes += R[g].flushes; X->d2h_bytes += R[g].d2h_bytes;
      X->rounds += R[g].rounds;   X->h2d_bytes += R[g].h2d_bytes;
      X->first_key_queries += R[g].first_key_queries;
      if (R[g].ms_loop > X->ms_pass1)  X->ms_pass1 = R[g].ms_loop;
      if (R[g].ms_flush > X->ms_flush) X->ms_flush = R[g].ms_flush;
      if (R[g].ms_pass2 > X->ms_pass2) X->ms_pass2 = R[g].ms_pass2;
    }
  for (int g = 0; g < G; g++)                  /* every shard's thread has been joined: free it all */
    stream_release(s,g,R+g);
  return rc;
}

extern "C" int hm_scan_spill_stats(const hm_scan *s, hm_spill_stats *out)
{ if (s == NULL || out == NULL)
    return hm_set_error(HM_EINVAL,"hm_scan_spill_stats: bad arguments");
  *out = s->spill;
  return HM_OK;
}

/* examine_table's decisions on a streamed scan: the trim minimum over the same middle entries, chunk by
 * chunk; the symmetry probe fetches entry sidx, and searches the stub-index bucket that must hold its
 * reverse complement                                                                                     */
static int examine_streamed(hm_scan *s, int ethresh, int *trim, int *symm)
{ DevTable *D = s->d;
  const hm_host_table *t = s->host;
  int      two = (s->kmer > 32), rc = HM_OK;
  int64_t  n = s->n, frst, last, cap = s->plan.chunk;
  int      h_min = 0x8000, *d_min = NULL;
  uint64_t *d_q = NULL;
  int64_t  *d_pos = NULL;
  void     *bucket = NULL;
  int      bits = hm_pick_bucket_bits(cap);
  Window   W;
  cudaError_t e;
  if ((rc = window_open(s,cap,&W)) != HM_OK)
    return rc;
  TRY(dev_alloc(D,&bucket,4*((1ll << bits)+1)));
  TRY(dev_alloc(D,&d_min,sizeof(int)));
  TRY(dev_alloc(D,&d_q,2*sizeof(uint64_t)));
  TRY(dev_alloc(D,&d_pos,sizeof(int64_t)));
  TRY(cudaMemcpyAsync(d_min,&h_min,sizeof(int),cudaMemcpyHostToDevice,D->st));

  if (n+3 < 100000000) { frst = 0; last = n; }
  else { frst = n/2-50000000; last = n/2+50000000; }
  for (int64_t o = frst; o < last && rc == HM_OK; o += cap)
    { int64_t m = last-o < cap ? last-o : cap;
      rc = window_load(s,&W,o,m);
      if (rc == HM_OK) rc = hm_k_min_count(W.cnt,0,m,d_min,D->st);
      s->launches += 1;
    }
  if (rc == HM_OK)
    { e = cudaMemcpyAsync(&h_min,d_min,sizeof(int),cudaMemcpyDeviceToHost,D->st);
      if (e == cudaSuccess) e = cudaStreamSynchronize(D->st);
      if (e != cudaSuccess) rc = hm_cuda_fail(e,"min_count");
    }
  if (rc == HM_OK)
    { *trim = (h_min >= ethresh);
      *symm = 1;
    }
  const int psh = 64 - 8*s->ibyte;                    /* the stub index is over the first ibyte bytes */
  for (int64_t sidx = 1; sidx < n && rc == HM_OK; sidx++)
    { uint64_t x, xw = 0, q[2];
      int64_t  pos = -1;
      if ((rc = window_load(s,&W,sidx,1)) != HM_OK) break;
      e = cudaMemcpy(&x,W.keys,sizeof(uint64_t),cudaMemcpyDeviceToHost);
      if (e == cudaSuccess && two) e = cudaMemcpy(&xw,W.klo,sizeof(uint64_t),cudaMemcpyDeviceToHost);
      if (e != cudaSuccess) { rc = hm_cuda_fail(e,"examine: key fetch"); break; }
      if (two) revcomp128(x,xw,s->kmer,q,q+1);
      else     { q[0] = revcomp64(x,s->kmer); q[1] = 0; }
      uint64_t p  = q[0] >> psh;
      int64_t  b0 = p > 0 ? t->index[p-1] : 0, b1 = t->index[p];
      if ((e = cudaMemcpy(d_q,q,2*sizeof(uint64_t),cudaMemcpyHostToDevice)) != cudaSuccess)
        { rc = hm_cuda_fail(e,"examine: key upload"); break; }
      for (int64_t o = b0; o < b1 && rc == HM_OK && pos < 0; o += cap)
        { int64_t m = b1-o < cap ? b1-o : cap;
          rc = window_load(s,&W,o,m);
          if (rc == HM_OK) rc = hm_k_build_bucket_index(W.keys,m,bits,bucket,0,D->st);
          if (rc == HM_OK) rc = hm_k_find_keys(W.keys,W.klo,m,bucket,bits,0,d_q,two ? d_q+1 : NULL,1,d_pos,D->st);
          s->launches += 2;
          if (rc != HM_OK) break;
          e = cudaMemcpyAsync(&pos,d_pos,sizeof(int64_t),cudaMemcpyDeviceToHost,D->st);
          if (e == cudaSuccess) e = cudaStreamSynchronize(D->st);
          if (e != cudaSuccess) { rc = hm_cuda_fail(e,"examine: lookup"); break; }
          if (pos >= 0) pos += o;
        }
      if (rc != HM_OK) break;
      if (pos < 0) { *symm = 0; break; }
      if (pos != sidx) { *symm = 1; break; }
    }
  dev_free(D,bucket); dev_free(D,d_min); dev_free(D,d_q); dev_free(D,d_pos);
  window_close(s,&W);
  return rc;
}

extern "C" int hm_scan_is_symmetric(const hm_scan *s) { return s->symmetric; }

/* The scan a run or an extraction takes: HETMERS_PATH (direct / symm) stands in for HM_PATH_AUTO, which takes the
 * symmetric scan on a strand-symmetric table and the direct passes on any other.  *symm: the route; *forced: the
 * symmetric scan was asked for, so it may not fall back to the direct passes.                                  */
static int choose_route(const hm_scan *s, int path, int *symm, int *forced)
{ if (path == HM_PATH_AUTO)
    { const char *e = getenv("HETMERS_PATH");
      if (e != NULL && strcmp(e,"direct") == 0) path = HM_PATH_DIRECT;
      if (e != NULL && strcmp(e,"symm") == 0)   path = HM_PATH_SYMM;
    }
  if (s->streamed && path == HM_PATH_DIRECT)
    return hm_set_error(HM_EUNSUPPORTED,"the direct passes need the table resident; this one does not fit in "
                                        "device memory (budget %lld bytes) and is streamed",(long long) s->budget);
  if (path != HM_PATH_AUTO && path != HM_PATH_DIRECT && path != HM_PATH_SYMM)
    return hm_set_error(HM_EINVAL,"hm_scan_run_path: unknown path %d",path);
  *forced = (path == HM_PATH_SYMM);
  *symm = s->streamed || path == HM_PATH_SYMM || (path == HM_PATH_AUTO && s->symmetric);
  if (!s->streamed && *symm && (s->kmer < HM_SYMM_MIN_KMER || !s->symmetric))
    return hm_set_error(HM_EINVAL,"the table is not strand-symmetric (or k < %d): the symmetric scan "
                                  "would not give the reference's answer",HM_SYMM_MIN_KMER);
  return HM_OK;
}

/* a symmetric run or listing whose status word is not 0: the fingerprint was fooled (2^-128) or a cut missed a run
 * boundary.  The direct passes are always right: HM_OK to fall back to them, unless the symmetric scan was forced */
static int symm_failed(hm_scan *s, int forced, uint64_t status)
{ if (forced)
    return hm_set_error(HM_EINVAL,"symmetric scan failed its own checks (status %llu)",(unsigned long long) status);
  s->symmetric = 0; s->symm_ready = 0;
  return HM_OK;
}

extern "C" int hm_scan_run_path(hm_scan *s, int path, int64_t *plot, hm_scan_stats *stats)
{ int symm = 0, forced = 0, rc;
  uint64_t status = 0;
  if (s->invalid)
    return hm_set_error(HM_EINVAL,"this scan was left unusable by a failed conditioning");
  if ((rc = choose_route(s,path,&symm,&forced)) != HM_OK)
    return rc;
  if (s->streamed)
    return run_stream(s,plot,stats);
  if (symm && ((rc = run_symm(s,plot,stats,&status)) != HM_OK || status == 0 ||
               (rc = symm_failed(s,forced,status)) != HM_OK))
    return rc;
  return run_direct(s,plot,stats);
}

extern "C" int hm_scan_run(hm_scan *s, int64_t *plot, hm_scan_stats *stats)
{ return hm_scan_run_path(s,HM_PATH_AUTO,plot,stats); }

/* extract / download need the incidence array and the recorded partners of the direct passes */
static int need_direct_results(hm_scan *s)
{ if (s->ran)
    return HM_OK;
  int64_t *tmp = (int64_t *) malloc(sizeof(int64_t)*HM_PLOT_CELLS);
  if (tmp == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory");
  int rc = run_direct(s,tmp,NULL);
  free(tmp);
  return rc;
}

static int rec_cmp(const void *a, const void *b)
{ const hm_pair_rec *x = (const hm_pair_rec *) a, *y = (const hm_pair_rec *) b;
  if (x->smudge != y->smudge) return (x->smudge < y->smudge ? -1 : 1);
  if (x->key_hi != y->key_hi) return (x->key_hi < y->key_hi ? -1 : 1);
  if (x->key_lo != y->key_lo) return (x->key_lo < y->key_lo ? -1 : 1);
  if (x->pos != y->pos)       return (x->pos < y->pos ? -1 : 1);
  return ((int) x->alt - (int) y->alt);
}

/* the order hm_scan_extract returns: qsort with rec_cmp.  Its time depends on the order the records arrive in, so
 * for long lists a stable counting pass by (smudge, first 8 bases) puts every record into its final bucket first
 * and qsort only has to order the buckets' insides.  configs[1] (2.6e7 records, the host of an H100 machine): a
 * whole call took 6.9-7.3 s on the direct route and 7.7-8.8 s on the symmetric one (half of its records, the
 * mirror images, come in no key order) with qsort alone, 4.7-4.8 s on either with the pass.  The result does not
 * depend on the pass (without host memory for its copy the records go to qsort as they are).                  */
static void sort_records(hm_pair_rec *r, int64_t n)
{ if (n >= (1 << 16))
    { uint32_t top = 0;
      for (int64_t i = 0; i < n; i++)
        if (r[i].smudge > top) top = r[i].smudge;
      int32_t *rank = top <= 0xffff ? (int32_t *) calloc((size_t) top+1,sizeof(int32_t)) : NULL;
      if (rank != NULL)
        { int32_t nl = 0;
          int     b  = 16;
          for (int64_t i = 0; i < n; i++)
            rank[r[i].smudge] = 1;
          for (uint32_t l = 0; l <= top; l++)                /* used labels in ascending order -> 0, 1, ... */
            rank[l] = rank[l] ? nl++ : -1;
          while (b > 4 && ((int64_t) nl << b) > (1ll << 22))
            b -= 1;
          int64_t     nb  = (int64_t) nl << b;
          int64_t    *at  = (int64_t *) calloc((size_t) nb+1,sizeof(int64_t));
          hm_pair_rec *o  = (hm_pair_rec *) malloc(sizeof(hm_pair_rec)*(size_t) n);
          if (at != NULL && o != NULL)
            { for (int64_t i = 0; i < n; i++)
                at[1 + ((int64_t) rank[r[i].smudge] << b) + (int64_t) (r[i].key_hi >> (64-b))] += 1;
              for (int64_t k = 0; k < nb; k++)
                at[k+1] += at[k];
              for (int64_t i = 0; i < n; i++)
                o[at[((int64_t) rank[r[i].smudge] << b) + (int64_t) (r[i].key_hi >> (64-b))]++] = r[i];
              memcpy(r,o,sizeof(hm_pair_rec)*(size_t) n);
            }
          free(at); free(o); free(rank);
        }
    }
  qsort(r,(size_t) n,sizeof(hm_pair_rec),rec_cmp);
}

/* the direct route of hm_scan_extract: the incidence array and recorded partners of the direct passes (run first if
 * the last run did not leave them).  Two launches per GPU: count, then fill.                                    */
static int extract_direct(hm_scan *s, const uint16_t *pixmap, hm_pair_rec **out, int64_t *n_out)
{ int G = s->ngpu, rc = HM_OK;
  if ((rc = need_direct_results(s)) != HM_OK)
    return rc;
  int64_t      total = 0, cnts[HM_MAX_GPUS];
  hm_pair_rec *d_out[HM_MAX_GPUS];
  uint16_t    *d_pix[HM_MAX_GPUS];
  unsigned long long *d_cnt[HM_MAX_GPUS];
  cudaError_t  e;
  memset(d_out,0,sizeof(d_out)); memset(d_pix,0,sizeof(d_pix)); memset(d_cnt,0,sizeof(d_cnt));
  for (int pass = 0; pass < 2 && rc == HM_OK; pass++)
    { for (int g = 0; g < G && rc == HM_OK; g++)
        { DevTable *D = s->d+g;
          TRY(cudaSetDevice(D->dev));
          if (pass == 0)
            { TRY(dev_alloc(D,&d_pix[g],sizeof(uint16_t)*HM_PLOT_CELLS));
              TRY(dev_alloc(D,&d_cnt[g],sizeof(unsigned long long)));
              TRY(cudaMemcpyAsync(d_pix[g],pixmap,sizeof(uint16_t)*HM_PLOT_CELLS,cudaMemcpyHostToDevice,D->st));
            }
          else if (cnts[g] > 0)
            TRY(dev_alloc(D,&d_out[g],sizeof(hm_pair_rec)*cnts[g]));
          TRY(cudaMemsetAsync(d_cnt[g],0,sizeof(unsigned long long),D->st));
          if (rc == HM_OK)
            { rc = hm_k_pass2_extract(D->keys,D->keys_lo,D->cnt,D->deg,D->up,s->idx64,D->lo,D->hi,d_pix[g],
                                      d_out[g],pass == 0 ? 0 : cnts[g],d_cnt[g],s->peer_mode ? &s->sh[g] : NULL,D->st);
              s->launches += (D->hi > D->lo);
            }
        }
      for (int g = 0; g < G && rc == HM_OK; g++)
        { unsigned long long c = 0;
          TRY(cudaSetDevice(s->d[g].dev));
          TRY(cudaMemcpyAsync(&c,d_cnt[g],sizeof(c),cudaMemcpyDeviceToHost,s->d[g].st));
          TRY(cudaStreamSynchronize(s->d[g].st));
          if (pass == 0) { cnts[g] = (int64_t) c; total += cnts[g]; }
        }
    }
  hm_pair_rec *host = rc == HM_OK ? (hm_pair_rec *) malloc(sizeof(hm_pair_rec)*(size_t) (total > 0 ? total : 1)) : NULL;
  if (host == NULL && rc == HM_OK)
    rc = hm_set_error(HM_ENOMEM,"out of host memory for %lld pair records",(long long) total);
  int64_t at = 0;
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      cudaSetDevice(D->dev);
      if (rc == HM_OK && cnts[g] > 0)
        { TRY(cudaMemcpy(host+at,d_out[g],sizeof(hm_pair_rec)*(size_t) cnts[g],cudaMemcpyDeviceToHost));
          at += cnts[g];
        }
      dev_free(D,d_out[g]); dev_free(D,d_pix[g]); dev_free(D,d_cnt[g]);
    }
  if (rc != HM_OK)
    { free(host); return rc; }
  *out = host; *n_out = total;
  return HM_OK;
}

/* appends c device records to the host list *host of *n records (capacity *cap, grown by doubling) */
static int append_records(hm_pair_rec **host, int64_t *n, int64_t *cap, const hm_pair_rec *d_rec, int64_t c)
{ if (*n + c > *cap)
    { int64_t      nh = 2 * *cap > *n + c ? 2 * *cap : *n + c;
      hm_pair_rec *h2 = (hm_pair_rec *) realloc(*host,sizeof(hm_pair_rec)*(size_t) nh);
      if (h2 == NULL)
        return hm_set_error(HM_ENOMEM,"out of host memory for %lld pair records",(long long) nh);
      *host = h2; *cap = nh;
    }
  cudaError_t e;
  if (c > 0 && (e = cudaMemcpy(*host + *n,d_rec,sizeof(hm_pair_rec)*(size_t) c,cudaMemcpyDeviceToHost)) != cudaSuccess)
    return hm_cuda_fail(e,"cudaMemcpy(pair records)");
  *n += c;
  return HM_OK;
}

/* the symmetric route: the candidates the last symmetric run left in each GPU's work area, listed by
 * hm_k_symm_extract against that GPU's replica (DESIGN.md §4a).  The record buffer of a GPU is what the device
 * budget leaves beyond the scan's own arrays (at most two records per candidate); the candidates go through it
 * in slices of half its records, and the host list grows slice by slice.  *status: the OR of the work areas'
 * status words afterwards (non-zero: the list must not be used).                                            */
static int extract_symm(hm_scan *s, const uint16_t *pixmap, hm_pair_rec **out, int64_t *n_out, uint64_t *status)
{ int     G = s->ngpu, rc = HM_OK;
  int64_t nc[HM_MAX_GPUS], c0[HM_MAX_GPUS], slice[HM_MAX_GPUS];
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      int64_t   room = s->budget - D->held;
      uint64_t  n_cand = 0;
      if (room < HM_EXTRACT_MIN_BYTES)
        return hm_set_error(HM_ENOMEM,"listing k-mer pairs needs at least %lld device bytes beside the scan's %lld on "
                            "GPU %d, but the device budget of %lld bytes leaves %lld",(long long) HM_EXTRACT_MIN_BYTES,
                            (long long) D->held,D->dev,(long long) s->budget,(long long) (room > 0 ? room : 0));
      HM_CUDA(cudaSetDevice(D->dev));
      if ((rc = hm_symm_status(D->symm_work,&D->symm_layout,&n_cand,NULL,D->st)) != HM_OK)
        return rc;
      nc[g] = (int64_t) n_cand < D->symm_layout.cand_cap ? (int64_t) n_cand : D->symm_layout.cand_cap;
      int64_t recs = (room - 2*(int64_t) HM_PLOT_CELLS - 256) / (int64_t) sizeof(hm_pair_rec);
      if (recs > 2*nc[g]) recs = 2*nc[g];
      slice[g] = recs/2 > 0 ? recs/2 : 1;
      c0[g] = 0;
    }
  hm_pair_rec *d_out[HM_MAX_GPUS], *host = NULL;
  uint16_t    *d_pix[HM_MAX_GPUS];
  unsigned long long *d_cnt[HM_MAX_GPUS];
  int64_t      total = 0, hcap = 0;
  memset(d_out,0,sizeof(d_out)); memset(d_pix,0,sizeof(d_pix)); memset(d_cnt,0,sizeof(d_cnt));
  for (int g = 0; g < G && rc == HM_OK; g++)
    { DevTable *D = s->d+g;
      cudaError_t e;
      TRY(cudaSetDevice(D->dev));
      TRY(dev_alloc(D,&d_pix[g],sizeof(uint16_t)*HM_PLOT_CELLS));
      TRY(dev_alloc(D,&d_cnt[g],256));
      TRY(dev_alloc(D,&d_out[g],sizeof(hm_pair_rec)*(2*slice[g])));
      TRY(cudaMemcpyAsync(d_pix[g],pixmap,sizeof(uint16_t)*HM_PLOT_CELLS,cudaMemcpyHostToDevice,D->st));
    }
  for (int more = 1; more && rc == HM_OK; )
    { int64_t c1[HM_MAX_GPUS];
      more = 0;
      for (int g = 0; g < G && rc == HM_OK; g++)             /* a slice on every GPU that has candidates left */
        { DevTable *D = s->d+g;
          c1[g] = c0[g] + slice[g] < nc[g] ? c0[g] + slice[g] : nc[g];
          if (c0[g] >= nc[g])
            continue;
          cudaError_t e;
          if ((e = cudaSetDevice(D->dev)) != cudaSuccess ||
              (e = cudaMemsetAsync(d_cnt[g],0,sizeof(unsigned long long),D->st)) != cudaSuccess)
            { rc = hm_cuda_fail(e,"extract slice"); break; }
          rc = hm_k_symm_extract(D->keys,D->keys_lo,D->cnt,s->n,D->bucket,s->bits,s->idx64,s->kmer,D->symm_work,
                                 &D->symm_layout,G > 1 ? &s->ssh[g] : NULL,d_pix[g],c0[g],c1[g],d_out[g],
                                 2*slice[g],d_cnt[g],D->st);
          s->launches += 1;
          more = 1;
        }
      for (int g = 0; g < G && rc == HM_OK; g++)
        { DevTable *D = s->d+g;
          unsigned long long c = 0;
          if (c0[g] >= nc[g])
            continue;
          cudaError_t e;
          if ((e = cudaSetDevice(D->dev)) != cudaSuccess ||
              (e = cudaMemcpyAsync(&c,d_cnt[g],sizeof(c),cudaMemcpyDeviceToHost,D->st)) != cudaSuccess ||
              (e = cudaStreamSynchronize(D->st)) != cudaSuccess)
            { rc = hm_cuda_fail(e,"extract_kernel"); break; }
          if ((int64_t) c > 2*slice[g])
            { rc = hm_set_error(HM_ECUDA,"extract_kernel listed %llu records for %lld candidates",c,
                                (long long) (c1[g]-c0[g]));
              break;
            }
          if ((rc = append_records(&host,&total,&hcap,d_out[g],(int64_t) c)) != HM_OK)
            break;
          c0[g] = c1[g];
        }
    }
  *status = 0;
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      uint64_t  st = 0;
      cudaSetDevice(D->dev);
      if (rc == HM_OK)
        { rc = hm_symm_status(D->symm_work,&D->symm_layout,NULL,&st,D->st);
          *status |= st;
        }
      dev_free(D,d_out[g]); dev_free(D,d_pix[g]); dev_free(D,d_cnt[g]);
    }
  if (rc == HM_OK && host == NULL && (host = (hm_pair_rec *) malloc(sizeof(hm_pair_rec))) == NULL)
    rc = hm_set_error(HM_ENOMEM,"out of host memory");
  if (rc != HM_OK)
    { free(host); return rc; }
  *out = host; *n_out = total;
  return HM_OK;
}

/* extract_kmer_pairs' output as a list (PloidyList.c:425-450).  The route follows hm_scan_run_path(HM_PATH_AUTO)'s
 * rule and HETMERS_PATH: the symmetric one lists the candidates of the last symmetric run (running one first if
 * the work areas do not hold a clean one), the direct one the direct passes' results; a symmetric run that fails
 * its own checks falls back to the direct route, as a run does.                                                */
extern "C" int hm_scan_extract(hm_scan *s, const uint16_t *pixmap, hm_pair_rec **out, int64_t *n_out)
{ int rc, symm = 0, forced = 0;
  if (s->streamed)
    return hm_set_error(HM_EUNSUPPORTED,"listing k-mer pairs needs the direct passes' arrays, and this table does not "
                                        "fit in device memory (budget %lld bytes)",(long long) s->budget);
  if (s->invalid)
    return hm_set_error(HM_EINVAL,"this scan was left unusable by a failed conditioning");
  if ((rc = choose_route(s,HM_PATH_AUTO,&symm,&forced)) != HM_OK)
    return rc;
  hm_pair_rec *host = NULL;
  int64_t      total = 0;
  if (symm)
    { uint64_t status = 0;
      if (!s->symm_ready)
        { int64_t *tmp = (int64_t *) malloc(sizeof(int64_t)*HM_PLOT_CELLS);
          if (tmp == NULL)
            return hm_set_error(HM_ENOMEM,"out of host memory");
          rc = run_symm(s,tmp,NULL,&status);
          free(tmp);
          if (rc != HM_OK)
            return rc;
        }
      if (status == 0)
        { if ((rc = extract_symm(s,pixmap,&host,&total,&status)) != HM_OK)
            return rc;
          if (status != 0)
            { free(host); host = NULL; total = 0; }
        }
      if (status != 0)
        { if ((rc = symm_failed(s,forced,status)) != HM_OK)
            return rc;
          symm = 0;
        }
    }
  if (!symm && (rc = extract_direct(s,pixmap,&host,&total)) != HM_OK)
    return rc;
  sort_records(host,total);                                       /* deterministic order */
  *out = host; *n_out = total;
  return HM_OK;
}

/* ------------------------------------------------------------------ pair files (DESIGN.md §6c) ---- */

/* what a pair-file call holds on each GPU: the pixmap, counters (one per window of a pass), the histogram, the
 * label bounds of a window, and the window buffers a (records) and b (the sort's other buffer and scratch, then
 * the window's text)                                                                                         */
typedef struct
  { uint16_t           *pix;
    unsigned long long *ctr, *hist, *bounds;
    hm_pair_rec        *a, *b;
    int64_t             held0, peak0;
  } PairBufs;

#define PAIR_SMALL_BYTES (2*(int64_t) HM_PLOT_CELLS + 256)    /* pixmap and counters, beside the window model */

static int pairs_hist_bits(int kmer) { return 2*kmer < HM_COND_HIST_BITS ? 2*kmer : HM_COND_HIST_BITS; }

static void pairs_free(hm_scan *s, PairBufs *B)
{ for (int g = 0; g < s->ngpu; g++)
    { DevTable *D = s->d+g;
      cudaSetDevice(D->dev);
      dev_free(D,B[g].pix); dev_free(D,B[g].ctr); dev_free(D,B[g].hist); dev_free(D,B[g].bounds);
      dev_free(D,B[g].a); dev_free(D,B[g].b);
      B[g].pix = NULL; B[g].ctr = NULL; B[g].hist = NULL; B[g].bounds = NULL; B[g].a = NULL; B[g].b = NULL;
    }
}

/* the device budget of the call, per GPU: the explicit one (hm_set_device_budget) or the scan's */
static int64_t pairs_budget(const hm_scan *s) { return g_budget > 0 ? g_budget : s->budget; }

/* The histogram sweep over each GPU's own candidates (symmetric route) or range (direct route), the route chosen
 * as hm_scan_extract chooses it: a symmetric run first when the work areas hold no clean one, and the direct route
 * when that run or the sweep ends with a dirty status word.  Allocates B[g].pix / ctr / hist / bounds (n_labels
 * + 1 label bounds).  hg: host int64[G][2^hb], each GPU's histogram; *symm_out: the route taken.                */
static int pairs_histogram(hm_scan *s, const uint16_t *pixmap, int n_labels, PairBufs *B, int64_t *hg,
                           int *symm_out)
{ int symm = 0, forced = 0, rc, G = s->ngpu;
  const int     hb = pairs_hist_bits(s->kmer);
  const int64_t np = (int64_t) 1 << hb;
  uint64_t      status = 0;
  if ((rc = choose_route(s,HM_PATH_AUTO,&symm,&forced)) != HM_OK)
    return rc;
  if (symm && !s->symm_ready)
    { int64_t *tmp = (int64_t *) malloc(sizeof(int64_t)*HM_PLOT_CELLS);
      if (tmp == NULL)
        return hm_set_error(HM_ENOMEM,"out of host memory");
      rc = run_symm(s,tmp,NULL,&status);
      free(tmp);
      if (rc != HM_OK)
        return rc;
    }
  cudaError_t e;
  rc = HM_OK;
  for (int g = 0; g < G && rc == HM_OK; g++)
    { DevTable *D = s->d+g;
      TRY(cudaSetDevice(D->dev));
      TRY(dev_alloc(D,&B[g].pix,sizeof(uint16_t)*HM_PLOT_CELLS));
      TRY(dev_alloc(D,&B[g].ctr,256));
      TRY(dev_alloc(D,&B[g].hist,sizeof(unsigned long long)*np));
      TRY(dev_alloc(D,&B[g].bounds,sizeof(unsigned long long)*2*(n_labels+1)));
      TRY(cudaMemcpyAsync(B[g].pix,pixmap,sizeof(uint16_t)*HM_PLOT_CELLS,cudaMemcpyHostToDevice,D->st));
      TRY(cudaMemsetAsync(B[g].hist,0,sizeof(unsigned long long)*np,D->st));
    }
  if (rc != HM_OK)
    return rc;
  if (symm && status == 0)
    { for (int g = 0; g < G && rc == HM_OK; g++)
        { DevTable *D = s->d+g;
          TRY(cudaSetDevice(D->dev));
          if (rc == HM_OK)
            rc = hm_symm_pairs_sweep(D->keys,D->keys_lo,D->cnt,s->n,D->bucket,s->bits,s->idx64,s->kmer,D->symm_work,
                                     &D->symm_layout,G > 1 ? &s->ssh[g] : NULL,B[g].pix,hb,B[g].hist,0,0,NULL,0,
                                     NULL,D->st);
          s->launches += 1;
        }
      for (int g = 0; g < G && rc == HM_OK; g++)
        { uint64_t st = 0;
          TRY(cudaSetDevice(s->d[g].dev));
          if (rc == HM_OK && (rc = hm_symm_status(s->d[g].symm_work,&s->d[g].symm_layout,NULL,&st,s->d[g].st)) == HM_OK)
            status |= st;
        }
      if (rc != HM_OK)
        return rc;
    }
  if (symm && status != 0)
    { if ((rc = symm_failed(s,forced,status)) != HM_OK)
        return rc;
      symm = 0;
    }
  if (!symm)
    { if ((rc = need_direct_results(s)) != HM_OK)
        return rc;
      for (int g = 0; g < G && rc == HM_OK; g++)
        { DevTable *D = s->d+g;
          TRY(cudaSetDevice(D->dev));
          TRY(cudaMemsetAsync(B[g].hist,0,sizeof(unsigned long long)*np,D->st));
          if (rc == HM_OK)
            rc = hm_pass2_pairs_sweep(D->keys,D->keys_lo,D->cnt,D->deg,D->up,s->idx64,D->lo,D->hi,B[g].pix,hb,
                                      B[g].hist,0,0,NULL,0,NULL,s->peer_mode ? &s->sh[g] : NULL,D->st);
          s->launches += (D->hi > D->lo);
        }
    }
  for (int g = 0; g < G && rc == HM_OK; g++)
    { TRY(cudaSetDevice(s->d[g].dev));
      TRY(cudaMemcpyAsync(hg+g*np,B[g].hist,sizeof(int64_t)*np,cudaMemcpyDeviceToHost,s->d[g].st));
      TRY(cudaStreamSynchronize(s->d[g].st));
    }
  *symm_out = symm;
  return rc;
}

/* the records of one window a pass lists on GPU g, into out (cap records), counted in *ctr */
static int pairs_window_sweep(hm_scan *s, int symm, int g, const PairBufs *B, uint64_t p0, uint64_t p1,
                              hm_pair_rec *out, int64_t cap, unsigned long long *ctr)
{ DevTable *D = s->d+g;
  const int hb = pairs_hist_bits(s->kmer);
  s->launches += 1;
  if (symm)
    return hm_symm_pairs_sweep(D->keys,D->keys_lo,D->cnt,s->n,D->bucket,s->bits,s->idx64,s->kmer,D->symm_work,
                               &D->symm_layout,s->ngpu > 1 ? &s->ssh[g] : NULL,B[g].pix,hb,NULL,p0,p1,out,cap,ctr,
                               D->st);
  return hm_pass2_pairs_sweep(D->keys,D->keys_lo,D->cnt,D->deg,D->up,s->idx64,D->lo,D->hi,B[g].pix,hb,NULL,p0,p1,
                              out,cap,ctr,s->peer_mode ? &s->sh[g] : NULL,D->st);
}

/* The writer thread: the text of a window reaches the host in pieces (two pinned buffers, alternating); each
 * piece's part of every label segment of its window is pwritten at its offset in the label's file.           */
typedef struct { int s; int64_t text_off, bytes, file_off; } PairSeg;

typedef struct
  { pthread_mutex_t mu;
    pthread_cond_t  cv;
    const int      *fd;
    char           *buf[2];
    int             full[2], quit, err;
    int64_t         t0[2], n[2];              /* the piece holds text bytes [t0, t0 + n) of its window */
    PairSeg        *seg[2];
    int             nseg[2];
    double          busy_ms;
  } PairWriter;

static void *pairs_writer_main(void *arg)
{ PairWriter *W = (PairWriter *) arg;
  for (int i = 0; ; i ^= 1)
    { pthread_mutex_lock(&W->mu);
      while (!W->full[i] && !W->quit)
        pthread_cond_wait(&W->cv,&W->mu);
      if (!W->full[i])
        { pthread_mutex_unlock(&W->mu); return NULL; }
      pthread_mutex_unlock(&W->mu);
      const double t = now_ms();
      for (int k = 0; k < W->nseg[i] && !W->err; k++)
        { const PairSeg *q = W->seg[i]+k;
          int64_t a = q->text_off > W->t0[i] ? q->text_off : W->t0[i];
          int64_t b = q->text_off+q->bytes < W->t0[i]+W->n[i] ? q->text_off+q->bytes : W->t0[i]+W->n[i];
          while (a < b && !W->err)
            { ssize_t w = pwrite(W->fd[q->s-1],W->buf[i]+(a-W->t0[i]),(size_t) (b-a),(off_t) (q->file_off+a-q->text_off));
              if (w < 0 && errno == EINTR) continue;
              if (w <= 0) { W->err = w < 0 ? errno : EIO; break; }
              a += w;
            }
        }
      pthread_mutex_lock(&W->mu);
      W->busy_ms += now_ms()-t;
      W->full[i] = 0;
      pthread_cond_broadcast(&W->cv);
      pthread_mutex_unlock(&W->mu);
    }
}

/* waits until piece i is free; the time waited goes to *ms */
static void pairs_writer_wait(PairWriter *W, int i, double *ms)
{ const double t = now_ms();
  pthread_mutex_lock(&W->mu);
  while (W->full[i])
    pthread_cond_wait(&W->cv,&W->mu);
  pthread_mutex_unlock(&W->mu);
  *ms += now_ms()-t;
}

static void pairs_remove(int n_labels, const char *const *paths)
{ for (int s = 0; s < n_labels; s++)
    unlink(paths[s]);
}

/* the most records one window may hold in `bytes` (hm_pairs_window_bytes, bisection); -1 below the fixed part */
static int64_t pairs_room(int kmer, int64_t bytes)
{ if (hm_pairs_window_bytes(kmer,0) > bytes)
    return -1;
  int64_t lo = 0, hi = bytes/24 > 1 ? bytes/24 : 1;
  while (lo < hi)
    { const int64_t m = lo + (hi-lo+1)/2;
      if (hm_pairs_window_bytes(kmer,m) <= bytes) lo = m; else hi = m-1;
    }
  return lo;
}

/* the room of the call on every GPU: the smallest, in records (-1 if some GPU cannot hold the fixed part);
 * *budget_out: the smallest device bytes the call may hold beside the scan                               */
static int64_t pairs_min_room(hm_scan *s, const PairBufs *B, int64_t *budget_out)
{ int64_t room = -2, budget = 0;
  for (int g = 0; g < s->ngpu; g++)
    { const DevTable *D = s->d+g;
      const int64_t own  = B != NULL ? dev_bytes(D,B[g].pix) + dev_bytes(D,B[g].ctr) + dev_bytes(D,B[g].hist) +
                                       dev_bytes(D,B[g].bounds) : 0;
      const int64_t left = pairs_budget(s) - (D->held - own);
      const int64_t r    = pairs_room(s->kmer,left - PAIR_SMALL_BYTES);
      if (room == -2 || r < room) room = r;
      if (g == 0 || left < budget) budget = left;
    }
  *budget_out = budget;
  return room;
}

extern "C" int hm_scan_pairs_hist(hm_scan *s, const uint16_t *pixmap, uint64_t *hist)
{ if (s == NULL || pixmap == NULL || hist == NULL)
    return hm_set_error(HM_EINVAL,"hm_scan_pairs_hist: NULL argument");
  if (s->streamed)
    return hm_set_error(HM_EUNSUPPORTED,"listing k-mer pairs needs the direct passes' arrays, and this table does not "
                                        "fit in device memory (budget %lld bytes)",(long long) s->budget);
  if (s->invalid)
    return hm_set_error(HM_EINVAL,"this scan was left unusable by a failed conditioning");
  const int64_t np = (int64_t) 1 << pairs_hist_bits(s->kmer);
  PairBufs B[HM_MAX_GPUS];
  memset(B,0,sizeof(B));
  int64_t *hg = (int64_t *) malloc(sizeof(int64_t)*(size_t) (np*s->ngpu));
  if (hg == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory");
  int symm = 0, rc = pairs_histogram(s,pixmap,0,B,hg,&symm);
  pairs_free(s,B);
  if (rc == HM_OK)
    for (int64_t p = 0; p < np; p++)
      { uint64_t t = 0;
        for (int g = 0; g < s->ngpu; g++) t += (uint64_t) hg[g*np+p];
        hist[p] = t;
      }
  free(hg);
  return rc;
}

extern "C" int hm_scan_write_pairs(hm_scan *s, const uint16_t *pixmap, int n_labels, const char *const *paths,
                                   hm_pairs_stats *st)
{ hm_pairs_stats S;
  memset(&S,0,sizeof(S));
  if (st != NULL) *st = S;
  if (s == NULL || pixmap == NULL || n_labels < 0 || (n_labels > 0 && paths == NULL))
    return hm_set_error(HM_EINVAL,"hm_scan_write_pairs: bad arguments");
  for (int l = 0; l < n_labels; l++)
    if (paths[l] == NULL)
      return hm_set_error(HM_EINVAL,"hm_scan_write_pairs: label %d has no path",l+1);
  if (s->streamed)
    return hm_set_error(HM_EUNSUPPORTED,"listing k-mer pairs needs the direct passes' arrays, and this table does not "
                                        "fit in device memory (budget %lld bytes)",(long long) s->budget);
  if (s->invalid)
    return hm_set_error(HM_EINVAL,"this scan was left unusable by a failed conditioning");
  const double  t_all = now_ms();
  const int     G = s->ngpu, kmer = s->kmer, hb = pairs_hist_bits(kmer);
  const int64_t np = (int64_t) 1 << hb, line = kmer+5;
  int64_t       budget = 0, room = pairs_min_room(s,NULL,&budget);
  if (room < 0)
    return hm_set_error(HM_ENOMEM,"writing the pair files needs %lld device bytes per GPU before any record beside the "
                        "scan's own; the device budget of %lld bytes leaves %lld",
                        (long long) (hm_pairs_window_bytes(kmer,0)+PAIR_SMALL_BYTES),(long long) pairs_budget(s),
                        (long long) (budget > 0 ? budget : 0));

  PairBufs B[HM_MAX_GPUS];
  memset(B,0,sizeof(B));
  for (int g = 0; g < G; g++)
    { B[g].held0 = s->d[g].held; B[g].peak0 = s->d[g].peak; s->d[g].peak = s->d[g].held; }
  int64_t *hg = (int64_t *) malloc(sizeof(int64_t)*(size_t) (np*G));
  int64_t *hsum = (int64_t *) malloc(sizeof(int64_t)*(size_t) np);
  int64_t *cuts = NULL, *before = (int64_t *) calloc((size_t) n_labels+1,sizeof(int64_t));
  int64_t *bh = (int64_t *) malloc(sizeof(int64_t)*(size_t) ((np+1)*G));      /* per GPU: records below prefix p */
  int     *fd = (int *) malloc(sizeof(int)*(size_t) (n_labels > 0 ? n_labels : 1));
  uint64_t *bounds = (uint64_t *) malloc(sizeof(uint64_t)*2*(size_t) (n_labels+1));
  PairSeg  *segs = (PairSeg *) malloc(sizeof(PairSeg)*3*(size_t) (n_labels+1));   /* the two pieces', a window's */
  char     *pin = NULL;
  int       rc = HM_OK, symm = 0, files = 0, writer = 0;
  int64_t   P = 0, piece = 0, ra = 0;
  PairWriter W;
  pthread_t  th;
  cudaError_t e;
  memset(&W,0,sizeof(W));
  if (hg == NULL || hsum == NULL || before == NULL || bh == NULL || fd == NULL || bounds == NULL || segs == NULL)
    rc = hm_set_error(HM_ENOMEM,"out of host memory");

  double t = now_ms();
  if (rc == HM_OK)
    rc = pairs_histogram(s,pixmap,n_labels,B,hg,&symm);
  S.path = symm ? HM_PATH_SYMM : HM_PATH_DIRECT;
  if (rc == HM_OK)
    { for (int64_t p = 0; p < np; p++)
        { int64_t c = 0;
          for (int g = 0; g < G; g++) c += hg[g*np+p];
          hsum[p] = c;
        }
      for (int g = 0; g < G; g++)
        { bh[g*(np+1)] = 0;
          for (int64_t p = 0; p < np; p++) bh[g*(np+1)+p+1] = bh[g*(np+1)+p] + hg[g*np+p];
        }
      room = pairs_min_room(s,B,&budget);            /* (the direct passes may have been run for the route) */
      S.room = room; S.budget = budget;
      if (room < 0)
        rc = hm_set_error(HM_ENOMEM,"writing the pair files needs %lld device bytes per GPU before any record beside "
                          "the scan's own; the device budget of %lld bytes leaves %lld",
                          (long long) (hm_pairs_window_bytes(kmer,0)+PAIR_SMALL_BYTES),(long long) pairs_budget(s),
                          (long long) (budget > 0 ? budget : 0));
    }
  if (rc == HM_OK && (rc = hm_pair_windows(hsum,np,G,room,&P,NULL)) == HM_OK)
    { if ((cuts = (int64_t *) malloc(sizeof(int64_t)*(size_t) (P*G+1))) == NULL)
        rc = hm_set_error(HM_ENOMEM,"out of host memory");
      else
        rc = hm_pair_windows(hsum,np,G,room,&P,cuts);
    }
  S.ms_hist = now_ms()-t;
  if (rc != HM_OK)                                     /* nothing written: HM_ENOMEM here is the plan's refusal */
    goto done;
  S.planned = 1;
  S.passes = P; S.windows = P*G;

  /* the window buffers, for the largest window (at most room records): a = records, b = the sort's other buffer
   * and its scratch, then the window's text                                                                  */
  { int64_t most = 0, text = 0, scratch = 0, rb = 0;
    for (int64_t j = 0; j < P*G; j++)
      { int64_t c = 0;
        for (int64_t p = cuts[j]; p < cuts[j+1]; p++) c += hsum[p];
        if (c > most) most = c;
        S.records += c;
      }
    scratch = hm_pairs_sort_scratch_bytes(most);
    text    = most*line;
    piece   = text < (64ll << 20) ? (text > 0 ? text : 1) : (64ll << 20);
    ra      = (24*most + 511) & ~511ll;
    rb      = ra + scratch > text ? ra + scratch : text;
    for (int g = 0; g < G && rc == HM_OK; g++)
      { DevTable *D = s->d+g;
        TRY(cudaSetDevice(D->dev));
        TRY(dev_alloc(D,&B[g].a,ra > 0 ? ra : 512));
        TRY(dev_alloc(D,&B[g].b,rb > 0 ? rb : 512));
      }
    if (rc == HM_OK)
      rc = sync_all(s,"pair-file buffers");
    if (rc == HM_OK && (e = cudaHostAlloc((void **) &pin,(size_t) (2*piece),cudaHostAllocDefault)) != cudaSuccess)
      rc = hm_cuda_fail(e,"cudaHostAlloc(pair-file pieces)");
    if (rc != HM_OK)
      goto done;
  }

  /* every label file created (or truncated) before pass 0, so that a label with no pair gets an empty file */
  for (int l = 0; l < n_labels && rc == HM_OK; l++)
    { fd[l] = open(paths[l],O_WRONLY | O_CREAT | O_TRUNC,0666);
      if (fd[l] < 0)
        rc = hm_set_error(HM_EIO,"cannot create the pair file %s: %s",paths[l],strerror(errno));
      else
        files = l+1;
    }
  if (rc != HM_OK)
    goto done;
  pthread_mutex_init(&W.mu,NULL);
  pthread_cond_init(&W.cv,NULL);
  W.fd = fd; W.buf[0] = pin; W.buf[1] = pin+piece; W.seg[0] = segs; W.seg[1] = segs+(n_labels+1);
  if (pthread_create(&th,NULL,pairs_writer_main,&W) != 0)
    { rc = hm_set_error(HM_EIO,"cannot start the pair-file writer thread");
      goto done;
    }
  writer = 1;

  { int side = 0;
    for (int64_t p = 0; p < P && rc == HM_OK; p++)
      { int64_t share[HM_MAX_GPUS][HM_MAX_GPUS], nwin[HM_MAX_GPUS];   /* [owner][lister] */
        unsigned long long got[HM_MAX_GPUS][HM_MAX_GPUS];
        t = now_ms();
        for (int o = 0; o < G; o++)
          { const int64_t j = p*G + o;
            nwin[o] = 0;
            for (int h = 0; h < G; h++)
              { share[o][h] = bh[h*(np+1)+cuts[j+1]] - bh[h*(np+1)+cuts[j]];
                nwin[o] += share[o][h];
              }
          }
        /* each GPU lists its share of every window of the pass: its own window's straight into its buffer, the
         * others' into b and from there to the owner, after the shares of the GPUs before it                    */
        for (int h = 0; h < G && rc == HM_OK; h++)
          { DevTable *D = s->d+h;
            TRY(cudaSetDevice(D->dev));
            TRY(cudaMemsetAsync(B[h].ctr,0,sizeof(unsigned long long)*G,D->st));
            for (int o = 0; o < G && rc == HM_OK; o++)
              { const int64_t j = p*G + o;
                int64_t off = 0;
                for (int q = 0; q < h; q++) off += share[o][q];
                if (share[o][h] == 0)
                  continue;
                rc = pairs_window_sweep(s,symm,h,B,(uint64_t) cuts[j],(uint64_t) cuts[j+1],o == h ? B[o].a+off : B[h].b,
                                        share[o][h],B[h].ctr+o);
                if (o != h)
                  TRY(cudaMemcpyPeerAsync(B[o].a+off,s->d[o].dev,B[h].b,D->dev,sizeof(hm_pair_rec)*share[o][h],D->st));
              }
            TRY(cudaMemcpyAsync(got[h],B[h].ctr,sizeof(unsigned long long)*G,cudaMemcpyDeviceToHost,D->st));
          }
        if (rc == HM_OK)
          rc = sync_all(s,"pair-file window sweep");
        for (int h = 0; h < G && rc == HM_OK; h++)
          { uint64_t stw = 0;
            if (symm && (rc = hm_symm_status(s->d[h].symm_work,&s->d[h].symm_layout,NULL,&stw,s->d[h].st)) != HM_OK)
              break;
            if (stw != 0)
              rc = hm_set_error(HM_ECUDA,"the symmetric scan failed its own checks while listing the pairs of pass "
                                "%lld (status %llu)",(long long) p,(unsigned long long) stw);
            for (int o = 0; o < G && rc == HM_OK; o++)
              if ((int64_t) got[h][o] != share[o][h])
                rc = hm_set_error(HM_ECUDA,"window %lld: GPU %d listed %llu records, its histogram %lld",
                                  (long long) (p*G+o),s->d[h].dev,got[h][o],(long long) share[o][h]);
          }
        S.ms_list += now_ms()-t;
        if (rc != HM_OK)
          break;

        t = now_ms();
        for (int o = 0; o < G && rc == HM_OK; o++)
          { DevTable *D = s->d+o;
            const int64_t n = nwin[o];
            int in_alt = 0;
            TRY(cudaSetDevice(D->dev));
            if (rc == HM_OK && n > 0)
              rc = hm_k_pairs_sort(B[o].a,B[o].b,n,(char *) B[o].b + ra,dev_bytes(D,B[o].b)-ra,&in_alt,D->st);
            if (in_alt)
              TRY(cudaMemcpyAsync(B[o].a,B[o].b,sizeof(hm_pair_rec)*n,cudaMemcpyDeviceToDevice,D->st));
            TRY(cudaMemsetAsync(B[o].bounds,0,sizeof(unsigned long long)*2*(n_labels+1),D->st));
            if (rc == HM_OK)
              rc = hm_k_pairs_label_bounds(B[o].a,n,n_labels,(uint64_t *) B[o].bounds,D->st);
            s->launches += (n > 0) ? 2 : 0;
          }
        if (rc == HM_OK)
          rc = sync_all(s,"pair-file sort");
        S.ms_sort += now_ms()-t;
        t = now_ms();
        for (int o = 0; o < G && rc == HM_OK; o++)
          { TRY(cudaSetDevice(s->d[o].dev));
            if (rc == HM_OK)
              rc = hm_k_pairs_format(B[o].a,nwin[o],kmer,(char *) B[o].b,s->d[o].st);
            s->launches += (nwin[o] > 0);
          }
        if (rc == HM_OK)
          rc = sync_all(s,"pair-file format");
        S.ms_format += now_ms()-t;

        /* window by window, in file order: the label segments, and the text through the pinned pieces */
        for (int o = 0; o < G && rc == HM_OK; o++)
          { DevTable *D = s->d+o;
            const int64_t n = nwin[o];
            int           nseg = 0;
            int64_t       lines = 0;
            TRY(cudaSetDevice(D->dev));
            TRY(cudaMemcpy(bounds,B[o].bounds,sizeof(uint64_t)*2*(n_labels+1),cudaMemcpyDeviceToHost));
            if (rc != HM_OK)
              break;
            PairSeg *ws = segs + 2*(n_labels+1);
            for (int l = 1; l <= n_labels; l++)
              { const int64_t c = (int64_t) (bounds[2*l+1] - bounds[2*l]);
                if (c <= 0)
                  continue;
                ws[nseg].s = l; ws[nseg].text_off = (int64_t) bounds[2*l]*line; ws[nseg].bytes = c*line;
                ws[nseg].file_off = before[l]*line;
                before[l] += c; lines += c; nseg += 1;
              }
            if (lines != n)
              { rc = hm_set_error(HM_EINVAL,"window %lld holds %lld records with a label beyond the %d labels",
                                  (long long) (p*G+o),(long long) (n-lines),n_labels);
                break;
              }
            for (int64_t t0 = 0; t0 < n*line && rc == HM_OK; t0 += piece)
              { const int64_t m = n*line - t0 < piece ? n*line - t0 : piece;
                pairs_writer_wait(&W,side,&S.ms_write);
                t = now_ms();
                TRY(cudaMemcpyAsync(W.buf[side],(char *) B[o].b + t0,(size_t) m,cudaMemcpyDeviceToHost,D->st));
                TRY(cudaStreamSynchronize(D->st));
                S.ms_d2h += now_ms()-t;
                if (rc != HM_OK)
                  break;
                memcpy(W.seg[side],ws,sizeof(PairSeg)*(size_t) nseg);
                pthread_mutex_lock(&W.mu);
                W.t0[side] = t0; W.n[side] = m; W.nseg[side] = nseg; W.full[side] = 1;
                pthread_cond_broadcast(&W.cv);
                pthread_mutex_unlock(&W.mu);
                side ^= 1;
              }
          }
      }
  }

done:
  if (writer)
    { pairs_writer_wait(&W,0,&S.ms_write);
      pairs_writer_wait(&W,1,&S.ms_write);
      pthread_mutex_lock(&W.mu);
      W.quit = 1;
      pthread_cond_broadcast(&W.cv);
      pthread_mutex_unlock(&W.mu);
      pthread_join(th,NULL);
      S.ms_writer_busy = W.busy_ms;
      if (rc == HM_OK && W.err != 0)
        rc = hm_set_error(HM_EIO,"writing the pair files: %s",strerror(W.err));
    }
  if (W.fd != NULL)
    { pthread_mutex_destroy(&W.mu); pthread_cond_destroy(&W.cv); }
  for (int l = 0; l < files; l++)
    if (close(fd[l]) != 0 && rc == HM_OK)
      rc = hm_set_error(HM_EIO,"closing the pair file %s: %s",paths[l],strerror(errno));
  if (rc != HM_OK && files > 0)                  /* no partial output is left looking complete */
    pairs_remove(n_labels,paths);
  if (pin != NULL)
    cudaFreeHost(pin);
  pairs_free(s,B);
  for (int g = 0; g < G; g++)
    { DevTable *D = s->d+g;
      if (D->peak - B[g].held0 > S.peak_bytes) S.peak_bytes = D->peak - B[g].held0;
      if (B[g].peak0 > D->peak) D->peak = B[g].peak0;
    }
  free(hg); free(hsum); free(cuts); free(before); free(bh); free(fd); free(bounds); free(segs);
  S.ms_total = now_ms()-t_all;
  if (st != NULL) *st = S;
  return rc;
}

extern "C" int hm_hetmers_host(const hm_host_table *t, const int *dev, int n_gpus,
                               int64_t *plot, hm_scan_stats *stats)
{ hm_scan *s = NULL;
  int rc = hm_scan_create(t,dev,n_gpus,&s);
  if (rc != HM_OK)
    return rc;
  rc = hm_scan_run(s,plot,stats);
  hm_scan_destroy(s);
  return rc;
}

extern "C" int hm_scan_download(hm_scan *s, uint64_t *keys, uint64_t *keys_lo, uint16_t *cnt, uint8_t *deg)
{ DevTable *D = s->d;
  if (s->streamed)
    return hm_set_error(HM_EUNSUPPORTED,"a streamed scan holds no table on the device to download");
  HM_CUDA(cudaSetDevice(D->dev));
  HM_CUDA(cudaStreamSynchronize(D->st));
  if (keys != NULL)
    HM_CUDA(cudaMemcpy(keys,D->keys,sizeof(uint64_t)*(size_t) s->n,cudaMemcpyDeviceToHost));
  if (keys_lo != NULL && D->keys_lo != NULL)
    HM_CUDA(cudaMemcpy(keys_lo,D->keys_lo,sizeof(uint64_t)*(size_t) s->n,cudaMemcpyDeviceToHost));
  if (cnt != NULL)
    HM_CUDA(cudaMemcpy(cnt,D->cnt,sizeof(uint16_t)*(size_t) s->n,cudaMemcpyDeviceToHost));
  if (deg != NULL)                      /* every owner's slice (identical copies in dense mode) */
    { int rc = need_direct_results(s);  /* (the symmetric scan never materialises the array) */
      if (rc != HM_OK) return rc;
    }
  if (deg != NULL)
    for (int g = 0; g < s->ngpu; g++)
      { DevTable *O = s->d+g;
        HM_CUDA(cudaSetDevice(O->dev));
        HM_CUDA(cudaStreamSynchronize(O->st));
        if (O->hi > O->lo)
          HM_CUDA(cudaMemcpy(deg+O->lo,O->deg+O->lo,(size_t) (O->hi-O->lo),cudaMemcpyDeviceToHost));
      }
  return HM_OK;
}

/* ---- one rank of a one-process-per-GPU job (DESIGN.md §4c, *Ranks*) ---------------------------------------
 * The rank streams its run-aligned share [c_rank, c_rank+1) through one device with the chunk loop of the
 * in-process shards (shard_pass1), and settles pass 2 without reading another rank's memory: the caller runs
 * the collectives between the calls (smudgeplot_b200/dist.py).                                              */
#define ROUTE_MIN_SLICE 256

struct hm_rank_scan
  { hm_scan      *s;                         /* one device (d[0]), s->nshard = world, s->rank = rank          */
    StreamRun     R;
    int           stage;                     /* 0 created, 1 pass 1 done, 2 pass 2 prepared, 3 buffers sized,
                                              * 4 listing prepared, 5 listing buffers sized                    */
    uint64_t      ns;                        /* S keys of this rank                                          */
    int           sbits, sidx64;
    int64_t       ncand, slice, rounds;
    hm_route_bufs B;
    uint64_t     *recv;                      /* keys that arrive: (world-1) * 2 * slice queries at most       */
    uint8_t      *ans_recv, *ans_sent;       /* answers to them / to this rank's queries                     */
    int64_t       n_sent, n_pend;            /* of the last round                                            */
    uint64_t      status;                    /* OR of the status words seen since pass 1                     */
    uint16_t     *pix;                       /* the listing: device pixmap, record counter, a round's records */
    unsigned long long *rec_n;
    hm_pair_rec  *rec;
    hm_pair_rec  *host;                      /* the records of the rounds so far                              */
    int64_t       host_n, host_cap;
    int64_t       list_cap;                  /* host bytes the lists may take (0: they stay on the device)   */
    int           lists_host;                /* the lists are in host memory (R.hc, R.hs): parked routed rounds */
    int           part_bits;
    int64_t       room, part, nparts;        /* pass 2's device room; S keys per partition, partitions       */
    hm_stream_lists X;                       /* (lists in host memory) one uploaded candidate slice           */
    uint64_t     *sorted;                    /* the keys received, sorted (2 words apiece at k > 32)          */
    uint32_t     *perm[2];
    uint8_t      *ans_sorted;
    void         *tmp;
    int64_t       tmp_bytes;
    uint64_t     *pkey, *plo;                /* one S partition and its bucket index                          */
    void         *pbucket;
    uint64_t     *hq;                        /* (host) the sorted keys received                               */
    SpillPart    *parts;
  };

static void rank_free_route(hm_rank_scan *r)
{ DevTable *D = r->s->d;
  cudaSetDevice(D->dev);
  dev_free(D,r->B.pend); dev_free(D,r->B.q_key); dev_free(D,r->B.q_lo); dev_free(D,r->B.q_tag);
  dev_free(D,r->B.send); dev_free(D,r->B.send_slot); dev_free(D,r->B.counts);
  dev_free(D,r->B.pend_key); dev_free(D,r->B.pend_lo); dev_free(D,r->rec);
  dev_free(D,r->recv); dev_free(D,r->ans_recv); dev_free(D,r->ans_sent);
  memset(&r->B,0,sizeof(r->B));
  r->recv = NULL; r->ans_recv = NULL; r->ans_sent = NULL; r->rec = NULL;
  if (r->R.sc) cudaStreamSynchronize(r->R.sc);           /* (lists in host memory) */
  dev_free(D,r->X.cand_key); dev_free(D,r->X.cand_meta); dev_free(D,r->X.cand_lo);
  dev_free(D,r->sorted); dev_free(D,r->perm[0]); dev_free(D,r->perm[1]); dev_free(D,r->ans_sorted); dev_free(D,r->tmp);
  dev_free(D,r->pkey); dev_free(D,r->plo); dev_free(D,r->pbucket);
  free(r->hq); free(r->parts);
  memset(&r->X,0,sizeof(r->X));
  r->sorted = NULL; r->perm[0] = r->perm[1] = NULL; r->ans_sorted = NULL; r->tmp = NULL; r->tmp_bytes = 0;
  r->pkey = r->plo = NULL; r->pbucket = NULL; r->hq = NULL; r->parts = NULL;   /* (nparts stays, for the stats) */
}

static void rank_free_listing(hm_rank_scan *r)
{ DevTable *D = r->s->d;
  cudaSetDevice(D->dev);
  dev_free(D,r->pix); dev_free(D,r->rec_n);
  free(r->host);
  r->pix = NULL; r->rec_n = NULL; r->host = NULL; r->host_n = r->host_cap = 0;
}

/* device bytes of the route buffers for slices of `slice` candidates */
static int64_t route_bytes(int64_t slice, int kmer, int world)
{ int64_t KW = kmer > 32 ? 2 : 1, q = 2*slice, o = world-1;
  return 8*slice + q*(8*KW+8+(KW == 2 ? 8 : 0)) + q*(8*KW+4) + o*q*8*KW + o*q + q + 16*HM_MAX_SHARDS + 10*256;
}

/* the routed listing's: the route buffers, the parked keys and two records per candidate of the slice */
static int64_t listing_bytes(int64_t slice, int kmer, int world)
{ int64_t KW = kmer > 32 ? 2 : 1;
  return route_bytes(slice,kmer,world) + 8*KW*slice + 2*slice*(int64_t) sizeof(hm_pair_rec) + 3*256;
}
#define LISTING_FIXED_BYTES (2ll*HM_PLOT_CELLS + 256)    /* the device pixmap and the record counter */

extern "C" void hm_rank_scan_destroy(hm_rank_scan *r)
{ if (r == NULL)
    return;
  if (r->s != NULL)
    { rank_free_route(r);
      rank_free_listing(r);
      stream_release(r->s,0,&r->R);
      hm_scan_destroy(r->s);
    }
  free(r);
}

/* a rank scan of a table of n entries streaming the host table t (the whole table, or the rank's share of it:
 * [0, t->nels) either way) through `device`; its cuts are set by the caller                                   */
static int rank_scan_open(const hm_host_table *t, int64_t n, int device, int rank, int world, const uint64_t seed[2],
                          hm_rank_scan **out)
{ if (t == NULL || out == NULL || seed == NULL || world < 1 || world > HM_MAX_GPUS || rank < 0 || rank >= world ||
      device < 0 || n < t->nels)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_create: bad arguments");
  if (t->kmer < HM_SYMM_MIN_KMER || t->kmer > HM_MAX_KMER)
    return hm_set_error(HM_EUNSUPPORTED,"the table does not fit in device memory and k = %d has no strand-symmetric "
                        "scan; the direct passes need it resident",t->kmer);
  if (t->ibyte < 1 || t->ibyte > 3 || t->ibyte > ((t->kmer+3)>>2))
    return hm_set_error(HM_EFORMAT,"table has ibyte=%d with k=%d",t->ibyte,t->kmer);
  prewarm_join();
  if (hm_device_count() <= device)
    return hm_set_error(HM_ECUDA,"CUDA device %d is not visible (this build has no CPU fallback)",device);
  hm_rank_scan *r = (hm_rank_scan *) calloc(1,sizeof(hm_rank_scan));
  hm_scan      *s = (hm_scan *) calloc(1,sizeof(hm_scan));
  if (r == NULL || s == NULL)
    { free(r); free(s); return hm_set_error(HM_ENOMEM,"out of host memory"); }
  r->s = s;
  s->kmer = t->kmer; s->ibyte = t->ibyte; s->n = n; s->ngpu = 1; s->nshard = world; s->rank = rank;
  s->bits = hm_pick_bucket_bits(s->n); s->fpos = hm_pick_filter_bits(s->n); s->idx64 = (s->n >= 0xFFFFFFF0ll);
  s->seed[0] = seed[0]; s->seed[1] = seed[1];               /* the same on every rank: the sums are added */
  s->list_knob = "the list_host_budget argument";
  s->budget = device_budget(&device,1);
  s->incore_bytes = incore_bytes(s->n,t->kmer,1,s->bits,s->idx64);
  int rc = stream_setup(s,t);
  DevTable *D = s->d;
  cudaError_t e;
  if (rc == HM_OK) rc = open_device(D,device,1);
  TRY(dev_alloc(D,&D->plot,sizeof(unsigned long long)*HM_PLOT_CELLS));
  TRY(dev_alloc(D,&D->fp_acc,4*sizeof(uint64_t)));
  D->lo = 0; D->hi = t->nels;
  if (rc != HM_OK)
    { r->s = NULL; free(r);
      hm_scan_destroy(s);
      return rc;
    }
  *out = r;
  return HM_OK;
}

extern "C" int hm_rank_scan_create(const hm_host_table *t, int device, int rank, int world, const uint64_t seed[2],
                                   hm_rank_scan **out)
{ hm_rank_scan *r = NULL;
  int rc = rank_scan_open(t,t != NULL ? t->nels : 0,device,rank,world,seed,&r);
  if (rc == HM_OK && world > 1 && (rc = stream_cuts(r->s)) != HM_OK)
    hm_rank_scan_destroy(r);
  else if (rc == HM_OK)
    *out = r;
  return rc;
}

extern "C" int hm_rank_scan_create_share(const hm_host_table *share, int64_t n_total, const int64_t *cuts,
                                         const uint64_t *first_keys, int device, int rank, int world,
                                         const uint64_t seed[2], hm_rank_scan **out)
{ int ok = share != NULL && cuts != NULL && first_keys != NULL && world >= 1 && world <= HM_MAX_GPUS && rank >= 0 &&
           rank < world && cuts[0] == 0 && cuts[world] == n_total;
  for (int q = 0; ok && q < world; q++)
    ok = cuts[q] <= cuts[q+1];
  if (!ok || cuts[rank+1]-cuts[rank] != share->nels)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_create_share: bad arguments (the share must hold entries "
                        "[cuts[rank], cuts[rank+1]) of cuts rising from 0 to n_total)");
  hm_rank_scan *r = NULL;
  int rc = rank_scan_open(share,n_total,device,rank,world,seed,&r);
  if (rc != HM_OK)
    return rc;
  if (world > 1)                              /* stream_cuts' descriptor, from the given cuts */
    { hm_symm_shards *sh = r->s->ssh;
      int live = 1;
      for (int q = 1; q < world; q++)
        if (cuts[q] < n_total) live = q+1;
      memset(sh,0,sizeof(*sh));
      sh->n_seg = live; sh->self = rank;
      for (int q = 0; q <= world; q++) sh->off[q] = cuts[q];
      for (int q = 0; q < world; q++)  sh->first_key[q] = first_keys[q];
    }
  *out = r;
  return HM_OK;
}

/* cuts: int64[world+1], c_0 = 0 ... c_world = n; first_keys (optional): uint64[world], word 0 of entry c_r */
extern "C" int hm_rank_scan_cuts(const hm_rank_scan *r, int64_t *cuts, uint64_t *first_keys)
{ if (r == NULL || cuts == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_cuts: bad arguments");
  const hm_scan *s = r->s;
  for (int q = 0; q <= s->nshard; q++)
    cuts[q] = s->nshard > 1 ? s->ssh[0].off[q] : (q == 0 ? 0 : s->n);
  if (first_keys != NULL)
    for (int q = 0; q < s->nshard; q++)
      first_keys[q] = s->nshard > 1 ? s->ssh[0].first_key[q] : 0;
  return HM_OK;
}

/* pass 1 over the rank's share; fp: host uint64[4], the fingerprint sums of the entries it scanned */
extern "C" int hm_rank_scan_pass1(hm_rank_scan *r, uint64_t *fp)
{ if (r == NULL || fp == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_pass1: bad arguments");
  hm_scan  *s = r->s;
  DevTable *D = s->d;
  rank_free_route(r);
  rank_free_listing(r);
  stream_release(s,0,&r->R);
  r->stage = 0; r->status = 0; r->nparts = 0; r->part = 0;
  D->peak = D->held; D->chunks = 0; s->stop = 0;
  memset(&s->spill,0,sizeof(s->spill));
  s->list_cap = r->list_cap; s->host_held = 0; r->lists_host = 0;
  r->R.spill = (r->list_cap > 0);
  if (r->R.spill && getenv("HETMERS_LIST_ROOM") != NULL)       /* smaller device lists than the budget allows */
    r->R.list_room = atoll(getenv("HETMERS_LIST_ROOM"));
  int rc = shard_pass1(s,0,&r->R);
  if (rc != HM_OK)
    return rc;
  uint64_t nc = 0, status = 0;
  if ((rc = hm_symm_stream_counts(r->R.work,&r->R.L,&nc,&status,&r->ns,r->R.sc)) != HM_OK)
    return rc;
  HM_CUDA(cudaMemcpy(fp,D->fp_acc,4*sizeof(uint64_t),cudaMemcpyDeviceToHost));
  r->ncand = (int64_t) nc;
  if (r->R.spilled)                              /* shard_pass1 flushed what was left */
    { r->lists_host = 1;
      r->ncand = host_list_entries(&r->R.hc); r->ns = (uint64_t) host_list_entries(&r->R.hs);
    }
  r->stage = 1;
  return HM_OK;
}

extern "C" int hm_rank_scan_set_list_host_budget(hm_rank_scan *r, int64_t bytes)
{ if (r == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_set_list_host_budget: bad arguments");
  r->list_cap = bytes > 0 ? bytes : 0;
  return HM_OK;
}

/* another rank spilled: this rank's lists (all of them on the device) go to host memory too */
extern "C" int hm_rank_scan_host_lists(hm_rank_scan *r)
{ if (r == NULL || r->stage != 1)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_host_lists: pass 1 first");
  if (r->lists_host)
    return HM_OK;
  hm_scan  *s = r->s;
  uint64_t nc = 0, status = 0, ns = 0;
  int rc;
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  if ((rc = hm_symm_stream_counts(r->R.work,&r->R.L,&nc,&status,&ns,r->R.sc)) != HM_OK ||
      (rc = stream_flush(s,s->d,&r->R,nc,ns)) != HM_OK)
    return rc;
  r->lists_host = 1;
  r->ncand = host_list_entries(&r->R.hc); r->ns = (uint64_t) host_list_entries(&r->R.hs);
  return HM_OK;
}

/* lists in host memory: the chunk buffers and stub index freed (no S index: S is not resident), the room that
 * leaves (HETMERS_SPILL_ROOM: less) and the largest slice the plan gives in it                              */
static int rank_host_prepare(hm_rank_scan *r, int listing, int64_t fixed, int64_t *max_slice)
{ hm_scan  *s = r->s;
  DevTable *D = s->d;
  hm_spill_layout P;
  HM_CUDA(cudaSetDevice(D->dev));
  stream_free_chunks(D,&r->R);
  dev_free(D,r->R.d_index); r->R.d_index = NULL;
  HM_CUDA(cudaStreamSynchronize(r->R.sc));
  int64_t room = s->budget - D->held - fixed;
  const char *e = getenv("HETMERS_SPILL_ROOM");              /* smaller slices and partitions than the room allows */
  if (e != NULL && atoll(e) > 0 && atoll(e) < room)
    room = atoll(e);
  int rc = hm_rank_spill_plan(r->ncand,(int64_t) r->ns,s->kmer,s->nshard,listing,room,&P);
  if (rc != HM_OK)
    return rc;
  r->room = room;
  *max_slice = P.slice;
  return HM_OK;
}

/* Bloom segments of the work area: segment q (seg_bytes each, world of them) is filled by rank q's pass 1 */
extern "C" int hm_rank_scan_bloom(const hm_rank_scan *r, void **d_segments, int64_t *seg_bytes)
{ if (r == NULL || r->stage < 1 || d_segments == NULL || seg_bytes == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_bloom: no pass 1 has run");
  *d_segments = (uint8_t *) r->R.work + r->R.L.off_bloom;
  *seg_bytes = 4*r->R.L.seg_words;
  return HM_OK;
}

/* the most candidates per slice whose buffers (bytes(slice, kmer, world)) fit in room */
static int64_t largest_slice(int64_t room, int kmer, int world, int64_t (*bytes)(int64_t, int, int))
{ int64_t lo = 0, hi = (int64_t) 1 << 31;
  while (lo < hi)
    { int64_t mid = lo + (hi-lo+1)/2;
      if (bytes(mid,kmer,world) <= room) lo = mid;
      else                               hi = mid-1;
    }
  return lo;
}

/* symmetric = the job-wide fingerprint verdict.  Frees the chunk buffers, indexes the S list and reports the
 * rank's candidates and the largest slice its budget leaves room for (HM_ENOMEM below ROUTE_MIN_SLICE).     */
extern "C" int hm_rank_scan_prepare(hm_rank_scan *r, int symmetric, int64_t *n_cand, int64_t *max_slice)
{ if (r == NULL || r->stage != 1 || n_cand == NULL || max_slice == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_prepare: pass 1 first");
  hm_scan *s = r->s;
  s->symmetric = symmetric != 0;
  if (!symmetric)
    return refuse_asymmetric(s);
  int rc;
  if (r->lists_host)
    { if ((rc = rank_host_prepare(r,0,0,max_slice)) != HM_OK)
        return rc;
      *n_cand = r->ncand;
      r->stage = 2;
      return HM_OK;
    }
  r->sidx64 = ((int64_t) r->ns >= 0xFFFFFFF0ll);
  if ((rc = stream_s_index(s,0,&r->R,r->ns,r->sidx64,1,&r->sbits)) != HM_OK)
    return rc;
  HM_CUDA(cudaStreamSynchronize(r->R.sc));
  int64_t room = s->budget - s->d[0].held, lo = largest_slice(room,s->kmer,s->nshard,route_bytes);
  if (lo < ROUTE_MIN_SLICE)
    return hm_set_error(HM_ENOMEM,"a device budget of %lld bytes leaves %lld bytes beside the resident lists of this rank "
                        "(%lld held), and pass 2's exchange buffers for a slice of %d candidates need %lld",
                        (long long) s->budget,(long long) (room > 0 ? room : 0),(long long) s->d[0].held,ROUTE_MIN_SLICE,
                        (long long) route_bytes(ROUTE_MIN_SLICE,s->kmer,s->nshard));
  *n_cand = r->ncand;
  *max_slice = lo;
  r->stage = 2;
  return HM_OK;
}

/* slice: the same on every rank (at most every rank's max_slice).  Allocates the route buffers; *rounds = the
 * slices this rank's candidates take.  The device buffers the caller's collectives read and write:
 * send (uint64, KW words per query, grouped by owner), recv (the same for what arrives), ans_recv (a byte per
 * key that arrived) and ans_sent (a byte per query sent, in send order).                                    */
/* the route buffers of slices of `slice` candidates (listing: with the parked keys and the records) */
static int rank_alloc_host(hm_rank_scan *r, int64_t slice, int listing, int64_t *rounds, void **d_send, void **d_recv,
                           void **d_ans_recv, void **d_ans_sent);

static int rank_alloc_route(hm_rank_scan *r, int64_t slice, int listing, int64_t *rounds, void **d_send, void **d_recv,
                            void **d_ans_recv, void **d_ans_sent)
{ if (r->lists_host)
    return rank_alloc_host(r,slice,listing,rounds,d_send,d_recv,d_ans_recv,d_ans_sent);
  hm_scan  *s = r->s;
  DevTable *D = s->d;
  int64_t   KW = s->kmer > 32 ? 2 : 1, q = 2*slice, o = s->nshard-1;
  int64_t   need = listing ? listing_bytes(slice,s->kmer,s->nshard) : route_bytes(slice,s->kmer,s->nshard);
  int       rc = HM_OK;
  cudaError_t e;
  if (D->held + need > s->budget)
    return hm_set_error(HM_ENOMEM,"%s for slices of %lld candidates need %lld bytes and the device budget of %lld bytes "
                        "has room for %lld",listing ? "the pair listing's buffers" : "pass 2's exchange buffers",
                        (long long) slice,(long long) need,(long long) s->budget,(long long) (s->budget-D->held));
  rank_free_route(r);
  TRY(cudaSetDevice(D->dev));
  TRY(dev_alloc(D,&r->B.pend,8*slice));
  TRY(dev_alloc(D,&r->B.q_key,8*q));
  if (KW == 2) TRY(dev_alloc(D,&r->B.q_lo,8*q));
  TRY(dev_alloc(D,&r->B.q_tag,8*q));
  TRY(dev_alloc(D,&r->B.send,8*KW*q));
  TRY(dev_alloc(D,&r->B.send_slot,4*q));
  TRY(dev_alloc(D,&r->B.counts,16*HM_MAX_SHARDS));
  TRY(dev_alloc(D,&r->recv,8*KW*(o*q > 0 ? o*q : 1)));
  TRY(dev_alloc(D,&r->ans_recv,o*q > 0 ? o*q : 1));
  TRY(dev_alloc(D,&r->ans_sent,q));
  if (listing)
    { TRY(dev_alloc(D,&r->B.pend_key,8*slice));
      if (KW == 2) TRY(dev_alloc(D,&r->B.pend_lo,8*slice));
      TRY(dev_alloc(D,&r->rec,2*slice*(int64_t) sizeof(hm_pair_rec)));
    }
  if (rc != HM_OK)
    { rank_free_route(r); return rc; }
  r->B.pend_cap = slice; r->B.q_cap = q;
  r->slice = slice;
  r->rounds = (r->ncand + slice-1)/slice;
  *rounds = r->rounds;
  if (d_send)     *d_send = r->B.send;
  if (d_recv)     *d_recv = r->recv;
  if (d_ans_recv) *d_ans_recv = r->ans_recv;
  if (d_ans_sent) *d_ans_sent = r->ans_sent;
  return HM_OK;
}

/* ---- a rank's lists in host memory (DESIGN.md §4c, *Lists in host memory*): the parked routed rounds ---- */

/* the slice of `slice` candidates, its queries and their exchange, what world ranks send for them, and one S
 * partition in the room prepare found (hm_rank_spill_plan); *rounds = the slices this rank's candidates take.
 * recv holds world x 2 x slice keys: every rank's queries, this rank's own among them.                       */
static int rank_alloc_host(hm_rank_scan *r, int64_t slice, int listing, int64_t *rounds, void **d_send, void **d_recv,
                           void **d_ans_recv, void **d_ans_sent)
{ hm_scan  *s = r->s;
  DevTable *D = s->d;
  const int KW = s->kmer > 32 ? 2 : 1, W = s->nshard;
  int64_t   q = 2*slice, qr = (int64_t) W*q, room = r->room;
  int       rc = HM_OK;
  cudaError_t e;
  rank_free_route(r);
  int64_t need = rank_spill_slice_bytes(slice,KW,W,listing);
  int64_t np = (int64_t) r->ns > 1 ? (int64_t) r->ns : 1;
  if (np > HM_SPILL_MAX_PART) np = HM_SPILL_MAX_PART;
  int64_t part = spill_largest(np,room-need,KW,spill_part_bytes);
  const char *env = getenv("HETMERS_SPILL_PART");                   /* smaller partitions */
  if (env != NULL && atoll(env) > 0 && atoll(env) < part)
    part = atoll(env);
  if (part < 1 || (part < (np < HM_SPILL_MIN ? np : HM_SPILL_MIN) && (env == NULL || atoll(env) <= 0)))
    return hm_set_error(HM_ENOMEM,"pass 2 of a rank's lists in host memory: slices of %lld candidates need %lld device "
                        "bytes of the %lld in the room, which leaves too little for S partitions",(long long) slice,
                        (long long) need,(long long) room);
  TRY(cudaSetDevice(D->dev));
  TRY(dev_alloc(D,&r->X.cand_key,8*slice));
  TRY(dev_alloc(D,&r->X.cand_meta,8*slice));
  if (KW == 2) TRY(dev_alloc(D,&r->X.cand_lo,8*slice));
  TRY(dev_alloc(D,&r->B.pend,8*slice));
  TRY(dev_alloc(D,&r->B.q_key,8*q));
  if (KW == 2) TRY(dev_alloc(D,&r->B.q_lo,8*q));
  TRY(dev_alloc(D,&r->B.q_tag,8*q));
  TRY(dev_alloc(D,&r->B.send,8*KW*q));
  TRY(dev_alloc(D,&r->B.send_slot,4*q));
  TRY(dev_alloc(D,&r->B.counts,16*HM_MAX_SHARDS));
  TRY(dev_alloc(D,&r->ans_sent,q));
  if (listing)
    { TRY(dev_alloc(D,&r->B.pend_key,8*slice));
      if (KW == 2) TRY(dev_alloc(D,&r->B.pend_lo,8*slice));
      TRY(dev_alloc(D,&r->rec,2*slice*(int64_t) sizeof(hm_pair_rec)));
    }
  r->tmp_bytes = hm_sort_perm_bytes(qr);
  TRY(dev_alloc(D,&r->recv,8*KW*qr));
  TRY(dev_alloc(D,&r->sorted,8*KW*qr));
  TRY(dev_alloc(D,&r->perm[0],4*qr));
  TRY(dev_alloc(D,&r->perm[1],4*qr));
  TRY(dev_alloc(D,&r->ans_recv,qr));
  TRY(dev_alloc(D,&r->ans_sorted,qr));
  TRY(dev_alloc(D,&r->tmp,r->tmp_bytes));
  TRY(dev_alloc(D,&r->pkey,8*part));
  if (KW == 2) TRY(dev_alloc(D,&r->plo,8*part));
  r->part_bits = hm_pick_bucket_bits(part);
  TRY(dev_alloc(D,&r->pbucket,4*((1ll << r->part_bits)+1)));
  if (rc == HM_OK && D->held > s->budget)
    rc = hm_set_error(HM_ENOMEM,"pass 2 of a rank's lists in host memory holds %lld device bytes, more than the budget "
                      "of %lld (the plan counted %lld)",(long long) D->held,(long long) s->budget,
                      (long long) (need + spill_part_bytes(part,KW)));
  int64_t nparts = spill_part_count(&r->R.hs,part);
  if (rc == HM_OK && ((r->hq = (uint64_t *) malloc(8*(size_t) KW*(size_t) qr)) == NULL ||
                      (r->parts = (SpillPart *) malloc(sizeof(SpillPart)*(size_t) (nparts > 0 ? nparts : 1))) == NULL))
    rc = hm_set_error(HM_ENOMEM,"out of host memory");
  if (rc != HM_OK)
    { rank_free_route(r); return rc; }
  r->nparts = 0;
  spill_cut_parts(&r->R.hs,part,KW,r->parts,&r->nparts);
  r->X.cand_cap = slice;
  r->B.pend_cap = slice; r->B.q_cap = q;
  r->slice = slice; r->part = part;
  r->rounds = (r->ncand + slice-1)/slice;
  r->R.rounds = r->R.h2d_bytes = r->R.first_key_queries = 0;
  r->R.ms_pass2 = 0;
  *rounds = r->rounds;
  if (d_send)     *d_send = r->B.send;
  if (d_recv)     *d_recv = r->recv;
  if (d_ans_recv) *d_ans_recv = r->ans_recv;
  if (d_ans_sent) *d_ans_sent = r->ans_sent;
  return HM_OK;
}

/* the candidates [c0, c1) of the host list uploaded into the slice buffers (they may span blocks) */
static int rank_host_upload(hm_rank_scan *r, int64_t c0, int64_t c1)
{ const int KW = r->s->kmer > 32 ? 2 : 1;
  int64_t   at = 0, base = 0;
  int       rc = HM_OK;
  for (int b = 0; b < r->R.hc.nb && at < c1-c0 && rc == HM_OK; b++)
    { const HostBlock *hb = r->R.hc.b+b;
      int64_t lo = c0+at-base;                                   /* where the slice goes on in this block */
      if (lo < hb->n)
        { int64_t m = hb->n-lo < c1-c0-at ? hb->n-lo : c1-c0-at;
          rc = stage_copy(&r->R,r->X.cand_key+at,hb->w+lo,8*m,0);
          if (rc == HM_OK) rc = stage_copy(&r->R,r->X.cand_meta+at,hb->w+hb->n+lo,8*m,0);
          if (rc == HM_OK && KW == 2) rc = stage_copy(&r->R,r->X.cand_lo+at,hb->w+2*hb->n+lo,8*m,0);
          at += m;
        }
      base += hb->n;
    }
  r->R.h2d_bytes += (c1-c0)*(8*KW+8);
  return rc;
}

/* a round of the parked routed pass: the slice [c0, c1) uploaded and swept (listing: extract_kernel), every Bloom
 * hit parked with a query per key that hit, tagged with the key's owner; the queries grouped by owner         */
static int rank_host_route(hm_rank_scan *r, int64_t c0, int64_t c1, int listing, int64_t *counts)
{ hm_scan  *s = r->s;
  DevTable *D = s->d;
  uint64_t  status = 0;
  double    t0 = now_ms();
  int       rc = rank_host_upload(r,c0,c1);
  const hm_symm_shards *sh = s->nshard > 1 ? s->ssh : NULL;
  if (rc == HM_OK)
    rc = listing
      ? hm_symm_park_extract(s->kmer,c1-c0,r->R.work,&r->R.L,&r->X,sh,&r->B,r->pix,r->rec,2*r->slice,r->rec_n,r->R.sc)
      : hm_symm_park_resolve(s->kmer,c1-c0,1,r->R.work,&r->R.L,&r->X,sh,&r->B,D->plot,r->R.sc);
  __sync_fetch_and_add(&s->launches,(int64_t) (c1 > c0));
  if (rc == HM_OK)
    rc = hm_symm_route_group(s->kmer,s->nshard,r->R.work,&r->R.L,&r->B,counts,&r->n_sent,&r->n_pend,&status,r->R.sc);
  r->status |= status;
  r->R.rounds += 1;
  r->R.ms_pass2 += now_ms()-t0;
  return rc;
}

/* the n keys received (every rank's queries to this one, its own among them): sorted by key, answered against the
 * rank's S list a partition at a time -- only the partitions some key falls in are uploaded and indexed -- and
 * the answers put back in receive order into ans_recv (synchronises)                                        */
static int rank_host_answer(hm_rank_scan *r, int64_t n)
{ hm_scan   *s = r->s;
  const int  KW = s->kmer > 32 ? 2 : 1;
  double     t0 = now_ms();
  uint32_t  *perm = NULL;
  int        rc = hm_symm_recv_sort(s->kmer,r->recv,n,r->sorted,r->perm[0],r->perm[1],r->tmp,r->tmp_bytes,&perm,r->R.sc);
  if (rc != HM_OK)
    return rc;
  if (n > 0)
    { HM_CUDA(cudaMemcpyAsync(r->hq,r->sorted,8*(size_t) KW*(size_t) n,cudaMemcpyDeviceToHost,r->R.sc));
      HM_CUDA(cudaMemsetAsync(r->ans_sorted,0,(size_t) n,r->R.sc));
      HM_CUDA(cudaStreamSynchronize(r->R.sc));
    }
  rc = spill_answer_parts(s,&r->R,r->parts,r->nparts,r->part_bits,r->hq,r->sorted,n,r->pkey,r->plo,r->pbucket,
                          r->ans_sorted);
  if (rc == HM_OK)
    rc = hm_symm_recv_unsort(r->ans_sorted,perm,n,r->ans_recv,r->R.sc);
  r->R.ms_pass2 += now_ms()-t0;
  return rc;
}

extern "C" int hm_rank_scan_spill_stats(const hm_rank_scan *r, hm_spill_stats *out)
{ if (r == NULL || out == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_spill_stats: bad arguments");
  const StreamRun *R = &r->R;
  memset(out,0,sizeof(*out));
  out->spilled = r->lists_host;
  out->flushes = R->flushes; out->d2h_bytes = R->d2h_bytes;
  out->host_peak_bytes = r->s->spill.host_peak_bytes;
  out->partitions = r->nparts; out->rounds = R->rounds; out->h2d_bytes = R->h2d_bytes;
  out->slice = r->lists_host ? r->slice : 0; out->part = r->part;
  out->first_key_queries = R->first_key_queries;
  out->ms_pass1 = R->ms_loop; out->ms_flush = R->ms_flush; out->ms_pass2 = R->ms_pass2;
  return HM_OK;
}

extern "C" int hm_rank_scan_slices(hm_rank_scan *r, int64_t slice, int64_t *rounds, void **d_send, void **d_recv,
                                   void **d_ans_recv, void **d_ans_sent)
{ if (r == NULL || r->stage != 2 || slice < 1 || rounds == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_slices: bad arguments");
  int rc = rank_alloc_route(r,slice,0,rounds,d_send,d_recv,d_ans_recv,d_ans_sent);
  if (rc == HM_OK)
    r->stage = 3;
  return rc;
}

/* the candidates [c0, c1) of round `round` (an empty slice once they are done) */
static void rank_round(const hm_rank_scan *r, int64_t round, int64_t *c0, int64_t *c1)
{ *c0 = round*r->slice < r->ncand ? round*r->slice : r->ncand;
  *c1 = *c0 + r->slice < r->ncand ? *c0 + r->slice : r->ncand;
}

/* round `round`: resolve the slice [round*slice, ...) of this rank's candidates (none once they are done) and
 * group its queries by owner; counts: int64[world], the queries for each rank, in the order of send       */
extern "C" int hm_rank_scan_route(hm_rank_scan *r, int64_t round, int64_t *counts)
{ if (r == NULL || r->stage != 3 || counts == NULL || round < 0)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_route: bad arguments");
  hm_scan  *s = r->s;
  DevTable *D = s->d;
  int64_t   c0, c1;
  int       KW = s->kmer > 32 ? 2 : 1, rc;
  uint64_t  status = 0;
  rank_round(r,round,&c0,&c1);
  HM_CUDA(cudaSetDevice(D->dev));
  if (round == 0)
    HM_CUDA(cudaEventRecord(D->ev[2],r->R.sc));
  if (r->lists_host)
    return rank_host_route(r,c0,c1,0,counts);
  if ((rc = hm_symm_route_resolve(r->R.R.s_key,KW == 2 ? r->R.R.s_lo : NULL,(int64_t) r->ns,r->R.s_bucket,r->sbits,
                                  r->sidx64,s->kmer,c0,c1,r->R.work,&r->R.L,&r->R.R,s->nshard > 1 ? s->ssh : NULL,&r->B,
                                  D->plot,r->R.sc)) != HM_OK)
    return rc;
  __sync_fetch_and_add(&s->launches,(int64_t) (c1 > c0));
  if ((rc = hm_symm_route_group(s->kmer,s->nshard,r->R.work,&r->R.L,&r->B,counts,&r->n_sent,&r->n_pend,&status,
                                r->R.sc)) != HM_OK)
    return rc;
  r->status |= status;
  return HM_OK;
}

/* the n keys that arrived in recv: one byte each into ans_recv (synchronises) */
extern "C" int hm_rank_scan_answer(hm_rank_scan *r, int64_t n)
{ hm_scan *s = r ? r->s : NULL;
  if (r == NULL || (r->stage != 3 && r->stage != 5) || n < 0 ||
      n > (s->nshard-1 + (r != NULL && r->lists_host))*2*r->slice)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_answer: bad arguments");
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  if (r->lists_host)
    return rank_host_answer(r,n);
  return hm_symm_route_answer(r->R.R.s_key,s->kmer > 32 ? r->R.R.s_lo : NULL,r->R.s_bucket,r->sbits,r->sidx64,s->kmer,
                              r->recv,n,r->ans_recv,r->R.sc);
}

/* ans_sent holds the answers to the round's queries: count the parked candidates none of whose keys was found */
extern "C" int hm_rank_scan_settle(hm_rank_scan *r)
{ if (r == NULL || r->stage != 3)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_settle: bad arguments");
  hm_scan *s = r->s;
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  double t0 = now_ms();
  int rc = hm_symm_route_settle(s->kmer,&r->B,r->ans_sent,r->n_sent,r->n_pend,s->d[0].plot,r->R.sc);
  __sync_fetch_and_add(&s->launches,2);
  if (r->lists_host) r->R.ms_pass2 += now_ms()-t0;
  return rc;
}

/* after the last round: this rank's partial plot (device int64[HM_PLOT_CELLS]) and the OR of its status words */
extern "C" int hm_rank_scan_result(hm_rank_scan *r, void **d_plot, uint64_t *status)
{ if (r == NULL || r->stage != 3 || d_plot == NULL || status == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_result: bad arguments");
  hm_scan *s = r->s;
  uint64_t nc = 0, st = 0, ns = 0;
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  HM_CUDA(cudaEventRecord(s->d[0].ev[3],r->R.sc));
  int rc = hm_symm_stream_counts(r->R.work,&r->R.L,&nc,&st,&ns,r->R.sc);     /* (synchronises) */
  if (rc != HM_OK)
    return rc;
  *d_plot = s->d[0].plot;
  *status = r->status | st;
  return HM_OK;
}

/* the most device memory the rank held since its last pass 1 began, and that pass's chunks; *budget: the budget */
extern "C" int hm_rank_scan_residency(const hm_rank_scan *r, int64_t *device_bytes, int64_t *chunks, int64_t *budget)
{ if (r == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_residency: bad arguments");
  if (device_bytes) *device_bytes = r->s->d[0].peak;
  if (chunks)       *chunks = r->s->d[0].chunks;
  if (budget)       *budget = r->s->budget;
  return HM_OK;
}

/* ---- the rank's pair listing (extract_kmer_pairs, DESIGN.md §4c, *Ranks*): the rounds of routed pass 2 over the
 * candidates pass 1 left resident, each listing its isolated candidates instead of counting them               */

/* stage >= 2: the candidates, the S index and the gathered Bloom filter of a pass 1 are resident.  Frees the
 * route buffers, uploads the pixmap and reports the largest slice the budget leaves room for (HM_ENOMEM below
 * ROUTE_MIN_SLICE, before any launch)                                                                        */
extern "C" int hm_rank_scan_extract_prepare(hm_rank_scan *r, const uint16_t *pixmap, int64_t *n_cand, int64_t *max_slice)
{ if (r == NULL || r->stage < 2 || pixmap == NULL || n_cand == NULL || max_slice == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_extract_prepare: needs a prepared pass 1");
  hm_scan  *s = r->s;
  DevTable *D = s->d;
  int       rc = HM_OK;
  cudaError_t e;
  rank_free_route(r);
  rank_free_listing(r);
  int64_t room = s->budget - D->held - LISTING_FIXED_BYTES, lo = 0;
  if (r->lists_host)
    { if ((rc = rank_host_prepare(r,1,LISTING_FIXED_BYTES,&lo)) != HM_OK)
        return rc;
    }
  else if ((lo = largest_slice(room,s->kmer,s->nshard,listing_bytes)) < ROUTE_MIN_SLICE)
    return hm_set_error(HM_ENOMEM,"a device budget of %lld bytes leaves %lld bytes beside the resident lists of this rank "
                        "(%lld held) and the pixmap (%lld), and listing k-mer pairs in slices of %d candidates needs %lld",
                        (long long) s->budget,(long long) (room > 0 ? room : 0),(long long) D->held,
                        (long long) LISTING_FIXED_BYTES,ROUTE_MIN_SLICE,
                        (long long) listing_bytes(ROUTE_MIN_SLICE,s->kmer,s->nshard));
  TRY(cudaSetDevice(D->dev));
  TRY(dev_alloc(D,&r->pix,sizeof(uint16_t)*HM_PLOT_CELLS));
  TRY(dev_alloc(D,&r->rec_n,256));
  TRY(cudaMemcpy(r->pix,pixmap,sizeof(uint16_t)*HM_PLOT_CELLS,cudaMemcpyHostToDevice));
  if (rc != HM_OK)
    { rank_free_listing(r); return rc; }
  *n_cand = r->ncand;
  *max_slice = lo;
  r->stage = 4;
  return HM_OK;
}

/* hm_rank_scan_slices for the listing (stage 4): also the parked keys and a round's records */
extern "C" int hm_rank_scan_extract_slices(hm_rank_scan *r, int64_t slice, int64_t *rounds, void **d_send,
                                           void **d_recv, void **d_ans_recv, void **d_ans_sent)
{ if (r == NULL || r->stage != 4 || slice < 1 || rounds == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_extract_slices: bad arguments");
  int rc = rank_alloc_route(r,slice,1,rounds,d_send,d_recv,d_ans_recv,d_ans_sent);
  if (rc == HM_OK)
    r->stage = 5;
  return rc;
}

/* hm_rank_scan_route for the listing: extract_kernel<..., LK_ROUTED> over the round's slice, its queries grouped
 * by owner */
extern "C" int hm_rank_scan_extract_route(hm_rank_scan *r, int64_t round, int64_t *counts)
{ if (r == NULL || r->stage != 5 || counts == NULL || round < 0)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_extract_route: bad arguments");
  hm_scan  *s = r->s;
  DevTable *D = s->d;
  int64_t   c0, c1;
  int       KW = s->kmer > 32 ? 2 : 1, rc;
  uint64_t  status = 0;
  rank_round(r,round,&c0,&c1);
  HM_CUDA(cudaSetDevice(D->dev));
  if (r->lists_host)
    return rank_host_route(r,c0,c1,1,counts);
  if ((rc = hm_symm_route_extract(r->R.R.s_key,KW == 2 ? r->R.R.s_lo : NULL,(int64_t) r->ns,r->R.s_bucket,r->sbits,
                                  r->sidx64,s->kmer,c0,c1,r->R.work,&r->R.L,&r->R.R,s->nshard > 1 ? s->ssh : NULL,&r->B,
                                  r->pix,r->rec,2*r->slice,r->rec_n,r->R.sc)) != HM_OK)
    return rc;
  __sync_fetch_and_add(&s->launches,(int64_t) (c1 > c0));
  if ((rc = hm_symm_route_group(s->kmer,s->nshard,r->R.work,&r->R.L,&r->B,counts,&r->n_sent,&r->n_pend,&status,
                                r->R.sc)) != HM_OK)
    return rc;
  r->status |= status;
  return HM_OK;
}

/* ans_sent holds the answers to the round's queries: list the parked candidates none of whose keys was found,
 * then append the round's records to the host list (synchronises)                                           */
extern "C" int hm_rank_scan_extract_settle(hm_rank_scan *r)
{ if (r == NULL || r->stage != 5)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_extract_settle: bad arguments");
  hm_scan *s = r->s;
  unsigned long long c = 0;
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  double t0 = now_ms();
  int rc = hm_symm_route_list(s->kmer,&r->B,r->ans_sent,r->n_sent,r->n_pend,r->pix,r->rec,2*r->slice,r->rec_n,r->R.sc);
  __sync_fetch_and_add(&s->launches,2);
  if (r->lists_host) r->R.ms_pass2 += now_ms()-t0;
  if (rc != HM_OK)
    return rc;
  HM_CUDA(cudaMemcpy(&c,r->rec_n,sizeof(c),cudaMemcpyDeviceToHost));
  if ((int64_t) c > 2*r->slice)
    return hm_set_error(HM_ECUDA,"the routed listing gave %llu records for a slice of %lld candidates",c,
                        (long long) r->slice);
  return append_records(&r->host,&r->host_n,&r->host_cap,r->rec,(int64_t) c);
}

/* after the last round: this rank's records (*records malloc'ed, the caller frees; sorted as hm_scan_extract sorts)
 * and the OR of its status words (non-zero: do not use them).  The listing's buffers are freed.             */
static int rank_extract_take(hm_rank_scan *r, hm_pair_rec **records, int64_t *n, uint64_t *status, int sorted);

extern "C" int hm_rank_scan_extract_result(hm_rank_scan *r, hm_pair_rec **records, int64_t *n, uint64_t *status)
{ if (r == NULL || r->stage != 5 || records == NULL || n == NULL || status == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_extract_result: bad arguments");
  return rank_extract_take(r,records,n,status,1);
}

/* hm_rank_scan_extract_result's records in the order they were listed (write_pairs sorts them on the device) */
extern "C" int hm_rank_scan_extract_records(hm_rank_scan *r, hm_pair_rec **records, int64_t *n, uint64_t *status)
{ if (r == NULL || r->stage != 5 || records == NULL || n == NULL || status == NULL)
    return hm_set_error(HM_EINVAL,"hm_rank_scan_extract_records: bad arguments");
  return rank_extract_take(r,records,n,status,0);
}

static int rank_extract_take(hm_rank_scan *r, hm_pair_rec **records, int64_t *n, uint64_t *status, int sorted)
{
  hm_scan *s = r->s;
  uint64_t nc = 0, st = 0, ns = 0;
  HM_CUDA(cudaSetDevice(s->d[0].dev));
  int rc = hm_symm_stream_counts(r->R.work,&r->R.L,&nc,&st,&ns,r->R.sc);     /* (synchronises) */
  if (rc != HM_OK)
    return rc;
  if (r->host == NULL && (r->host = (hm_pair_rec *) malloc(sizeof(hm_pair_rec))) == NULL)
    return hm_set_error(HM_ENOMEM,"out of host memory");
  if (sorted)
    sort_records(r->host,r->host_n);
  *records = r->host; *n = r->host_n;
  *status = r->status | st;
  r->host = NULL;
  rank_free_route(r);
  rank_free_listing(r);
  r->stage = 2;                                  /* (pass 1 stays resident: another listing may follow) */
  return HM_OK;
}

extern "C" int hm_sort_pair_records(hm_pair_rec *records, int64_t n)
{ if (n < 0 || (n > 0 && records == NULL))
    return hm_set_error(HM_EINVAL,"hm_sort_pair_records: bad arguments");
  sort_records(records,n);
  return HM_OK;
}

/*******************************************************************************************
 * hm_peer.cu -- the two exchange steps of the multi-GPU path when all GPUs are driven from
 * ONE process (the `hetmers` executable): hand-written peer-memory kernels over NVLink /
 * NVSwitch instead of a library collective.
 *
 *   peer_sum_deg_kernel   all-reduce(sum) of the per-GPU partial incidence arrays between
 *                         pass 1 and pass 2.  GPU g owns word slice g: it LOADS that slice from
 *                         every peer's array (peer reads), adds the byte-packed words, and
 *                         STORES the total back into every peer's array (peer writes) -- a fused
 *                         reduce-scatter + all-gather, one kernel per GPU, no staging copies.
 *   peer_sum_plot_kernel  final reduction of the 1001x501 plot onto GPU 0; the reference does
 *                         this serially over its threads (PloidyPlot.c:1569-1575).
 *
 * Byte-packed adds cannot carry between bytes: a k-mer has at most 3k <= 192 < 256 neighbours (k <= 64;
 * static_assert next to book_pair in hm_kernels.cu).
 * (The one-process-per-GPU variant uses NCCL through torch.distributed: smudgeplot_b200/dist.py.)
 *******************************************************************************************/
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <pthread.h>

#include "hetmers_b200.h"
#include "hm_internal.h"

#define PEER_MAX 16

typedef struct { uint32_t *p[PEER_MAX]; } DegPtrs;
typedef struct { unsigned long long *p[PEER_MAX]; } PlotPtrs;

typedef struct { const int *dev; int n, a, rc; char msg[256]; } PeerJob;

static int peer_enable_one(const int *dev, int n, int a)
{ int da = dev ? dev[a] : a;
  HM_CUDA(cudaSetDevice(da));
  for (int b = 0; b < n; b++)
    { int db = dev ? dev[b] : b, can = 0;
      if (da == db) continue;
      HM_CUDA(cudaDeviceCanAccessPeer(&can,da,db));
      if (!can)
        return hm_set_error(HM_ECUDA,"GPU %d cannot access GPU %d's memory (no NVLink/P2P)",da,db);
      cudaError_t e = cudaDeviceEnablePeerAccess(db,0);
      if (e == cudaErrorPeerAccessAlreadyEnabled)
        cudaGetLastError();
      else if (e != cudaSuccess)
        return hm_cuda_fail(e,"cudaDeviceEnablePeerAccess");
    }
  return HM_OK;
}

static void *peer_worker(void *arg)
{ PeerJob *J = (PeerJob *) arg;
  J->rc = peer_enable_one(J->dev,J->n,J->a);
  if (J->rc != HM_OK)
    { strncpy(J->msg,hm_last_error(),sizeof(J->msg)-1); J->msg[sizeof(J->msg)-1] = 0; }
  return NULL;
}

/* every GPU maps every other GPU's memory: n*(n-1) driver calls, one host thread per GPU */
int hm_peer_enable(const int *dev, int n)
{ PeerJob   job[PEER_MAX];
  pthread_t th[PEER_MAX];
  int       made[PEER_MAX], rc = HM_OK;
  if (n > PEER_MAX)
    return hm_set_error(HM_EINVAL,"at most %d GPUs",PEER_MAX);
  for (int a = 0; a < n; a++)
    { job[a].dev = dev; job[a].n = n; job[a].a = a; job[a].rc = HM_OK; job[a].msg[0] = 0;
      made[a] = (a+1 < n) && (pthread_create(th+a,NULL,peer_worker,job+a) == 0);
      if (!made[a])
        peer_worker(job+a);
    }
  for (int a = 0; a < n; a++)
    { if (made[a]) pthread_join(th[a],NULL);
      if (job[a].rc != HM_OK && rc == HM_OK)
        rc = hm_set_error(job[a].rc,"%s",job[a].msg);
    }
  return rc;
}

/* ---- CUDA IPC plumbing for the one-process-per-GPU job (layer A callers) ---- */

extern "C" int hm_dev_alloc(int64_t bytes, void **dptr)
{ if (bytes <= 0 || dptr == NULL)
    return hm_set_error(HM_EINVAL,"hm_dev_alloc: bad arguments");
  HM_CUDA(cudaMalloc(dptr,(size_t) bytes));
  HM_CUDA(cudaMemset(*dptr,0,(size_t) bytes));
  return HM_OK;
}

extern "C" int hm_dev_free(void *dptr)
{ if (dptr != NULL)
    HM_CUDA(cudaFree(dptr));
  return HM_OK;
}

extern "C" int hm_ipc_export(void *dptr, unsigned char handle[64])
{ cudaIpcMemHandle_t h;
  static_assert(sizeof(cudaIpcMemHandle_t) == 64,"IPC handle size");
  HM_CUDA(cudaIpcGetMemHandle(&h,dptr));
  memcpy(handle,&h,64);
  return HM_OK;
}

extern "C" int hm_ipc_open(const unsigned char handle[64], void **dptr)
{ cudaIpcMemHandle_t h;
  memcpy(&h,handle,64);
  HM_CUDA(cudaIpcOpenMemHandle(dptr,h,cudaIpcMemLazyEnablePeerAccess));
  return HM_OK;
}

extern "C" int hm_ipc_close(void *dptr)
{ if (dptr != NULL)
    HM_CUDA(cudaIpcCloseMemHandle(dptr));
  return HM_OK;
}

extern "C" int hm_p2p_native_atomics(int dev_a, int dev_b)
{ int ab = 0, ba = 0, can1 = 0, can2 = 0;
  if (dev_a == dev_b)
    return 1;
  if (cudaDeviceCanAccessPeer(&can1,dev_a,dev_b) != cudaSuccess ||
      cudaDeviceCanAccessPeer(&can2,dev_b,dev_a) != cudaSuccess || !can1 || !can2)
    { cudaGetLastError(); return 0; }
  if (cudaDeviceGetP2PAttribute(&ab,cudaDevP2PAttrNativeAtomicSupported,dev_a,dev_b) != cudaSuccess ||
      cudaDeviceGetP2PAttribute(&ba,cudaDevP2PAttrNativeAtomicSupported,dev_b,dev_a) != cudaSuccess)
    { cudaGetLastError(); return 0; }
  return (ab && ba);
}

__global__ void __launch_bounds__(256)
peer_sum_deg_kernel(DegPtrs P, int npeer, int64_t w0, int64_t w1)
{ int64_t stride = (int64_t) gridDim.x * blockDim.x * 4;
  for (int64_t w = w0 + ((int64_t) blockIdx.x * blockDim.x + threadIdx.x) * 4; w < w1; w += stride)
    { if (w+4 <= w1)
        { uint4 acc = make_uint4(0,0,0,0);
          for (int p = 0; p < npeer; p++)
            { uint4 v = *reinterpret_cast<const uint4 *>(P.p[p]+w);
              acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
            }
          for (int p = 0; p < npeer; p++)
            *reinterpret_cast<uint4 *>(P.p[p]+w) = acc;
        }
      else
        for (int64_t u = w; u < w1; u++)
          { uint32_t acc = 0;
            for (int p = 0; p < npeer; p++) acc += P.p[p][u];
            for (int p = 0; p < npeer; p++) P.p[p][u] = acc;
          }
    }
}

int hm_peer_sum_deg(uint8_t **deg, const int64_t *lo, const int64_t *hi, const int *dev,
                    cudaStream_t *st, int n, int64_t nels)
{ (void) lo; (void) hi;
  DegPtrs P;
  int64_t words = (nels+3)/4;
  int64_t quads = (words+3)/4;
  for (int g = 0; g < n; g++)
    P.p[g] = (uint32_t *) deg[g];
  for (int g = 0; g < n; g++)                /* pass 1 finished everywhere */
    { HM_CUDA(cudaSetDevice(dev[g])); HM_CUDA(cudaStreamSynchronize(st[g])); }
  for (int g = 0; g < n; g++)
    { int64_t w0 = (quads*g/n)*4, w1 = (quads*(g+1)/n)*4;
      if (w1 > words) w1 = words;
      if (w0 >= w1) continue;
      HM_CUDA(cudaSetDevice(dev[g]));
      int64_t want = ((w1-w0)/4+255)/256;
      int     grid = (int) (want < 132*4 ? (want > 0 ? want : 1) : 132*4);
      peer_sum_deg_kernel<<<grid,256,0,st[g]>>>(P,n,w0,w1);
      cudaError_t e = cudaGetLastError();
      if (e != cudaSuccess) return hm_cuda_fail(e,"peer_sum_deg_kernel");
    }
  for (int g = 0; g < n; g++)                /* totals visible everywhere before pass 2 */
    { HM_CUDA(cudaSetDevice(dev[g])); HM_CUDA(cudaStreamSynchronize(st[g])); }
  return HM_OK;
}

__global__ void __launch_bounds__(256)
peer_sum_plot_kernel(PlotPtrs P, int npeer)
{ int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= HM_PLOT_CELLS)
    return;
  unsigned long long acc = P.p[0][t];
  for (int p = 1; p < npeer; p++)
    acc += P.p[p][t];
  P.p[0][t] = acc;
}

int hm_peer_sum_plot(unsigned long long **plot, const int *dev, cudaStream_t *st, int n)
{ PlotPtrs P;
  for (int g = 0; g < n; g++)
    P.p[g] = plot[g];
  for (int g = 1; g < n; g++)
    { HM_CUDA(cudaSetDevice(dev[g])); HM_CUDA(cudaStreamSynchronize(st[g])); }
  HM_CUDA(cudaSetDevice(dev[0]));
  peer_sum_plot_kernel<<<(HM_PLOT_CELLS+255)/256,256,0,st[0]>>>(P,n);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return hm_cuda_fail(e,"peer_sum_plot_kernel");
  return HM_OK;
}

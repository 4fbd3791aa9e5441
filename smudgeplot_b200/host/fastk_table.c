/*******************************************************************************************
 * fastk_table.c -- layer C of include/hetmers_b200.h: FastK .ktab stub/part parser and the
 * .smu writer.  Plain C host code, no CUDA.
 *
 * Restates what Open_Kmer_Stream does with the files (smudgeplot's src/lib/libfastk.c
 * :786-908): stub = int32 kmer,nparts,minval,ibyte + int64 index[1<<(8*ibyte)]; hidden part
 * files ".<root>.ktab.<p>" = int32 kmer, int64 n, then n records of kbyte-ibyte+2 bytes.
 * Unlike the reference (1024-entry read() buffers, :749-784) the part payloads are mapped whole
 * and handed to the GPU loader; and unlike the reference (:11 of Appendix C in SURVEY.md: read()
 * results unchecked) truncated files are reported.
 *******************************************************************************************/
#define _GNU_SOURCE
#include <errno.h>
#include <fcntl.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
#include <pthread.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include "hetmers_b200.h"
#include "hm_internal.h"

#define PART_HEADER 12      /* int32 kmer + int64 n   (libfastk.c:860-861) */

struct hm_table
  { hm_host_table   view;
    int64_t        *index;
    int64_t        *part_nels;
    const uint8_t **part_rec;
    void          **map_base;
    size_t         *map_len;
    int32_t        *part_fd;
    int64_t        *part_fd_off;
  };

/* dir and root of <name> as PathTo()/Root(name,".ktab") give them (gene_core.c:64-114) */
static void split_name(const char *name, char *dir, char *root)
{ const char *slash = strrchr(name,'/');
  const char *base  = slash ? slash+1 : name;
  size_t      n;

  if (slash == NULL)
    strcpy(dir,".");
  else if (slash == name)
    strcpy(dir,"/");
  else
    { memcpy(dir,name,(size_t) (slash-name)); dir[slash-name] = 0; }
  strcpy(root,base);
  n = strlen(root);
  if (n > 5 && strcasecmp(root+n-5,".ktab") == 0)
    root[n-5] = 0;
}

void hm_table_close(hm_table *t)
{ int p;
  if (t == NULL)
    return;
  if (t->map_base != NULL)
    for (p = 0; p < t->view.nparts; p++)
      if (t->map_base[p] != NULL)
        munmap(t->map_base[p],t->map_len[p]);
  if (t->part_fd != NULL)
    for (p = 0; p < t->view.nparts; p++)
      if (t->part_fd[p] >= 0)
        close(t->part_fd[p]);
  free(t->map_base); free(t->map_len); free(t->part_fd); free(t->part_fd_off);
  free(t->index); free(t->part_nels); free((void *) t->part_rec);
  free(t);
}

const hm_host_table *hm_table_view(const hm_table *t) { return &t->view; }

int hm_table_open(const char *name, hm_table **out)
{ hm_table *t;
  char     *dir, *root, *path;
  int       f, p, rc = HM_OK;
  int32_t   hdr[4];
  int64_t   ixlen, nels;
  int       kbyte, pbyte;

  if (name == NULL || out == NULL)
    return hm_set_error(HM_EINVAL,"hm_table_open: NULL argument");
  dir  = malloc(strlen(name)+8);
  root = malloc(strlen(name)+8);
  path = malloc(2*strlen(name)+64);
  t    = calloc(1,sizeof(hm_table));
  if (dir == NULL || root == NULL || path == NULL || t == NULL)
    { free(dir); free(root); free(path); free(t);
      return hm_set_error(HM_ENOMEM,"Out of memory (Allocating table record)");
    }
  split_name(name,dir,root);

  sprintf(path,"%s/%s.ktab",dir,root);
  f = open(path,O_RDONLY);
  if (f < 0)
    { rc = hm_set_error(HM_EIO,"Cannot open k-mer table %s",name); goto fail; }
  if (read(f,hdr,sizeof(hdr)) != (ssize_t) sizeof(hdr))
    { close(f); rc = hm_set_error(HM_EFORMAT,"%s: truncated stub header",path); goto fail; }
  t->view.kmer = hdr[0]; t->view.nparts = hdr[1]; t->view.minval = hdr[2]; t->view.ibyte = hdr[3];
  if (hdr[0] < 1 || hdr[1] < 0 || hdr[3] < 1 || hdr[3] > 3)
    { close(f); rc = hm_set_error(HM_EFORMAT,"%s: implausible stub header (k=%d parts=%d ibyte=%d)",
                                  path,hdr[0],hdr[1],hdr[3]); goto fail; }
  kbyte = (hdr[0]+3)>>2;
  if (hdr[3] > kbyte)
    { close(f); rc = hm_set_error(HM_EFORMAT,"%s: ibyte=%d exceeds k-mer bytes %d",path,hdr[3],kbyte); goto fail; }
  pbyte = kbyte-hdr[3]+2;
  ixlen = ((int64_t) 1) << (8*hdr[3]);
  t->index = malloc(sizeof(int64_t)*(size_t) ixlen);
  if (t->index == NULL)
    { close(f); rc = hm_set_error(HM_ENOMEM,"Out of memory (Allocating table prefix index)"); goto fail; }
  { size_t want = sizeof(int64_t)*(size_t) ixlen, got = 0;
    while (got < want)
      { ssize_t r = read(f,((char *) t->index)+got,want-got);
        if (r <= 0) break;
        got += (size_t) r;
      }
    close(f);
    if (got != want)
      { rc = hm_set_error(HM_EFORMAT,"%s: truncated prefix index",path); goto fail; }
  }
  t->view.index = t->index;

  t->part_nels = calloc((size_t) hdr[1]+1,sizeof(int64_t));
  t->part_rec  = calloc((size_t) hdr[1]+1,sizeof(uint8_t *));
  t->map_base  = calloc((size_t) hdr[1]+1,sizeof(void *));
  t->map_len   = calloc((size_t) hdr[1]+1,sizeof(size_t));
  t->part_fd     = malloc(((size_t) hdr[1]+1)*sizeof(int32_t));
  t->part_fd_off = calloc((size_t) hdr[1]+1,sizeof(int64_t));
  if (t->part_fd != NULL)
    for (p = 0; p <= hdr[1]; p++)
      t->part_fd[p] = -1;
  if (t->part_nels == NULL || t->part_rec == NULL || t->map_base == NULL || t->map_len == NULL ||
      t->part_fd == NULL || t->part_fd_off == NULL)
    { rc = hm_set_error(HM_ENOMEM,"Out of memory (Allocating parts table)"); goto fail; }
  t->view.part_nels   = t->part_nels;
  t->view.part_rec    = t->part_rec;
  t->view.part_fd     = t->part_fd;
  t->view.part_fd_off = t->part_fd_off;

  nels = 0;
  for (p = 1; p <= hdr[1]; p++)
    { struct stat sb;
      int32_t pk;
      int64_t n;
      char    head[PART_HEADER];
      void   *m;

      sprintf(path,"%s/.%s.ktab.%d",dir,root,p);
      f = open(path,O_RDONLY);
      if (f < 0)
        { rc = hm_set_error(HM_EIO,"Table part %s is missing ?",path); goto fail; }      /* libfastk.c:851 */
      if (read(f,head,PART_HEADER) != PART_HEADER || fstat(f,&sb) != 0)
        { close(f); rc = hm_set_error(HM_EFORMAT,"Table part %s is truncated",path); goto fail; }
      memcpy(&pk,head,4); memcpy(&n,head+4,8);
      if (pk != hdr[0])
        { close(f);
          rc = hm_set_error(HM_EFORMAT,"Table part %s does not have k-mer length matching stub ?",path);
          goto fail;                                                                        /* libfastk.c:859 */
        }
      if (n < 0 || (int64_t) sb.st_size < PART_HEADER + n*pbyte)
        { close(f); rc = hm_set_error(HM_EFORMAT,"Table part %s is truncated",path); goto fail; }
      if (n > 0)
        { size_t len = (size_t) (PART_HEADER + n*pbyte);
          m = mmap(NULL,len,PROT_READ,MAP_PRIVATE,f,0);
          if (m == MAP_FAILED)
            { close(f); rc = hm_set_error(HM_EIO,"cannot map %s: %s",path,strerror(errno)); goto fail; }
          t->map_base[p-1] = m;
          t->map_len[p-1]  = len;
          t->part_rec[p-1] = ((const uint8_t *) m)+PART_HEADER;
          t->part_fd[p-1]     = f;               /* kept open: the GPU loader pread()s the payload */
          t->part_fd_off[p-1] = PART_HEADER;
        }
      else
        close(f);
      t->part_nels[p-1] = n;
      nels += n;
    }
  t->view.nels = nels;
  free(dir); free(root); free(path);
  *out = t;
  return HM_OK;

fail:
  free(dir); free(root); free(path);
  hm_table_close(t);
  return rc;
}

/* ---- incremental writer ------------------------------------------------------------------------
 * Records arrive in table order, announced bucket by bucket (hm_table_write_buckets) before they are
 * appended.  Part q (q = 1..nparts-1) ends where fastk.write_ktab(cut_on_buckets=True) ends it for a
 * table of nels_hint entries: at the start of the bucket holding ordinal nels_hint*q/nparts (the last
 * bucket's start when there are fewer entries).  That bucket may have begun before the ordinal is
 * reached, so a cut moves the bucket's records written so far from the old part to the new one --
 * at most one bucket's worth per part.  Everything is written under temporary names and renamed into
 * place by hm_table_write_close; any failure removes the temporaries.
 *
 * Positional mode (hm_table_write_place / _at / _seal): ranges are announced in table order, each getting its
 * first ordinal, and their records are written at their final offsets by any thread in any order.  A cut is
 * fixed the moment the bucket holding its ordinal is announced (at that bucket's start, as the append path
 * cuts); until then it lies at or after the start of the last bucket announced, so only records of that bucket
 * can be in doubt.  hm_table_write_at never waits: it copies those records and the place or seal that settles
 * them writes them (at most one bucket's records are held).  Nothing written is ever moved.                 */
static int pwrite_all(int fd, const void *buf, size_t len, off_t off)
{ const char *b = (const char *) buf;
  while (len > 0)
    { ssize_t r = pwrite(fd,b,len,off);
      if (r <= 0) return -1;
      b += r; len -= (size_t) r; off += r;
    }
  return 0;
}

typedef struct pending { int64_t first, n; struct pending *next; uint8_t rec[]; } pending;

struct hm_table_writer
  { int      kmer, ibyte, minval, nparts, pbyte, part;   /* part: the one being written (0-based)  */
    int64_t  hint, ixlen;
    int64_t *count;                    /* records per bucket, as announced                         */
    int64_t  declared, written, last;  /* records announced / appended; last bucket announced      */
    int64_t  cur, cur_start, cur_left; /* bucket being appended, its first ordinal, records to come */
    int64_t *part_first;               /* [nparts] first ordinal of each part                      */
    int     *fd;                       /* [nparts] temporary part files                            */
    char    *dir, *root, *tmp_tag;
    int      failed;
    int      positional, sealed, known;/* (positional) part_first[0, known) is fixed               */
    int64_t  last_start;               /* (positional) first ordinal of the last bucket announced  */
    struct pending *held;              /* (positional) records written while their part was open  */
    int64_t  held_from;                /*   the open ordinal they wait on (the last bucket's start)*/
    pthread_mutex_t mu;                /* (positional) guards the above, declared and written      */
    uint8_t *mem;                      /* memory target (one part): room for mem_cap records, else */
    int64_t  mem_cap;                  /*   NULL and the records go to the part files             */
  };

/* n bytes at byte offset off of part p's payload: into the part file, or the memory target's buffer */
static int writer_sink(const hm_table_writer *w, int p, const void *buf, size_t n, off_t off)
{ if (w->mem != NULL)
    { memcpy(w->mem+off,buf,n);
      return 0;
    }
  return pwrite_all(w->fd[p],buf,n,PART_HEADER+off);
}

/* records to announce beyond the memory target's room (the records every later call assumes placed) */
static int writer_over(const hm_table_writer *w, int64_t more)
{ return w->mem != NULL && w->declared+more > w->mem_cap;
}

static char *writer_path(const hm_table_writer *w, int part, int tmp)   /* part 0 = the stub */
{ size_t len = strlen(w->dir)+strlen(w->root)+strlen(w->tmp_tag)+48;
  char  *p = malloc(len);
  if (p == NULL)
    return NULL;
  if (part == 0) snprintf(p,len,"%s/%s.ktab%s",w->dir,w->root,tmp ? w->tmp_tag : "");
  else           snprintf(p,len,"%s/.%s.ktab.%d%s",w->dir,w->root,part,tmp ? w->tmp_tag : "");
  return p;
}

static void writer_free(hm_table_writer *w, int unlink_tmp)
{ if (w == NULL)
    return;
  for (int p = 0; p < w->nparts && w->fd != NULL; p++)
    { if (w->fd[p] >= 0) close(w->fd[p]);
      if (unlink_tmp)
        { char *q = writer_path(w,p+1,1);
          if (q != NULL) { unlink(q); free(q); }
        }
    }
  if (unlink_tmp && w->dir != NULL)
    { char *q = writer_path(w,0,1);
      if (q != NULL) { unlink(q); free(q); }
    }
  free(w->count); free(w->part_first); free(w->fd); free(w->dir); free(w->root); free(w->tmp_tag); free(w->mem);
  while (w->held != NULL)
    { pending *nx = w->held->next;
      free(w->held);
      w->held = nx;
    }
  pthread_mutex_destroy(&w->mu);
  free(w);
}

void hm_table_write_abort(hm_table_writer *w) { writer_free(w,1); }

/* the writer's state shared by both targets (*out = NULL on failure) */
static int writer_new(int kmer, int ibyte, int minval, int nparts, int64_t nels_hint, hm_table_writer **out)
{ hm_table_writer *w = calloc(1,sizeof(*w));
  *out = NULL;
  if (w == NULL)
    return hm_set_error(HM_ENOMEM,"Out of memory (table writer)");
  w->kmer = kmer; w->ibyte = ibyte; w->minval = minval; w->nparts = nparts; w->hint = nels_hint;
  w->pbyte = ((kmer+3)>>2) - ibyte + 2;
  w->ixlen = (int64_t) 1 << (8*ibyte);
  w->cur = -1;
  w->known = 1;
  pthread_mutex_init(&w->mu,NULL);
  w->count      = calloc((size_t) w->ixlen,sizeof(int64_t));
  w->part_first = calloc((size_t) nparts,sizeof(int64_t));
  if (w->count == NULL || w->part_first == NULL)
    { writer_free(w,0); return hm_set_error(HM_ENOMEM,"Out of memory (table writer)"); }
  *out = w;
  return HM_OK;
}

int hm_table_write_open_host(int kmer, int ibyte, int minval, int64_t nels_cap, hm_table_writer **out)
{ hm_table_writer *w;
  if (out == NULL || kmer < 1 || ibyte < 1 || ibyte > 3 || ibyte > ((kmer+3)>>2) || nels_cap < 0)
    return hm_set_error(HM_EINVAL,"hm_table_write_open_host: bad arguments");
  int rc = writer_new(kmer,ibyte,minval,1,0,&w);
  if (rc != HM_OK)
    return rc;
  w->mem_cap = nels_cap;
  w->mem     = malloc(nels_cap > 0 ? (size_t) (nels_cap*w->pbyte) : 1);
  if (w->mem == NULL)
    { rc = hm_set_error(HM_ENOMEM,"Out of memory (a table of %lld records: %lld host bytes)",(long long) nels_cap,
                        (long long) (nels_cap*w->pbyte));
      writer_free(w,0);
      return rc;
    }
  *out = w;
  return HM_OK;
}

int hm_table_write_open(const char *name, int kmer, int ibyte, int minval, int nparts, int64_t nels_hint,
                        hm_table_writer **out)
{ hm_table_writer *w;
  if (name == NULL || out == NULL || kmer < 1 || ibyte < 1 || ibyte > 3 || ibyte > ((kmer+3)>>2) ||
      nparts < 1 || nels_hint < 0)
    return hm_set_error(HM_EINVAL,"hm_table_write_open: bad arguments");
  int rc = writer_new(kmer,ibyte,minval,nparts,nels_hint,&w);
  if (rc != HM_OK)
    return rc;
  w->fd         = malloc(sizeof(int)*(size_t) nparts);
  w->dir        = malloc(strlen(name)+8);
  w->root       = malloc(strlen(name)+8);
  w->tmp_tag    = malloc(64);
  for (int p = 0; p < nparts && w->fd != NULL; p++) w->fd[p] = -1;
  if (w->fd == NULL || w->dir == NULL || w->root == NULL || w->tmp_tag == NULL)
    { writer_free(w,0); return hm_set_error(HM_ENOMEM,"Out of memory (table writer)"); }
  split_name(name,w->dir,w->root);
  snprintf(w->tmp_tag,64,".tmp%ld",(long) getpid());
  for (int p = 0; p < nparts; p++)
    { char   *q = writer_path(w,p+1,1);
      char    head[PART_HEADER];
      int32_t k32 = kmer;
      int64_t zero = 0;
      if (q == NULL)
        { writer_free(w,1); return hm_set_error(HM_ENOMEM,"Out of memory (table writer)"); }
      w->fd[p] = open(q,O_RDWR|O_CREAT|O_TRUNC,0644);
      memcpy(head,&k32,4); memcpy(head+4,&zero,8);
      if (w->fd[p] < 0 || pwrite_all(w->fd[p],head,PART_HEADER,0) != 0)
        { int rc = hm_set_error(HM_EIO,"Cannot create %s: %s",q,strerror(errno));
          free(q); writer_free(w,1);
          return rc;
        }
      free(q);
    }
  *out = w;
  return HM_OK;
}

int hm_table_write_buckets(hm_table_writer *w, int64_t b0, int64_t nb, const int64_t *counts)
{ if (w == NULL || w->failed || w->positional)
    return hm_set_error(HM_EINVAL,"hm_table_write_buckets: no usable writer");
  for (int64_t i = 0; i < nb; i++)
    { int64_t b = b0+i;
      if (counts[i] == 0)
        continue;
      if (b < 0 || b >= w->ixlen || counts[i] < 0 || b < w->last)
        { w->failed = 1;
          return hm_set_error(HM_EINVAL,"hm_table_write_buckets: bucket %lld announced out of order",(long long) b);
        }
      if (writer_over(w,counts[i]))
        { w->failed = 1;
          return hm_set_error(HM_EINVAL,"hm_table_write_buckets: more than the %lld records the table has room for",
                              (long long) w->mem_cap);
        }
      w->count[b] += counts[i];
      w->declared += counts[i];
      w->last = b;
      if (b == w->cur)                                      /* more of the bucket being appended */
        w->cur_left += counts[i];
    }
  return HM_OK;
}

/* part w->part+1 begins at ordinal `at` (<= written): the records [at, written) move into it */
static int writer_cut(hm_table_writer *w, int64_t at)
{ int     p = w->part, q = p+1;
  int64_t moved = w->written-at;
  off_t   src = PART_HEADER + (off_t) (at-w->part_first[p])*w->pbyte;
  char    buf[1 << 16];
  int64_t left = moved*w->pbyte;
  off_t   o = 0;
  while (left > 0)
    { size_t  m = left < (int64_t) sizeof(buf) ? (size_t) left : sizeof(buf);
      ssize_t r = pread(w->fd[p],buf,m,src+o);
      if (r != (ssize_t) m || pwrite_all(w->fd[q],buf,m,PART_HEADER+o) != 0)
        return hm_set_error(HM_EIO,"writing table part %d: %s",q+1,strerror(errno));
      o += (off_t) m; left -= (int64_t) m;
    }
  if (ftruncate(w->fd[p],src) != 0)
    return hm_set_error(HM_EIO,"writing table part %d: %s",p+1,strerror(errno));
  w->part = q;
  w->part_first[q] = at;
  return HM_OK;
}

/* the ordinal part q+1 is cut at (write_ktab's c = n*q/nparts), for q = w->part+1 */
static int64_t writer_target(const hm_table_writer *w, int q)
{ return (int64_t) ((__int128) w->hint*q/w->nparts); }

/* records [from, w->written) of the current part, held at rec, go to its file in one write */
static int writer_flush(hm_table_writer *w, const uint8_t *rec, int64_t from)
{ if (w->written > from &&
      writer_sink(w,w->part,rec,(size_t) (w->written-from)*w->pbyte,(off_t) (from-w->part_first[w->part])*w->pbyte) != 0)
    return hm_set_error(HM_EIO,"writing table part %d: %s",w->part+1,strerror(errno));
  return HM_OK;
}

int hm_table_write_append(hm_table_writer *w, const uint8_t *rec, int64_t n)
{ if (w == NULL || w->failed || w->positional)
    return hm_set_error(HM_EINVAL,"hm_table_write_append: no usable writer");
  if (w->written+n > w->declared)
    { w->failed = 1;
      return hm_set_error(HM_EINVAL,"hm_table_write_append: %lld records beyond the announced buckets",
                          (long long) (w->written+n-w->declared));
    }
  int64_t from = w->written;                                /* not yet in a file: [from, written) at rec */
  while (n > 0)
    { if (w->cur_left == 0)                                 /* the next non-empty bucket starts here */
        { do w->cur++; while (w->count[w->cur] == 0);
          w->cur_start = w->written;
          w->cur_left  = w->count[w->cur];
        }
      int64_t m = n < w->cur_left ? n : w->cur_left;
      /* cuts whose ordinal falls in [written, written+m) lie in this bucket: they begin at its start */
      while (w->part+1 < w->nparts && w->hint > 0 && writer_target(w,w->part+1) < w->written+m)
        { if (writer_flush(w,rec,from) != HM_OK || writer_cut(w,w->cur_start) != HM_OK)
            { w->failed = 1; return HM_EIO; }
          rec += (w->written-from)*w->pbyte;
          from = w->written;
        }
      n -= m; w->written += m; w->cur_left -= m;
    }
  if (writer_flush(w,rec,from) != HM_OK)
    { w->failed = 1; return HM_EIO; }
  return HM_OK;
}

/* ---- positional mode ---- */

/* records [first, first+n) at rec into their parts; pf[0, known): the fixed part starts, every cut not yet fixed
 * lying at or beyond first+n -- the part of ordinal o is the last p with pf[p] <= o                          */
static int writer_put(const hm_table_writer *w, const int64_t *pf, int known, int64_t first, const uint8_t *rec,
                      int64_t n)
{ const int64_t end = first+n;
  int p = 0;
  for (int64_t o = first; o < end; )
    { while (p+1 < known && pf[p+1] <= o) p++;
      int64_t e = p+1 < known && pf[p+1] < end ? pf[p+1] : end;
      if (writer_sink(w,p,rec+(o-first)*w->pbyte,(size_t) (e-o)*w->pbyte,(off_t) (o-pf[p])*w->pbyte) != 0)
        return hm_set_error(HM_EIO,"writing table part %d: %s",p+1,strerror(errno));
      o = e;
    }
  return HM_OK;
}

/* the first ordinal whose part may still change: the last bucket's start while a cut is open, else none */
static int64_t writer_open_from(const hm_table_writer *w)
{ return w->known < w->nparts && w->hint > 0 ? w->last_start : INT64_MAX; }

/* (mutex held) the part starts fixed so far, copied to *pf (cut or malloc'ed); 0 when out of memory */
static int writer_cuts(hm_table_writer *w, int64_t *cut, int64_t **pf)
{ *pf = cut;
  if (w->known > 64 && (*pf = malloc(sizeof(int64_t)*(size_t) w->known)) == NULL)
    return 0;
  memcpy(*pf,w->part_first,sizeof(int64_t)*(size_t) w->known);
  return 1;
}

/* (mutex held, released on return) the held records are written once nothing held can change part any more */
static int writer_release(hm_table_writer *w)
{ pending *q = NULL;
  int64_t  cut[64], *pf = cut;
  int      known = w->known, rc = HM_OK;
  if (w->held != NULL && !w->failed && writer_open_from(w) > w->held_from)
    { q = w->held; w->held = NULL;
      if (!writer_cuts(w,cut,&pf))
        { w->failed = 1; rc = hm_set_error(HM_ENOMEM,"Out of memory (table writer)"); }
    }
  pthread_mutex_unlock(&w->mu);
  while (q != NULL)
    { pending *nx = q->next;
      if (rc == HM_OK) rc = writer_put(w,pf,known,q->first,q->rec,q->n);
      free(q);
      q = nx;
    }
  if (pf != cut) free(pf);
  if (rc != HM_OK)
    { pthread_mutex_lock(&w->mu); w->failed = 1; pthread_mutex_unlock(&w->mu); }
  return rc;
}

int hm_table_write_place(hm_table_writer *w, int64_t b0, int64_t nb, const int64_t *counts, int64_t *first)
{ int rc = HM_OK;
  if (w == NULL || first == NULL || nb < 0 || (nb > 0 && counts == NULL))
    return hm_set_error(HM_EINVAL,"hm_table_write_place: bad arguments");
  pthread_mutex_lock(&w->mu);
  if (w->failed || w->sealed || (!w->positional && w->declared > 0))
    rc = hm_set_error(HM_EINVAL,"hm_table_write_place: no usable writer");
  else
    w->positional = 1;
  *first = w->declared;
  for (int64_t i = 0; i < nb && rc == HM_OK; i++)
    { int64_t b = b0+i;
      if (counts[i] == 0)
        continue;
      if (b < 0 || b >= w->ixlen || counts[i] < 0 || b < w->last)
        { w->failed = 1;
          rc = hm_set_error(HM_EINVAL,"hm_table_write_place: bucket %lld announced out of order",(long long) b);
          break;
        }
      if (writer_over(w,counts[i]))
        { w->failed = 1;
          rc = hm_set_error(HM_EINVAL,"hm_table_write_place: more than the %lld records the table has room for",
                            (long long) w->mem_cap);
          break;
        }
      if (w->declared == 0 || b != w->last)                 /* a new bucket starts here */
        w->last_start = w->declared;
      w->count[b] += counts[i];
      w->declared += counts[i];
      w->last = b;
      while (w->known < w->nparts && w->hint > 0 && writer_target(w,w->known) < w->declared)
        w->part_first[w->known++] = w->last_start;          /* the bucket holding the cut's ordinal */
    }
  if (rc != HM_OK)
    { pthread_mutex_unlock(&w->mu);
      return rc;
    }
  return writer_release(w);
}

static int writer_seal(hm_table_writer *w)
{ pthread_mutex_lock(&w->mu);
  w->sealed = 1;
  while (w->known < w->nparts)
    w->part_first[w->known++] = w->hint > 0 && w->declared > 0 ? w->last_start : w->declared;
  return writer_release(w);
}

void hm_table_write_seal(hm_table_writer *w)
{ if (w != NULL)
    writer_seal(w);
}

int hm_table_write_at(hm_table_writer *w, int64_t first, const uint8_t *rec, int64_t n)
{ if (w == NULL || first < 0 || n < 0 || (n > 0 && rec == NULL))
    return hm_set_error(HM_EINVAL,"hm_table_write_at: bad arguments");
  const int64_t end = first+n;
  int64_t cut[64], *pf = cut;
  pthread_mutex_lock(&w->mu);
  if (w->failed || !w->positional || end > w->declared)
    { if (w->positional && !w->failed && end > w->declared) w->failed = 1;
      pthread_mutex_unlock(&w->mu);
      return hm_set_error(HM_EINVAL,"hm_table_write_at: no usable writer or records %lld..%lld not placed",
                          (long long) first,(long long) end);
    }
  /* records from the last bucket's start on may still fall on either side of an open cut: held (copied) until
   * a later place or the seal fixes it; the rest go to their files now                                      */
  const int64_t open = writer_open_from(w);
  const int64_t mid = end < open ? end : (first > open ? first : open);
  int rc = HM_OK;
  if (mid < end)
    { pending *q = malloc(sizeof(pending) + (size_t) (end-mid)*w->pbyte);
      if (q == NULL)
        rc = hm_set_error(HM_ENOMEM,"Out of memory (table writer)");
      else
        { q->first = mid; q->n = end-mid;
          memcpy(q->rec,rec+(mid-first)*w->pbyte,(size_t) (end-mid)*w->pbyte);
          if (w->held == NULL) w->held_from = open;
          q->next = w->held; w->held = q;
        }
    }
  const int known = w->known;
  if (rc == HM_OK && !writer_cuts(w,cut,&pf))
    rc = hm_set_error(HM_ENOMEM,"Out of memory (table writer)");
  if (rc != HM_OK)
    { w->failed = 1;
      pthread_mutex_unlock(&w->mu);
      return rc;
    }
  pthread_mutex_unlock(&w->mu);
  rc = writer_put(w,pf,known,first,rec,mid-first);
  if (pf != cut) free(pf);
  pthread_mutex_lock(&w->mu);
  if (rc == HM_OK) w->written += n;
  else             w->failed = 1;
  pthread_mutex_unlock(&w->mu);
  return rc;
}

/* what closing takes on either target: positional, the cuts not reached are fixed (as hm_table_write_close fixes
 * them) and the records still held written; then every announced record must have been written.  w is freed on
 * failure.                                                                                                    */
static int writer_finish(hm_table_writer *w, const char *who)
{ int rc;
  if (w->positional && writer_seal(w) != HM_OK)
    { writer_free(w,1);
      return HM_EIO;
    }
  if (w->failed || w->written != w->declared)
    { rc = w->failed ? hm_set_error(HM_EINVAL,"%s: an earlier call failed",who)
                     : hm_set_error(HM_EINVAL,"%s: %lld announced records were not appended",who,
                                    (long long) (w->declared-w->written));
      writer_free(w,1);
      return rc;
    }
  return HM_OK;
}

/* the memory target's table: its records and index leave the writer with it */
typedef struct
  { hm_host_table  view;
    int64_t        part_nels[1];
    const uint8_t *part_rec[1];
  } host_table;

int hm_table_write_close_host(hm_table_writer *w, hm_host_table **out)
{ int rc;
  if (w == NULL || out == NULL || w->mem == NULL)
    { writer_free(w,1);
      return hm_set_error(HM_EINVAL,"hm_table_write_close_host: no memory writer");
    }
  *out = NULL;
  if ((rc = writer_finish(w,"hm_table_write_close_host")) != HM_OK)
    return rc;
  host_table *h = calloc(1,sizeof(*h));
  if (h == NULL)
    { writer_free(w,1);
      return hm_set_error(HM_ENOMEM,"Out of memory (table record)");
    }
  int64_t acc = 0;
  for (int64_t b = 0; b < w->ixlen; b++)                    /* counts -> bucket END offsets, as the stub holds */
    { acc += w->count[b]; w->count[b] = acc; }
  if (w->written > 0 && w->written < w->mem_cap)            /* the room was a bound: give back what was not used */
    { uint8_t *m = realloc(w->mem,(size_t) (w->written*w->pbyte));
      if (m != NULL) w->mem = m;
    }
  h->part_nels[0] = w->written;
  h->part_rec[0]  = w->mem;
  h->view.kmer = w->kmer; h->view.ibyte = w->ibyte; h->view.nparts = 1; h->view.minval = w->minval;
  h->view.nels = w->written;
  h->view.index = w->count;
  h->view.part_nels = h->part_nels;
  h->view.part_rec  = h->part_rec;
  w->count = NULL; w->mem = NULL;
  writer_free(w,1);
  *out = &h->view;
  return HM_OK;
}

void hm_host_table_free(hm_host_table *t)
{ if (t == NULL)
    return;
  free((void *) t->index);
  free((void *) t->part_rec[0]);
  free(t);
}

int hm_table_write_close(hm_table_writer *w)
{ int rc = HM_OK;
  if (w == NULL)
    return hm_set_error(HM_EINVAL,"hm_table_write_close: no writer");
  if (w->mem != NULL)
    { writer_free(w,1);
      return hm_set_error(HM_EINVAL,"hm_table_write_close: a memory writer closes with hm_table_write_close_host");
    }
  if ((rc = writer_finish(w,"hm_table_write_close")) != HM_OK)
    return rc;
  /* cuts not reached (fewer entries than the hint): at the last bucket's start, as write_ktab cuts */
  while (rc == HM_OK && !w->positional && w->part+1 < w->nparts)
    rc = writer_cut(w,w->hint > 0 && w->written > 0 ? w->cur_start : w->written);
  for (int p = 0; p < w->nparts && rc == HM_OK; p++)
    { int64_t end = p+1 < w->nparts ? w->part_first[p+1] : w->written;
      int64_t cnt = end-w->part_first[p];
      if (pwrite_all(w->fd[p],&cnt,8,4) != 0)
        rc = hm_set_error(HM_EIO,"writing table part %d: %s",p+1,strerror(errno));
    }
  char *stub = writer_path(w,0,1);
  if (rc == HM_OK)
    { int     f = stub ? open(stub,O_WRONLY|O_CREAT|O_TRUNC,0644) : -1;
      int32_t hdr[4] = { w->kmer, w->nparts, w->minval, w->ibyte };
      int64_t acc = 0;
      for (int64_t b = 0; b < w->ixlen; b++)                /* counts -> bucket END offsets */
        { acc += w->count[b]; w->count[b] = acc; }
      if (f < 0 || pwrite_all(f,hdr,sizeof(hdr),0) != 0 ||
          pwrite_all(f,w->count,sizeof(int64_t)*(size_t) w->ixlen,sizeof(hdr)) != 0)
        rc = hm_set_error(HM_EIO,"Cannot write %s: %s",stub ? stub : "table stub",strerror(errno));
      if (f >= 0 && close(f) != 0 && rc == HM_OK)
        rc = hm_set_error(HM_EIO,"Cannot write %s: %s",stub,strerror(errno));
    }
  for (int p = 0; p < w->nparts; p++)
    { if (w->fd[p] >= 0 && close(w->fd[p]) != 0 && rc == HM_OK)
        rc = hm_set_error(HM_EIO,"writing table part %d: %s",p+1,strerror(errno));
      w->fd[p] = -1;
    }
  /* into place: the parts, then (last) the stub that names them; parts an older table of this name
   * had beyond nparts go                                                                           */
  int old_parts = 0;
  { char *final = writer_path(w,0,0);
    int   f = final ? open(final,O_RDONLY) : -1;
    int32_t hdr[4];
    if (f >= 0 && read(f,hdr,sizeof(hdr)) == (ssize_t) sizeof(hdr) && hdr[1] > 0)
      old_parts = hdr[1];
    if (f >= 0) close(f);
    free(final);
  }
  int renamed = 0;
  for (int p = 0; p <= w->nparts && rc == HM_OK; p++)
    { int   part = p < w->nparts ? p+1 : 0;
      char *a = writer_path(w,part,1), *b = writer_path(w,part,0);
      if (a == NULL || b == NULL || rename(a,b) != 0)
        rc = hm_set_error(HM_EIO,"Cannot rename %s into place: %s",a ? a : "table part",strerror(errno));
      else
        renamed = p+1;
      free(a); free(b);
    }
  if (rc != HM_OK)                                          /* nothing half-written under the final names */
    for (int p = 0; p < renamed && p < w->nparts; p++)
      { char *b = writer_path(w,p+1,0);
        if (b != NULL) { unlink(b); free(b); }
      }
  else
    for (int p = w->nparts+1; p <= old_parts; p++)
      { char *b = writer_path(w,p,0);
        if (b != NULL) { unlink(b); free(b); }
      }
  free(stub);
  writer_free(w,1);
  return rc;
}

/* "min \t sum-min \t count" for sum ascending, then min ascending, min < FMAX only
 * (PloidyPlot.c:1612-1615; the i < FMAX bound silently drops bin 500, kept for parity)        */
int hm_write_smu(const char *path, const int64_t *plot)
{ FILE *f = fopen(path,"w");
  int   a, i;
  if (f == NULL)
    return hm_set_error(HM_EIO,"Could not open %s",path);
  for (a = 0; a <= HM_SMAX; a++)
    for (i = 0; i < HM_FMAX; i++)
      if (plot[a*HM_PLOT_W+i] > 0)
        fprintf(f,"%i\t%i\t%lld\n",i,a-i,(long long) plot[a*HM_PLOT_W+i]);
  if (fclose(f) != 0)
    return hm_set_error(HM_EIO,"error writing %s",path);
  return HM_OK;
}

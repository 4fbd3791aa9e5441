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
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>
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

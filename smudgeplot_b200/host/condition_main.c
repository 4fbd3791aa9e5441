/*******************************************************************************************
 * condition_main.c -- `condition_kmer_table`: trim and symmetrise a FastK table of any size on the
 * GPU into a new table, the conditioning `hetmers` needs before it scans (plain C host; the work is
 * hm_scan_condition_files of include/hetmers_b200.h, DESIGN.md §4d).
 *
 *     condition_kmer_table [-v] [-T<int(4)>] [-e<int(4)>] <source>[.ktab] <target>[.ktab]
 *
 * It takes hetmers' decisions (hm_scan_examine with the same -e): trim if the table is untrimmed,
 * symmetrise if the probe finds it not symmetric; -v prints hetmers' verdict and step lines.  A table
 * that needs neither is left alone: nothing is written and the exit code is 0.  Tables larger than the
 * GPU are streamed (HETMERS_DEVICE_BUDGET and HETMERS_STREAM as for hetmers).  HETMERS_GPUS=<n>|all (default 1,
 * as for hetmers) scans on devices 0..n-1 and conditions on all of them: the key ranges are dealt round-robin and
 * each GPU's writer thread writes its ranges' records at their offsets; the files are those of one GPU.
 * Then `hetmers <target>` finds the table trimmed and symmetric and scans it, streamed if it must.
 *******************************************************************************************/
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <strings.h>

#include "hetmers_b200.h"

static const char *Prog_Name = "condition_kmer_table";

static int positive_arg(const char *arg, const char *what)
{ char *eptr;
  long  v = strtol(arg+2,&eptr,10);
  if (*eptr != '\0' || arg[2] == '\0')
    { fprintf(stderr,"%s: -%c '%s' argument is not an integer\n",Prog_Name,arg[1],arg+2);
      exit (1);
    }
  if (v <= 0)
    { fprintf(stderr,"%s: %s must be positive (%d)\n",Prog_Name,what,(int) v);
      exit (1);
    }
  return ((int) v);
}

/* HETMERS_GPUS as hetmers reads it: <n> or "all", default 1, at most the visible devices (with a warning) and 16;
 * main has already refused a machine with no visible device                                                  */
static int pick_gpus(int *devs)
{ int ngpu = 1, navail = hm_device_count(), i;
  const char *g = getenv("HETMERS_GPUS");

  if (g != NULL && *g != '\0')
    { if (strcasecmp(g,"all") == 0)
        ngpu = navail;
      else
        ngpu = atoi(g);
      if (ngpu < 1) ngpu = 1;
      if (ngpu > navail)
        { fprintf(stderr,"%s: Warning, only %d GPUs are visible\n",Prog_Name,navail);
          ngpu = navail;
        }
    }
  if (ngpu > 16) ngpu = 16;
  for (i = 0; i < ngpu; i++)
    devs[i] = i;
  return (ngpu);
}

static void die_hm(void)
{ fprintf(stderr,"%s: %s\n",Prog_Name,hm_last_error());
  exit (1);
}

int main(int argc, char *argv[])
{ int VERBOSE = 0, NTHREADS = 4, ETHRESH = 4;
  int i, j, k;

  j = 1;
  for (i = 1; i < argc; i++)
    if (argv[i][0] == '-')
      switch (argv[i][1])
      { default:
          for (k = 1; argv[i][k] != '\0'; k++)
            { if (argv[i][k] != 'v')
                { fprintf(stderr,"%s: -%c is an illegal option\n",Prog_Name,argv[i][k]);
                  exit (1);
                }
              VERBOSE = 1;
            }
          break;
        case 'e':
          ETHRESH = positive_arg(argv[i],"Error-mer threshold");
          break;
        case 'T':
          NTHREADS = positive_arg(argv[i],"Number of threads");
          if (NTHREADS > 64)
            { fprintf(stderr,"%s: Warning, only 64 threads will be used\n",Prog_Name);
              NTHREADS = 64;
            }
          break;
      }
    else
      argv[j++] = argv[i];
  argc = j;

  if (argc != 3)
    { fprintf(stderr,"\nUsage: %s [-v] [-T<int(4)>] [-e<int(4)>] <source>[.ktab] <target>[.ktab]\n",Prog_Name);
      fprintf(stderr,"\n");
      fprintf(stderr,"      -e: count threshold below which k-mers are considered erroneous\n");
      fprintf(stderr,"      -v: verbose mode\n");
      fprintf(stderr,"      -T: number of threads to use\n");
      exit (1);
    }

  hm_table *T;
  hm_scan  *S;
  int       dev[16], ngpu, trim, symm;

  if (hm_table_open(argv[1],&T) != HM_OK)
    { if (strncmp(hm_last_error(),"Cannot open",11) == 0)
        fprintf(stderr,"%s: Cannot open k-mer table %s\n",Prog_Name,argv[1]);
      else
        fprintf(stderr,"%s: %s\n",Prog_Name,hm_last_error());
      exit (1);
    }
  if (hm_device_count() < 1)
    { fprintf(stderr,"%s: no CUDA device is visible (conditioning runs on the GPU)\n",Prog_Name);
      exit (1);
    }
  hm_set_io_threads(NTHREADS);
  { const char *b = getenv("HETMERS_DEVICE_BUDGET");       /* device bytes per GPU, as for hetmers */
    if (b != NULL && *b != '\0')
      hm_set_device_budget(strtoll(b,NULL,10));
  }
  ngpu = pick_gpus(dev);
  if (hm_scan_create(hm_table_view(T),dev,ngpu,&S) != HM_OK)
    die_hm();
  hm_set_condition_gpus(ngpu);
  if (hm_scan_examine(S,ETHRESH,&trim,&symm) != HM_OK)
    die_hm();

  if (VERBOSE)
    { fprintf(stderr,"\n  The input table is");
      if (trim)
        fprintf(stderr,symm ? " trimmed and symmetric\n" : " trimmed but not symmetric\n");
      else
        fprintf(stderr,symm ? " untrimmed yet symmetric\n" : " untrimmed and not symmetric\n");
    }

  if (trim && symm)
    { fprintf(stderr,"%s: %s is already trimmed and symmetric, nothing written\n",Prog_Name,argv[1]);
      hm_scan_destroy(S);
      hm_table_close(T);
      exit (0);
    }
  if (VERBOSE && !trim)
    fprintf(stderr,"\n  Trimming k-mers in table with count < %d\n",ETHRESH);
  if (VERBOSE && !symm)
    fprintf(stderr,trim ? "\n  Making table symmetric\n" : "\n  Making trimmed table symmetric\n");

  hm_condition_stats st;
  if (hm_scan_condition_files(S,ETHRESH,!trim,!symm,argv[2],&st) != HM_OK)
    die_hm();
  if (VERBOSE && st.gpus > 1)
    fprintf(stderr,"\n  Wrote %lld k-mers to %s (%d key ranges, %d passes over the source, %d GPUs)\n",
            (long long) st.nels_out,argv[2],st.ranges,st.passes,st.gpus);
  else if (VERBOSE)
    fprintf(stderr,"\n  Wrote %lld k-mers to %s (%d key ranges, %d passes over the source)\n",
            (long long) st.nels_out,argv[2],st.ranges,st.passes);

  hm_scan_destroy(S);
  hm_table_close(T);
  exit (0);
}

/* hm_internal.h -- shared by the translation units of libhetmers_b200.so (not installed) */
#ifndef HM_INTERNAL_H
#define HM_INTERNAL_H

#include <stdarg.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* record a message for hm_last_error() and return `code` */
int hm_set_error(int code, const char *fmt, ...);

#ifdef __cplusplus
}
#endif

#ifdef __CUDACC__
/* chunk-wise index construction for the loader (hm_kernels.cu) */
int hm_build_bucket_index_range(const uint64_t *d_keys, int64_t n, int bits, void *d_bucket,
                                int idx64, int64_t i0, int64_t i1, void *stream);
int hm_build_filter_range(const uint64_t *d_keys, int filter_bits, uint32_t *d_filter,
                          int64_t i0, int64_t i1, void *stream);

/* streamed symmetric scan (hm_symm.cu; driven by hm_scan.cu, DESIGN.md §4c): resident candidate records and
 * the S list (every key pass 1 puts into the Bloom filter), appended to by the chunks                        */
typedef struct hm_stream_lists
  { uint64_t *cand_key, *cand_lo, *cand_meta;
    int64_t   cand_cap;
    uint64_t *s_key, *s_lo;
    int64_t   s_cap;
    uint64_t *runs;                         /* heads of the current chunk's runs of three or more entries */
    int64_t   runs_cap;
  } hm_stream_lists;

/* several shards: the sorted S list of one shard and its bucket index, as the other shards' pass 2 reads it (peer
 * memory when the shard is on another GPU).  The shards' views form a device array of the reading shard.     */
typedef struct hm_stream_sview
  { const uint64_t *s_key, *s_lo;
    const void     *s_bucket;                /* uint32 or uint64 offsets: the same width for every shard */
    int64_t         n_s;
    int32_t         bits, pad;
  } hm_stream_sview;

/* shards: NULL (or n_seg == 1) for one shard; else this shard's descriptor -- n_seg = the shards up to the last
 * non-empty one, self, first_key -- over a work area of hm_symm_plan(n, 0, kmer, G) (G >= n_seg segments)   */
int hm_symm_stream_begin(void *d_work, const hm_symm_layout *L, void *stream);
int hm_symm_stream_chunk(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                         int64_t n, const void *d_bucket, int bits, int kmer, int64_t hi,
                         void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                         const hm_symm_shards *shards, void *stream);
int hm_symm_stream_counts(const void *d_work, const hm_symm_layout *L, uint64_t *n_cand,
                          uint64_t *status, uint64_t *n_s, void *stream);
int hm_symm_stream_reset_lists(void *d_work, const hm_symm_layout *L, void *stream);
/* one shard: the exact checks look up this shard's S list (d_s_key ...); several: the owner's, through
 * d_views[owner] (device array of shards->n_seg views)                                                 */
int hm_symm_stream_resolve(const uint64_t *d_s_key, const uint64_t *d_s_lo, int64_t n_s,
                           const void *d_s_bucket, int bits, int idx64, int kmer, int64_t range,
                           void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                           const hm_symm_shards *shards, const hm_stream_sview *d_views,
                           unsigned long long *d_plot, void *stream);

/* routed pass 2 of one rank of a one-process-per-GPU job (hm_rank_scan_*): over candidate slices [c0, c1) of at
 * most pend_cap candidates, resolve parks every candidate with a Bloom hit on a key another rank owns (pend, one
 * meta each) and lists those keys as queries (q_key / q_lo / q_tag = owner << 32 | pending slot, 2 per candidate
 * at most); route_group sorts them by owner into send (KW words per query) and send_slot; counts: device
 * uint64[2 * HM_MAX_SHARDS] scratch                                                                         */
typedef struct hm_route_bufs
  { uint64_t *pend;
    int64_t   pend_cap;
    uint64_t *q_key, *q_lo, *q_tag;
    int64_t   q_cap;
    uint64_t *send;
    uint32_t *send_slot;
    unsigned long long *counts;
    uint64_t *pend_key, *pend_lo;            /* the routed listing only: the parked candidates' key words      */
  } hm_route_bufs;

int hm_symm_route_resolve(const uint64_t *d_s_key, const uint64_t *d_s_lo, int64_t n_s,
                          const void *d_s_bucket, int bits, int idx64, int kmer, int64_t c0, int64_t c1,
                          void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                          const hm_symm_shards *shards, const hm_route_bufs *B, unsigned long long *d_plot, void *stream);
int hm_symm_route_group(int kmer, int world, void *d_work, const hm_symm_layout *L, const hm_route_bufs *B,
                        int64_t *counts, int64_t *n_sent, int64_t *n_pend, uint64_t *status, void *stream);
int hm_symm_route_answer(const uint64_t *d_s_key, const uint64_t *d_s_lo, const void *d_s_bucket, int bits,
                         int idx64, int kmer, const uint64_t *d_recv, int64_t n, uint8_t *d_ans, void *stream);
int hm_symm_route_settle(int kmer, const hm_route_bufs *B, const uint8_t *d_ans, int64_t n_sent, int64_t n_pend,
                         unsigned long long *d_plot, void *stream);
/* the routed listing of extract_kmer_pairs (hm_rank_scan_extract_*): route_extract lists the slice's settled
 * candidates into d_out (cap >= 2 per candidate; *d_count counts every record) and parks the rest with their
 * keys (pend_key / pend_lo); route_group as above; route_list lists the parked ones none of whose keys was found */
int hm_symm_route_extract(const uint64_t *d_s_key, const uint64_t *d_s_lo, int64_t n_s,
                          const void *d_s_bucket, int bits, int idx64, int kmer, int64_t c0, int64_t c1,
                          void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                          const hm_symm_shards *shards, const hm_route_bufs *B, const uint16_t *d_pixmap,
                          hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count, void *stream);
int hm_symm_route_list(int kmer, const hm_route_bufs *B, const uint8_t *d_ans, int64_t n_sent, int64_t n_pend,
                       const uint16_t *d_pixmap, hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count,
                       void *stream);

/* the pair files' sweeps over one GPU's share of the pairs (hm_scan_write_pairs, DESIGN.md §6c): the records that
 * hm_k_symm_extract (every candidate of the work area) or hm_k_pass2_extract ([lo, hi)) would list, none of them
 * stored in full.  d_hist != NULL: histogram sweep, d_hist[top hb bits of key_hi] += 1 per record (hb <= 32;
 * zeroed by the caller).  Else window sweep: the records with p0 <= prefix < p1 go to d_out, *d_count (zeroed by
 * the caller) counting all of them, also those beyond cap.                                                      */
int hm_symm_pairs_sweep(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt, int64_t n,
                        const void *d_bucket, int bits, int idx64, int kmer, void *d_work,
                        const hm_symm_layout *layout, const hm_symm_shards *shards, const uint16_t *d_pixmap,
                        int hb, unsigned long long *d_hist, uint64_t p0, uint64_t p1, hm_pair_rec *d_out,
                        int64_t cap, unsigned long long *d_count, void *stream);
int hm_pass2_pairs_sweep(const uint64_t *d_keys, const uint64_t *d_keys_lo, const uint16_t *d_cnt,
                         const uint8_t *d_deg, const void *d_up, int idx64, int64_t lo, int64_t hi,
                         const uint16_t *d_pixmap, int hb, unsigned long long *d_hist, uint64_t p0, uint64_t p1,
                         hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count, const hm_shards *shards,
                         void *stream);
/* device bytes of one pair-file window of `records` records: hm_pairs_bytes without its route term */
int64_t hm_pairs_window_bytes(int kmer, int64_t records);

#include <cuda_runtime.h>
int hm_cuda_fail(cudaError_t e, const char *what);
/* sort n packed keys (two words for k > 32) in place, in scratch of hm_sort_keys_bytes (hm_condition.cu) */
int64_t hm_sort_keys_bytes(int64_t n, int kmer);
int     hm_sort_keys(uint64_t *keys, uint64_t *lo, int64_t n, int kmer, void *scratch, int64_t scratch_bytes,
                     cudaStream_t st);
/* a stable radix sort of n one-word keys carrying uint32 values, in CUB scratch of hm_sort_perm_bytes (hm_condition.cu) */
int64_t hm_sort_perm_bytes(int64_t n);
int     hm_sort_perm(const uint64_t *k_in, uint64_t *k_out, const uint32_t *v_in, uint32_t *v_out, int64_t n,
                     void *tmp, int64_t tmp_bytes, cudaStream_t st);
/* lists in host memory (DESIGN.md §4c): a slice of n candidates (R's cand arrays, R->cand_cap >= n) swept by
 * resolve_kernel<..., LK_PARK> into B's pending list and queries (reset: the slice opens a round); the round's
 * counts (synchronises); its queries sorted by key into B->send, their slots into perm_a or perm_b (B->send_slot
 * is set to it; at k > 32 B->send has 2 q_cap words); then hm_symm_route_answer per S partition and
 * hm_symm_route_settle                                                                                      */
int hm_symm_park_resolve(int kmer, int64_t n, int reset, void *d_work, const hm_symm_layout *L,
                         const hm_stream_lists *R, const hm_symm_shards *shards, const hm_route_bufs *B,
                         unsigned long long *d_plot, void *stream);
int hm_symm_park_counts(const void *d_work, const hm_symm_layout *L, int64_t *n_pend, int64_t *n_q, uint64_t *status,
                        void *stream);
int hm_symm_park_sort(int kmer, hm_route_bufs *B, int64_t n_q, uint32_t *perm_a, uint32_t *perm_b,
                      void *tmp, int64_t tmp_bytes, void *stream);
/* a rank's lists in host memory (hm_rank_scan_*): hm_symm_park_resolve or hm_symm_park_extract sweep a slice (the
 * queries tagged with their owners, this rank included); the keys the rank receives sorted by key
 * (hm_symm_recv_sort: *perm = each sorted key's receive index), answered per S partition with
 * hm_symm_route_answer, and the answers put back in receive order (hm_symm_recv_unsort)                    */
int hm_symm_park_extract(int kmer, int64_t n, void *d_work, const hm_symm_layout *L, const hm_stream_lists *R,
                         const hm_symm_shards *shards, const hm_route_bufs *B, const uint16_t *d_pixmap,
                         hm_pair_rec *d_out, int64_t cap, unsigned long long *d_count, void *stream);
int hm_symm_recv_sort(int kmer, const uint64_t *recv, int64_t n, uint64_t *sorted, uint32_t *perm_a, uint32_t *perm_b,
                      void *tmp, int64_t tmp_bytes, uint32_t **perm, void *stream);
int hm_symm_recv_unsort(const uint8_t *d_ans_sorted, const uint32_t *d_perm, int64_t n, uint8_t *d_ans, void *stream);
/* conditioning, a key range at a time (hm_condition.cu; driven by hm_scan_condition and hm_scan_condition_files
 * in hm_scan.cu and by hm_k_shard_settle): the device buffers of one range of at most `cap` output entries.
 * key / lo / cnt: the region the kept originals fill from the front and the reverse complements from the back;
 * alt_*, idx: sort buffers; m_*: where the settled range goes (NULL when only trimming: the region is the
 * range); rec: its records; bcount: stub-bucket counts; ctr: [0] originals, [1] reverse complements, [3]
 * overflow, [4..5] merge scratch                                                                             */
typedef struct hm_cond_bufs
  { int       kmer, ibyte, hb, ethresh, do_symm;
    int64_t   cap;
    uint64_t *key, *lo, *alt_key, *alt_lo, *m_key, *m_lo;
    uint16_t *cnt, *alt_cnt, *m_cnt;
    uint32_t *idx[2];
    uint8_t  *rec;
    unsigned long long *mtiles, *ctr, *bcount;
    void     *sort_tmp;
    int64_t   sort_bytes;
  } hm_cond_bufs;

/* pass 0: hist[prefix] += kept originals (+ their reverse complements) of a chunk of m source entries */
int hm_cond_hist(const uint64_t *keys, const uint64_t *klo, const uint16_t *cnt, int64_t m, int kmer, int ethresh,
                 int do_symm, int hb, unsigned long long *hist, cudaStream_t st);
/* a chunk's share of the range [p0, p1) of key prefixes into B's region (tiles: hm_cond_tiles_bytes(m)) */
int hm_cond_gather(const uint64_t *keys, const uint64_t *klo, const uint16_t *cnt, int64_t m, const hm_cond_bufs *B,
                   uint64_t p0, uint64_t p1, unsigned long long *tiles, cudaStream_t st);
/* the range gathered in B settled: when symmetrising, its reverse complements sorted and merged with its
 * originals into B->m_* (the originals copied there when it has no reverse complements); *n_out: its entries,
 * in B->m_*, or in the region when B->m_key is NULL.  Synchronises st.                                    */
int hm_cond_settle(const hm_cond_bufs *B, int64_t *n_out, cudaStream_t st);
/* the settled range's n entries -> FastK records in B->rec and the counts of stub buckets [b0, b0+nb) in
 * B->bcount.  Synchronises st.                                                                            */
int hm_cond_pack(const hm_cond_bufs *B, int64_t n, uint64_t b0, int64_t nb, cudaStream_t st);
/* tile counts -> exclusive offsets (+ *base; *base += total) */
int hm_cond_scan_tiles(unsigned long long *tiles, int64_t nt, unsigned long long *base, cudaStream_t st);
int64_t hm_cond_chunk(int64_t n, int kmer, int ibyte, int64_t budget);
int64_t hm_cond_tiles_bytes(int64_t n);
int64_t hm_cond_sort_room(int64_t c);
/* the plan's two halves shared by the drivers: the most output entries one range may hold when a range of t
 * needs bytes(t, do_symm, kmer, ibyte) <= room (bisection), and the greedy cuts of np key prefixes into
 * ranges of at most `limit` entries (cuts[0..R], R returned; *range_cap: the largest range; *big: the largest
 * prefix -- 0 ranges when it alone exceeds the limit)                                                     */
typedef int64_t (*hm_cond_bytes_fn)(int64_t t, int do_symm, int kmer, int ibyte);
int64_t hm_cond_range_limit(int64_t room, hm_cond_bytes_fn bytes, int do_symm, int kmer, int ibyte);
int     hm_cond_cut(const int64_t *hist, int64_t np, int64_t limit, int64_t *cuts, int64_t *range_cap, int64_t *big);
#define HM_CUDA(call)                                             \
  do { cudaError_t _e = (call);                                    \
       if (_e != cudaSuccess) return hm_cuda_fail(_e,#call);       \
     } while (0)
#endif

#endif

/* herro_b200.h — C ABI of the H100-native HERRO hot path (features -> inference -> consensus).
 *
 * The reference (lbcb-sci/herro @ 9cd0296) has no FFI layer: the three stages are Rust
 * worker threads joined by crossbeam channels.  This header is what a `mod ffi` in the Rust
 * host binds so that `herro inference` keeps its CLI, FASTQ loading, `--read-alns` batches,
 * windowing and FASTA writer (src/main.rs, src/lib.rs, src/haec_io.rs, src/overlaps.rs,
 * src/windowing.rs) and replaces
 *
 *   features::extract_features      src/features.rs:326-583   (called at src/lib.rs:176-183)
 *   inference::inference_worker     src/inference.rs:177-212  (spawned at src/lib.rs:189-196)
 *   consensus::consensus_worker     src/consensus.rs:229-263  (spawned at src/lib.rs:198-199)
 *
 * (all three at once through hb_submit_*; each also alone: hb_features_batch, hb_forward_batch, hb_consensus_batch)
 * with calls into this library (INTEGRATION.md shows the Rust side).  Plain pointers and
 * sizes only; no torch types; never unwinds or aborts (the reference is `panic = "abort"`,
 * Cargo.toml:14-16): every entry point returns HB_OK or a negative hb_status, and
 * hb_last_error() gives the message.
 *
 * Threading: hb_submit_* may be called concurrently from the host's feature threads
 * (`-t`, src/lib.rs:159-187); hb_poll_corrected / hb_release_result from one thread per
 * context (the former consensus thread feeding correction_writer, src/lib.rs:267-291).
 * One context per GPU (`-d`), like the reference's per-device worker group.  Every call
 * returns with the calling thread's current CUDA device as it found it, unless that device
 * had no primary context yet: making it current again would create one.
 */
#ifndef HERRO_B200_H
#define HERRO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define HB_ABI_VERSION 1

typedef enum hb_status {
    HB_OK = 0,
    HB_ERR_ARG = -1,      /* bad argument / NULL pointer / out-of-range id                      */
    HB_ERR_CUDA = -2,     /* CUDA runtime failure (no device, OOM, launch error)                */
    HB_ERR_MODEL = -3,    /* weights file missing / malformed / unsupported dimensions          */
    HB_ERR_INPUT = -4,    /* input on which the reference itself would panic (bad CIGAR, ...)   */
    HB_ERR_CAPACITY = -5, /* an internal capacity was exceeded and could not be grown (e.g. more   */
                          /* than 60000 overlaps covering one window, out of memory)            */
    HB_ERR_STATE = -6     /* call sequence error (e.g. submit before hb_upload_reads)           */
} hb_status;

/* Overlap + CIGAR of one alignment — `struct Overlap` / `struct Alignment`
 * (src/overlaps.rs:44-55,91-95).  strand: 0 = '+', 1 = '-'.  cigar: ASCII `[0-9]+[MID]`
 * exactly as parsed from the PAF `cg:Z:` field (src/overlaps.rs:172); caller-owned, copied
 * before the call returns. */
typedef struct hb_overlap {
    uint32_t qid, qlen, qstart, qend;
    uint32_t strand;
    uint32_t tid, tlen, tstart, tend;
    const uint8_t* cigar;
    uint32_t cigar_len;
} hb_overlap;

/* One OverlapWindow (src/windowing.rs:6-16) plus the window it was pushed to
 * (`windows[i].push(...)`, src/windowing.rs:161,233,262).  cigar_*_idx are BYTE offsets into
 * the overlap's CIGAR, cigar_*_offset are base counts from the start of that op
 * (SURVEY.md App. G). */
typedef struct hb_overlap_window {
    uint32_t overlap_idx; /* index into the `ovl` array of the same hb_submit_target call */
    uint32_t window_idx;  /* 0 .. n_windows-1                                             */
    uint32_t tstart, qstart, qend;
    uint32_t cigar_start_idx, cigar_start_offset, cigar_end_idx, cigar_end_offset;
} hb_overlap_window;

typedef struct hb_options {
    uint32_t struct_size;    /* = sizeof(hb_options)                                                     */
    uint32_t window_size;    /* `-w` (src/main.rs:69-74), default 4096                                    */
    uint32_t batch_size;     /* `-b` (src/main.rs:98-102): the reference groups consecutive windows of a  */
                             /* read in chunks of b and pads each chunk to its longest window             */
                             /* (src/features.rs:884-893, src/inference.rs:73-97); that padding is part   */
                             /* of the model input, so it is reproduced per window (DESIGN.md, H10)       */
    uint32_t launch_targets; /* target reads per device launch (cross-read batching); 0 = default         */
    uint32_t flags;          /* HB_FLAG_*                                                                */
} hb_options;

#define HB_FLAG_KEEP_DEBUG 1u /* keep per-window intermediates of the last launch for hb_debug_*        */
#define HB_FLAG_NO_MODEL   2u /* load no weights (model_path may be NULL): hb_features_batch and hb_consensus_batch only;   */
                              /* hb_submit_*, hb_flush and hb_forward_batch return HB_ERR_STATE                          */

typedef struct hb_ctx hb_ctx; /* one per GPU: streams, weights, read-store replica, staging buffers */

/* Create a context on `cuda_device` and load the forward weights (replaces tch::CModule::load_on_device,
 * src/inference.rs:185).  `model_path` is what `-m` names: a TorchScript archive (`torch.jit.save`; ZIP with stored
 * entries + data.pkl, read natively, no libtorch) of a module with the architecture this library implements
 * (oracle/forward_ref.py naming; an optional `stem_bn` is folded), or the HB200W1 blob of herro_b200/weights.py.
 * Any other graph is HB_ERR_MODEL with the first missing parameter named: TorchScript code is not executed.
 * With HB_FLAG_NO_MODEL in opt->flags no weights are loaded and model_path may be NULL (it is ignored): such a context runs
 * the features stage and consensus around a model the host executes itself (hb_features_batch, hb_consensus_batch). */
int hb_create(hb_ctx** out, int cuda_device, const char* model_path, const hb_options* opt);
void hb_destroy(hb_ctx* ctx);

/* Architecture of a model file without creating a context (host only, no CUDA call): dims = stem_k, channels, heads,
 * layers, ffn, collapse; *params_hash (may be NULL) = FNV-1a-64 over the canonical fp32 tensors in name order, equal for
 * a blob and an archive holding the same weights.  `err` (may be NULL) receives the message on failure. */
int hb_inspect_model(const char* model_path, uint32_t dims[6], uint64_t* params_hash, char* err, size_t err_cap);
/* Same, with dims = stem_k, channels, heads, layers, ffn, collapse, pos_layers, pos_heads, pos_ffn: the last three describe
 * the optional encoder stage across each window's supported positions (all 0 without one). */
int hb_inspect_model_ex(const char* model_path, uint32_t dims[9], uint64_t* params_hash, char* err, size_t err_cap);

/* Replicate the read store on the GPU.  Layout is HAECRecord verbatim (src/haec_io.rs:19-24,
 * 77-81): seq_words[i] = 2-bit little-endian packing, 32 bases per u64, A0 C1 G2 T3
 * (src/haec_io.rs:121-136); seq_len[i] bases; qual[i] = raw Phred+33 bytes (seq_len[i] of them).
 * Read ids are positions in this array (`rid`), as in the reference (src/overlaps.rs:332-336). */
int hb_upload_reads(hb_ctx* ctx, uint32_t n_reads, const uint64_t* const* seq_words, const uint32_t* seq_len,
                    const uint8_t* const* qual);

/* ---- the read store in host memory ------------------------------------------------------ */
/* For read sets larger than the GPU's memory (a 50x human set is ~200 GB packed): the reads stay in host RAM, as the reference keeps
 * them (src/lib.rs:241-265), and every launch copies only its own reads to the device.
 *
 * hb_read_store_create takes hb_upload_reads' arguments and layout rules and copies the reads into ONE page-locked, portable,
 * device-mapped host allocation (each read's words and qualities 16-byte aligned) that contexts on any GPU of the process share.
 * It needs no context and does no GPU work; errors (HB_ERR_ARG for a NULL pointer, zero reads or a NULL read, checked before any
 * CUDA call; HB_ERR_CAPACITY / HB_ERR_CUDA when the allocation fails) are reported through hb_last_error(NULL).  The caller's arrays
 * may be freed once it returns: peak host memory is briefly twice the store.
 *
 * hb_attach_read_store replaces hb_upload_reads for one context: it frees a store uploaded earlier and uploads only len[]
 * (4 * n_reads bytes) and the ln table (8 * (max_len + 2) bytes), which is all it adds to h2d_bytes.  Same preconditions as
 * hb_upload_reads (HB_ERR_STATE with targets pending; not beside hb_features_batch).  A later hb_upload_reads or
 * hb_attach_read_store detaches again; the launch hb_replay_last_launch would re-run is dropped by either.
 *
 * Lifetime: the store counts the contexts attached to it.  hb_read_store_destroy returns HB_ERR_STATE while any is (the store is
 * then left intact and usable); hb_destroy detaches.  The store must outlive every context attached to it.
 * Threading: any number of contexts, on any devices, may share one store and run at the same time; the store is read-only.
 *
 * What a launch (hb_submit_*, hb_features_batch) reads over PCIe: its distinct reads (targets and every query of its alignments),
 * each read's words and qualities rounded up to 16 bytes, plus a read list of 40 bytes per read.  A kernel (k_reads_in) gathers
 * them from the mapped store into the launch's scratch, so HBM use is set by the launch size (hb_set_launch_targets bounds it),
 * not by the read set.  Scratch that cannot grow fails the launch's targets with HB_ERR_CAPACITY, as other scratch does.
 * hb_replay_last_launch re-runs the gather too, so its time includes PCIe reads in this mode.
 *
 * Counters: h2d_bytes grows by the gathered bytes and the read list; the gather kernel counts under HB_K_LISTS and inside
 * ms_features; building the read list is part of ms_worker_phase[0].
 * Results: every output is identical to that of an uploaded store holding the same reads. */
typedef struct hb_read_store hb_read_store;
int hb_read_store_create(hb_read_store** out, uint32_t n_reads, const uint64_t* const* seq_words, const uint32_t* seq_len,
                         const uint8_t* const* qual);
int hb_read_store_destroy(hb_read_store* store);
int hb_attach_read_store(hb_ctx* ctx, hb_read_store* store);

/* Submit one target read: the replacement of extract_features(rid, reads, overlaps, ...)
 * (src/features.rs:326-333) for a host that still runs windowing::extract_windows itself.
 * n_windows = ceil(len/W) (src/features.rs:338).  `ow` lists the OverlapWindows in the order
 * extract_windows pushed them (alignment order), each tagged with its window.  Every
 * overlap must have tid == rid (src/overlaps.rs:189-192).  Results become available through
 * hb_poll_corrected after enough targets were submitted or after hb_flush. */
int hb_submit_target(hb_ctx* ctx, uint32_t rid, uint32_t n_windows, const hb_overlap* ovl, uint32_t n_ovl,
                     const hb_overlap_window* ow, uint32_t n_ow);

/* Same, but the library also performs windowing::extract_windows (src/windowing.rs:44-273)
 * on the raw alignments — for hosts that hand over `(tid, Vec<Alignment>)` straight from
 * alignment_reader (src/overlaps.rs:371-373).  The windowing runs ON THE DEVICE (SURVEY.md §8f-1): the calling
 * thread only derives, from the PAF coordinates, which windows each alignment contributes to, and copies the CIGARs;
 * no CIGAR byte is parsed on the host.  Consequently a malformed CIGAR (or one that does not span its PAF
 * coordinates) is reported for its target by hb_poll_corrected (HB_ERR_INPUT), not by this call; coordinate errors
 * (inverted ranges, windows past the end of the target) still fail here. */
int hb_submit_alignments(hb_ctx* ctx, uint32_t rid, const hb_overlap* ovl, uint32_t n_ovl);

/* ---- the features stage alone ------------------------------------------------------------ */
#define HB_FEAT_DEVICE_PTRS 1u /* hb_features_fetch: bases, quals, batch_bases and batch_quals are device pointers on the context's device */

typedef struct hb_features_shape {  /* what one hb_features_batch produced                                                   */
    uint64_t ticket;                /* names the result for hb_features_fetch                                                */
    uint32_t n_targets, n_windows, n_batches, n_failed;
    uint64_t n_rows, n_sup, n_ids;  /* N = sum rows, S = sum n_sup, sum n_ids                                                */
    uint64_t n_batch_rows;          /* sum over the reference batches of B * Lmax                                            */
} hb_features_shape;

typedef struct hb_features_out {    /* = sizeof(hb_features_out); any other pointer may be NULL: that output is not written  */
    uint32_t struct_size;
    int32_t*  status;      /* [n_targets] host: HB_OK, HB_ERR_INPUT or HB_ERR_CAPACITY                                       */
    uint32_t* n_windows;   /* [n_targets] host: ceil(len / W), n_total_wins                                                  */
    uint32_t* rows;        /* [n_windows] host: L' of each window; 0 for the windows of a failed target                      */
    uint8_t*  n_alns;      /* [n_windows] host: min(n_ids, 30)                                                               */
    uint32_t* n_sup;       /* [n_windows] host: supported positions                                                          */
    uint32_t* n_ids;       /* [n_windows] host: overlaps that survived the filter                                            */
    uint8_t*  bases;       /* [N][31] BASES_MAP tokens, window after window      (host; device with HB_FEAT_DEVICE_PTRS)     */
    uint8_t*  quals;       /* [N][31] raw quality bytes                          (host; device with HB_FEAT_DEVICE_PTRS)     */
    uint32_t* supported;   /* [S][2] host: (pos, ins), window after window                                                   */
    int32_t*  indices;     /* [S] host: the row of each supported entry inside its window (collate's indices)                */
    uint32_t* ids;         /* [sum n_ids] host: query read id of every surviving overlap, in final rank order, window after window */
    uint32_t* batch_B;     /* [n_batches] host: windows in each reference batch                                              */
    uint32_t* batch_Lmax;  /* [n_batches] host: its longest window                                                           */
    uint32_t* batch_win;   /* [sum batch_B] host: the window (index into the window order above) of each batch slot          */
    uint8_t*  batch_bases; /* [n_batch_rows][31] tokens, padded with 11          (host; device with HB_FEAT_DEVICE_PTRS)     */
    uint8_t*  batch_quals; /* [n_batch_rows][31] quality bytes, padded with 126  (host; device with HB_FEAT_DEVICE_PTRS)     */
} hb_features_out;

/* The replacement of extract_features (src/features.rs:326-583) on many targets at once, for a host that keeps its own model call
 * (and perhaps its own consensus): what the reference's feature threads compute, without the model call and consensus that
 * hb_submit_* chain onto it.  The input is hb_submit_alignments' for n_targets targets: target i is rids[i] with the n_ovl[i]
 * alignments that follow those of target i-1 in `ovl` (every tid == rid), windowed on the device as hb_submit_alignments does.
 * hb_features_batch computes and fills *shape with the sizes of every output; hb_features_fetch then copies out any subset of
 * them, as often as wanted (for example the metadata first, then the bulk arrays into buffers of the sizes it gave).
 *
 * The windows: every target has all of its ceil(len / W) windows, in wid order, also those without alignments; targets in the
 * order given.  Per window, exactly the arguments of FeaturesOutput::update (src/features.rs:570-578): the [L', 31] tokens and
 * qualities, the (pos, ins) SupportedPos list with the row each entry names (collate's indices), and the ids.
 * The reference batches: each target's windows are taken `-b` (hb_options.batch_size) at a time in wid order, as
 * FeaturesOutput::update hands them to InferenceOutput::update; the windows of a group with at least one supported position form one
 * batch (prepare_examples), padded to its longest window with token 11 and quality 126 (collate, src/inference.rs:73-140,214-250).
 * batch_bases / batch_quals are those [B, Lmax, 31] tensors back to back, batch_win says which window each slot holds, and the
 * indices of slot k are those of window batch_win[k]: the arguments of hb_forward_batch, whose output in turn orders the logits the
 * way hb_consensus_batch takes them.
 *
 * Per-target failures (the call still returns HB_OK; hb_last_error names the first failed target): a malformed CIGAR or coordinates
 * the reference would panic on are HB_ERR_INPUT, more than 60000 overlap-windows covering one window HB_ERR_CAPACITY.  A failed
 * target keeps its n_windows, and its windows have no rows, positions or ids; it has no batches.  The other targets are unaffected.
 *
 * Errors of the call (the previous result is gone; nothing is written; the context stays usable):
 *   HB_ERR_ARG       a NULL pointer, a rid out of range, an alignment with tid != rid, a qid out of range or a strand other than 0 / 1;
 *                    for fetch also a struct_size mismatch, unknown flags, or a pointer that does not match the flag (bulk outputs
 *                    must be device memory of the context's device with HB_FEAT_DEVICE_PTRS and host memory without; the others
 *                    host memory always)
 *   HB_ERR_STATE     no hb_upload_reads yet; for fetch, a shape whose ticket is not the context's latest result
 *   HB_ERR_CAPACITY  a batch too large (2^32 CIGAR op slots, as a launch), or scratch that could not grow
 *   HB_ERR_CUDA      a CUDA failure
 *
 * Synchronous: both calls return when their work is done.  With HB_FEAT_DEVICE_PTRS the library's stream first waits, through an
 * event, for the work already enqueued on `stream` (NULL: the legacy default stream), so a caller can hand over freshly allocated
 * tensors.  Scratch only grows, so repeated calls of the same or a smaller shape allocate nothing.  Host-bound bulk outputs are copied
 * straight into the caller's memory.  A result stays valid until the next hb_features_batch on the context.
 *
 * Threading: calls of hb_features_batch / hb_features_fetch on one context serialise among themselves on a lane of their own; they may
 * run beside hb_submit_*, hb_flush, hb_poll_corrected, hb_forward_batch and hb_consensus_batch (not beside hb_upload_reads), and never
 * touch the pipeline's scratch, the debug taps or the launch hb_replay_last_launch re-runs.
 *
 * Counters: adds to kernel_launches, n_kernel / ms_kernel (the output kernels under HB_K_LISTS), ms_features, h2d_bytes, d2h_bytes
 * and host_allocs when scratch grows; targets, windows, rows, supported and corrected_bases are untouched. */
int hb_features_batch(hb_ctx* ctx, uint32_t n_targets, const uint32_t* rids, const uint32_t* n_ovl, const hb_overlap* ovl,
                      hb_features_shape* shape);
int hb_features_fetch(hb_ctx* ctx, const hb_features_shape* shape, const hb_features_out* out, uint32_t flags, void* stream);

/* ---- the base-level alignment of overlaps ------------------------------------------------- */
#define HB_ALN_BAND_EDGE 1  /* hb_align_fetch status: aligned, but the path touched the band's edge (it may have left the band) */

typedef struct hb_align_shape {     /* what one hb_align_overlaps produced                                                    */
    uint64_t ticket;                /* names the result for hb_align_fetch                                                   */
    uint32_t n_overlaps, n_failed, n_band_edge;
    uint64_t cigar_bytes, cells;    /* total CIGAR text; DP cells computed, sum over aligned overlaps of (n + 1) * 2w         */
    double ms_device;               /* device time of the alignment kernels                                                  */
} hb_align_shape;

/* The alignment `minimap2 -c` adds to an overlap-only PAF line, done on the device: per overlap (its cigar is ignored and may be
 * NULL), a banded two-piece affine alignment of the target slice t[tstart, tend) against the query slice q[qstart, qend),
 * reverse-complemented on strand 1, with minimap2's default scores (match 2, mismatch 4, gap min(4 + 2l, 24 + l)).  Row i of
 * the n + 1 target rows holds the 2w columns c(i) - w <= j < c(i) + w (c(i) = floor(i m / n)) that lie in 0..m.  The traceback
 * from (n, m) goes through the reference's fix_cigar (src/aligners.rs:138-250: indels flanked by matches left-aligned, a leading
 * gap dropped, equal ops merged), then gaps left at either end are dropped too: the coordinates move inwards by the dropped
 * lengths and the CIGAR, which starts and ends with M, spans them exactly.  DESIGN.md §12 gives the definition in full.
 * hb_align_overlaps computes and fills *shape; hb_align_fetch copies out any subset of the results, as often as wanted:
 *   out         [n] the input overlaps in input order with the new coordinates; cigar points into cigar_text (cigar_len bytes),
 *               ready for hb_submit_alignments or hb_features_batch.  A failed overlap keeps its coordinates and has no CIGAR.
 *   cigar_text  [shape->cigar_bytes] every CIGAR, back to back
 *   status      [n] HB_OK, HB_ALN_BAND_EDGE, HB_ERR_INPUT (a coordinate outside its read, an empty span, or one span more than
 *               twice the other) or HB_ERR_CAPACITY (its traceback alone exceeds the 8 GiB wave region)
 *   matches     [n] identical base pairs inside M (PAF column 10); column 11 is the sum of the CIGAR's op lengths
 * band_w: w, a multiple of 16 up to 256; 0 takes the default, 128.  Failed overlaps fail alone (the call returns HB_OK and
 * hb_last_error names the first).
 *
 * Errors of the call (the previous result is gone):
 *   HB_ERR_ARG       a NULL pointer, a qid or tid out of range, a strand other than 0 / 1, or a bad band_w
 *   HB_ERR_STATE     no reads yet (hb_upload_reads / hb_attach_read_store); for fetch, a shape whose ticket is not the latest result
 *   HB_ERR_CUDA      a CUDA failure
 *
 * Synchronous: both calls return when their work is done.  The overlaps run in waves whose traceback (one byte per cell) and
 * op slots fit a grow-only region, longest overlaps first.  A wave takes at most 8 GiB and at most half of the device memory
 * that is free when the call starts (the region's own bytes count as free); the region stays allocated until the context is
 * destroyed.  With a host read store the call's reads are
 * gathered once, as a launch gathers its own.  Works on an HB_FLAG_NO_MODEL context.
 *
 * Threading: calls of hb_align_overlaps / hb_align_fetch on one context serialise among themselves on a lane of their own; they may
 * run beside hb_submit_*, hb_flush, hb_poll_corrected and the other single-stage calls (not beside hb_upload_reads).
 *
 * Counters: adds to kernel_launches, h2d_bytes, d2h_bytes and host_allocs when scratch grows; the kernel time and the cells are in
 * the shape. */
int hb_align_overlaps(hb_ctx* ctx, uint32_t n, const hb_overlap* ovl, uint32_t band_w, hb_align_shape* shape);
int hb_align_fetch(hb_ctx* ctx, const hb_align_shape* shape, hb_overlap* out, uint8_t* cigar_text, int32_t* status, uint32_t* matches);

/* ---- all-vs-all read overlaps ----------------------------------------------------------------- */
typedef struct hb_ovl_params {  /* 0 in any field takes its default                                                             */
    uint32_t k;                 /* k-mer length, 12..28 (25)                                                                  */
    uint32_t w;                 /* minimizer window, 2..32 k-mers (17)                                                        */
    uint32_t min_score;         /* a chain's least score (2500)                                                               */
    uint32_t min_anchors;       /* a chain's least number of anchors (3)                                                      */
    uint32_t max_gap;           /* the largest gap between chained anchors, on either read (5000)                             */
    uint32_t bandwidth;         /* the largest |dx - dy| between chained anchors (150)                                        */
    uint32_t max_iter;          /* predecessors tried per anchor (5000)                                                       */
    uint32_t top_frac_ppm;      /* the share of distinct index hashes, in parts per million, above the occurrence threshold (5000) */
    uint32_t min_occ;           /* the occurrence threshold's floor (10)                                                      */
} hb_ovl_params;

typedef struct hb_ovl_shape {   /* what one hb_find_overlaps produced                                                         */
    uint64_t ticket;            /* names the result for hb_find_fetch                                                         */
    uint32_t n_targets, n_overlaps, max_occ, n_filtered_hashes;
    uint64_t index_entries, query_minimizers, anchors, chained_groups;
    double ms_device;           /* device time of the call's kernels and sorts                                               */
} hb_ovl_shape;

/* The overlaps `minimap2 -x ava-ont` finds between reads, by the definition of DESIGN.md §13 (minimizer sketch, an occurrence
 * filter on the targets' index, anchors, a chaining dynamic program): each read of the store (the queries) against the n_targets
 * reads target_rids (the call's targets, distinct).  At most one record per (target, query) pair, query != target: the better of
 * its two strands.  hb_find_fetch copies out any subset, as often as wanted, in call-target order and then ascending qid:
 *   out        [n_overlaps] hb_overlap without a CIGAR (cigar NULL, cigar_len 0), ready for hb_align_overlaps
 *   score      [n_overlaps] the chain's score
 *   n_anchors  [n_overlaps] the chain's anchors
 *   covered    [n_overlaps] target bases covered by the chain's k-mers (PAF column 10)
 *
 * Errors of the call (the previous result is gone; nothing runs):
 *   HB_ERR_ARG       a NULL pointer, n_targets == 0, or a parameter out of range
 *   HB_ERR_INPUT     a target rid out of range or repeated
 *   HB_ERR_STATE     no reads yet (hb_upload_reads / hb_attach_read_store); for fetch, a shape whose ticket is not the latest result
 *   HB_ERR_CAPACITY  a region cannot grow (the index, or the anchors of one query read)
 *   HB_ERR_CUDA      a CUDA failure
 *
 * Synchronous.  The queries run in chunks of reads in rid order; a chunk's anchors take at most half of the device memory that is
 * free when the call starts (the regions' own bytes count as free), and the regions stay allocated until the context is destroyed.
 * With a host read store the targets and each chunk are gathered as a launch gathers its reads.  Works on an HB_FLAG_NO_MODEL
 * context.  Calls of hb_find_overlaps / hb_find_fetch serialise among themselves on a lane of their own; they may run beside
 * hb_submit_*, hb_flush, hb_poll_corrected and the other single-stage calls (not beside hb_upload_reads).
 *
 * Counters: adds to kernel_launches, h2d_bytes, d2h_bytes and host_allocs when scratch grows; the rest is in the shape. */
int hb_find_overlaps(hb_ctx* ctx, uint32_t n_targets, const uint32_t* target_rids, const hb_ovl_params* params, hb_ovl_shape* shape);
int hb_find_fetch(hb_ctx* ctx, const hb_ovl_shape* shape, hb_overlap* out, uint32_t* score, uint32_t* n_anchors, uint32_t* covered);

/* ---- the model call alone ---------------------------------------------------------------- */
#define HB_FWD_DEVICE_PTRS 1u  /* bases, quals and both outputs are device pointers on the context's device */
/* The replacement of inference() (src/inference.rs:147-175) on one collated batch, for a host that keeps its own features stage,
 * batching and consensus.
 *
 *   bases, quals   [B][Lmax][31] u8, C order: BASES_MAP tokens (src/inference.rs:23-31) / raw quality bytes
 *   lens           [B] i32, host memory: supported positions of each window
 *   indices        [sum lens] i32, host memory: the rows of window b's positions, window after window
 *   info_logits    [sum lens] f32, bases_logits [sum lens][5] f32: in `indices` order
 *   stream         with HB_FWD_DEVICE_PTRS: the cudaStream_t whose pending work produces the inputs (NULL: the legacy default stream)
 *
 * What it computes: the model's graph over the whole tensor, as collate + forward_is do.  Rows [0, Lmax) are taken as given,
 * wherever token 11 (the batch padding) appears; rows outside [0, Lmax) contribute nothing (the conv's zero padding).  The
 * qualities are normalised on the device as inference() does, fl(fl(q * fl(2/93)) - fl(66/93 + 1)), for any byte 0-255.  A model
 * with the encoder stage across positions attends within each of the B windows.  Nothing of consensus runs.
 *
 * Synchronous: returns when the outputs are written.  With HB_FWD_DEVICE_PTRS the library's stream first waits, through an event,
 * for the work already enqueued on `stream`; host inputs and outputs go through pinned staging that only grows, so repeated
 * calls of the same or smaller shape allocate nothing.
 *
 * Errors (the context stays usable for the pipeline and the next call; nothing is written to the outputs):
 *   HB_ERR_ARG       a NULL pointer, B == 0 or Lmax == 0, a negative length, an index outside [0, Lmax), or a pointer that does
 *                    not match the flag (with it: host memory or another device's memory; without it: device memory)
 *   HB_ERR_INPUT     a token above 11 (the reference's Embedding would raise); the message names the first offending (b, row, col)
 *                    in row-major order
 *   HB_ERR_CAPACITY  scratch could not grow
 *   HB_ERR_CUDA      a CUDA failure
 * sum lens == 0 is HB_OK and writes nothing.  Duplicated and unsorted indices are fine.
 *
 * Threading: may be called from any thread, concurrently with hb_submit_*, hb_flush and hb_poll_corrected on the same context;
 * calls of hb_forward_batch on one context serialise among themselves.  It needs no hb_upload_reads, and never touches the
 * pipeline's scratch, the debug taps or the launch hb_replay_last_launch re-runs.
 *
 * Counters: adds to kernel_launches, n_kernel / ms_kernel (the input kernel under HB_K_LISTS), ms_forward, supported, the FLOP
 * counters (per position, as the pipeline counts them) and host_allocs when scratch grows; targets, windows, rows and
 * corrected_bases are untouched. */
int hb_forward_batch(hb_ctx* ctx, uint32_t B, uint32_t Lmax, const uint8_t* bases, const uint8_t* quals, const int32_t* lens,
                     const int32_t* indices, float* info_logits, float* bases_logits, uint32_t flags, void* stream);

/* ---- consensus alone --------------------------------------------------------------------- */
#define HB_CONS_DEVICE_PTRS 1u /* bases and bases_logits are device pointers on the context's device */
/* The replacement of consensus() (src/consensus.rs:86-227) on the windows of n_reads reads, for a host that keeps its own features
 * stage and model call: what consensus_worker does once a read's windows are complete and sorted by wid (src/consensus.rs:246-253).
 * With W = sum n_windows, N = sum rows and S = sum n_sup:
 *
 *   n_windows     [n_reads] host: every window of each read (n_total_wins), 0 allowed
 *   rows          [W] host: L' of each window (the rows of ConsensusWindow.bases), 0 allowed
 *   n_alns        [W] host: at most 30
 *   bases         [N][31] u8: BASES_MAP tokens (src/inference.rs:23-31), window after window, at any alignment
 *   n_sup         [W] host: supported positions of each window
 *   supported     [S][2] u32 host: (pos, ins) of each supported position (pos <= 65535, ins <= 255), window after window
 *   bases_logits  [S][5] f32: one row per supported entry, in the same order (hb_forward_batch returns them so); info logits are
 *                 not taken, consensus never reads them
 *   seqs          host, room for N bytes: the segments, read after read, as ASCII ACGT
 *   seg_len       host, room for W entries: the segment lengths, read after read
 *   n_segs        [n_reads] host: segments of each read; 0 = no record (consensus() returned None or nothing), as hb_poll_corrected
 *   stream        with HB_CONS_DEVICE_PTRS: the cudaStream_t whose pending work produces bases / bases_logits (NULL: legacy default)
 *
 * What it computes, with the reference's rules where they depart from the obvious:
 *   - Only the windows from a read's first to its last with n_alns > 1 are kept; one inside that range with n_alns < 2 ends the
 *     current segment.  Empty segments are never emitted.
 *   - Row keys: pos starts at -1 and increments on every row whose column 0 is not '*' (token 4); ins counts consecutive '*' rows
 *     and resets to 0 on any other row.  The key is (pos as u16, ins as u8) with wrap-around, so leading '*' rows have pos 65535 and
 *     a run of 256 '*' rows wraps ins to 0.  Such windows are taken as they are.
 *   - The supported entries of a window are collected into a map in order: a later duplicate (pos, ins) replaces an earlier one;
 *     an entry that matches no row is ignored; rows that share a key after a wrap all use its entry.
 *   - A supported row emits the argmax of its 5 logits under OrderedFloat: the last maximum wins, NaN is greatest, -0 == +0.
 *     Class 4 ('*') emits nothing.
 *   - Any other row votes over columns [0, n_alns]: token 10 ('.') is skipped, the rest counted by BASES_UPPER_COUNTER; the two
 *     largest counts are taken by a stable descending sort (ties go A < C < G < T < '*'); with tbase = BASES_UPPER[column 0] the row
 *     emits tbase if the largest count is below 2, or if the two are equal and tbase is one of them, and the largest's base
 *     otherwise.  '*' emits nothing.
 *   Columns past n_alns are never read, nor are windows with n_alns < 2.
 *
 * Synchronous: returns when the outputs are written.  With HB_CONS_DEVICE_PTRS the library's stream first waits, through an event,
 * for the work already enqueued on `stream`.  Scratch only grows, so repeated calls of the same or a smaller shape allocate nothing.
 * It needs no hb_upload_reads and no model call.
 *
 * Errors (nothing is written to the outputs; the context stays usable):
 *   HB_ERR_ARG       a NULL pointer, n_alns above 30, a supported pos above 65535 or ins above 255, or a pointer that does not
 *                    match the flag (as hb_forward_batch checks it)
 *   HB_ERR_INPUT     exactly where consensus() would panic: in a voting row of a window with n_alns >= 2, a token >= 11 in a counted
 *                    column (BASES_UPPER_COUNTER) or token 10 in column 0 (BASES_UPPER).  The message names the first such
 *                    (read, window, row, column) in row-major order.  The same bytes in a supported row, a column past n_alns or a
 *                    window with n_alns < 2 are fine.
 *   HB_ERR_CAPACITY  a batch too large for the scratch or its indexing (2^31 windows, 2^32 supported entries)
 *   HB_ERR_CUDA      a CUDA failure
 *
 * Threading: may be called from any thread, concurrently with hb_submit_*, hb_flush, hb_poll_corrected and hb_forward_batch on the
 * same context; calls of hb_consensus_batch on one context serialise among themselves.
 *
 * Counters: adds to kernel_launches, n_kernel / ms_kernel (HB_K_CONSENSUS; HB_K_SCAN for the scan), ms_consensus and host_allocs
 * when scratch grows; nothing else. */
int hb_consensus_batch(hb_ctx* ctx, uint32_t n_reads, const uint32_t* n_windows, const uint32_t* rows, const uint8_t* n_alns,
                       const uint8_t* bases, const uint32_t* n_sup, const uint32_t* supported, const float* bases_logits, uint8_t* seqs,
                       uint32_t* seg_len, uint32_t* n_segs, uint32_t flags, void* stream);

/* Host-only utility: the windows [*first_window, *end_window) one alignment contributes OverlapWindows to — the
 * coordinate-only part of extract_windows (src/windowing.rs:53-125,260-272).  HB_ERR_INPUT where the reference panics. */
int hb_window_range(const hb_overlap* ovl, uint32_t window_size, uint32_t n_windows, uint32_t* first_window, uint32_t* end_window);

/* Host-only utility (no context, no GPU): windowing::extract_windows (src/windowing.rs:44-273) of
 * the n_ovl alignments of one target that has n_windows windows (overlap_idx = position in
 * `ovl`).  Writes up to `cap` records in push order, returns the number produced in *n_out
 * (may exceed cap: call again with a larger buffer); HB_ERR_INPUT if the reference would panic. */
int hb_extract_windows(const hb_overlap* ovl, uint32_t n_ovl, uint32_t window_size, uint32_t n_windows,
                       hb_overlap_window* out, uint32_t cap, uint32_t* n_out);

/* Change hb_options.launch_targets (targets per device launch, staged per feature thread) for subsequent
 * submissions.  Call between hb_flush and the next hb_submit_*. */
int hb_set_launch_targets(hb_ctx* ctx, uint32_t launch_targets);

/* Per-kernel CUDA-event timing (hb_stats.ms_kernel / n_kernel) for subsequent launches: off by default, because
 * the two event records around each of the ~25 kernels of a launch cost device time; bench.py switches it on
 * for the one isolated launch its roofline is computed from.  Stage-level times (ms_features, ...) are always kept. */
int hb_set_kernel_timing(hb_ctx* ctx, int on);

/* Launch whatever is pending (every feature thread stages its own batch) and wait until every submitted
 * target has a result queued.  Call it once the submitting threads are quiescent (the reference's
 * equivalent is the alignment channel closing, src/lib.rs:186); it must not race with hb_submit_*. */
int hb_flush(hb_ctx* ctx);

/* Pop one finished target: the `(rid, Vec<Vec<u8>>)` of src/consensus.rs:253-257.
 * Returns 1 and fills the outputs if a result was popped, 0 if none is queued, <0 if the popped target
 * failed: then *rid names it, *seqs / *seg_len are NULL, *n_segs is 0 (nothing to release), hb_last_error()
 * says why (HB_ERR_INPUT: the reference would have panicked on its alignments; HB_ERR_CAPACITY / HB_ERR_CUDA:
 * its launch failed), and the other targets are unaffected — a host that wants the reference's behaviour
 * aborts, one that wants to keep going logs the read and polls on.
 * `*seqs` = the segments back to back (ASCII ACGT), `*seg_len[k]` their lengths; n_segs == 0
 * means consensus() returned None or produced nothing — the read is omitted from the FASTA
 * (src/consensus.rs:95-98, src/lib.rs:282-288).  Buffers stay valid until
 * hb_release_result(ctx, *seqs). */
int hb_poll_corrected(hb_ctx* ctx, uint32_t* rid, uint8_t** seqs, uint32_t** seg_len, uint32_t* n_segs);
void hb_release_result(hb_ctx* ctx, uint8_t* seqs);

const char* hb_last_error(hb_ctx* ctx); /* ctx may be NULL: error of a failed hb_create */

/* Bind the calling thread to the CPUs of the NUMA node the context's GPU is attached to (the library's own
 * launch workers always are).  For the host's feature / consumer threads of this device (src/lib.rs:159-199) on
 * multi-socket boxes.  Returns 1 if bound, 0 if the topology is unknown (nothing changed), <0 on error. */
int hb_bind_calling_thread(hb_ctx* ctx);

/* ---- counters (the reference only has progress bars, src/pbars.rs) -------------------- */
#define HB_NUM_KERNEL_CLASSES 16
/* kernel classes of ms_kernel[] / n_kernel[] */
enum { HB_K_TOKENIZE = 0, HB_K_PASS1, HB_K_SCORES, HB_K_PASS2A, HB_K_SCAN, HB_K_PILEUP, HB_K_LISTS, HB_K_STEM,
       HB_K_LAYERNORM, HB_K_GEMM, HB_K_ATTENTION, HB_K_HEADS, HB_K_CONSENSUS,
       HB_K_FFN /* fused FFN kernel */, HB_K_QKV_ATTN /* fused QKV projection + attention kernel */,
       HB_K_POS_ATTN /* attention across a window's supported positions (position-axis stage) */ };
typedef struct hb_stats {
    uint64_t targets, windows, overlap_windows, rows, supported, corrected_bases;
    uint64_t h2d_bytes, d2h_bytes, kernel_launches, device_launches /* batches */;
    uint64_t pileup_algo_bytes; /* algorithmic bytes of the pileup-build kernel (DESIGN.md; SURVEY.md §8d) */
    uint64_t gemm_flops;        /* algorithmic FLOPs of the dense contractions (QKV/out/FFN/collapse)     */
    uint64_t forward_flops;     /* all forward FLOPs at the supported positions                            */
    double ms_features, ms_forward, ms_consensus;  /* CUDA-event time per stage, summed over launches      */
    double ms_kernel[HB_NUM_KERNEL_CLASSES];       /* CUDA-event time per kernel class (timed launches)    */
    uint64_t n_kernel[HB_NUM_KERNEL_CLASSES];      /* launches per kernel class                            */
    uint64_t last_launch_targets, last_launch_windows, last_launch_bases; /* what hb_replay_last_launch re-runs */
    double ms_worker_busy;   /* host wall time the launch worker spent inside launches (staging+GPU+copy-back) */
    double ms_worker_gpu_wait; /* of which: blocked in stream synchronisation                               */
    uint64_t host_allocs;    /* page-locked / device allocations made since the last reset (0 in steady state)  */
    double ms_host_alloc;    /* wall time spent in them                                                         */
    double ms_submit_wait;   /* wall time hb_submit_* callers were blocked on back-pressure (summed over threads) */
    uint64_t class_flops[HB_NUM_KERNEL_CLASSES]; /* algorithmic FLOPs (31 read tokens per supported position) by kernel class */
    double ms_worker_phase[8]; /* launch-worker wall time by phase: 0 buffers+H2D enqueue, 1 feature launches,
                                  2 wait (row counts), 3 forward+consensus launches, 4 wait (results),
                                  5 per-read reassembly, 6 publish                                               */
} hb_stats;
int hb_get_stats(hb_ctx* ctx, hb_stats* out);
int hb_reset_stats(hb_ctx* ctx);

/* ---- parity taps (need HB_FLAG_KEEP_DEBUG; valid for targets of the most recent launch) -- */
/* shape4 = L' (rows), n_alns, n_supported, has_logits */
int hb_debug_window_shape(hb_ctx* ctx, uint32_t rid, uint32_t wid, uint32_t* shape4);
/* bases/quals: [L',31] u8 (tokens of BASES_MAP src/inference.rs:23-31 / raw quals), i.e. the
 * arguments of FeaturesOutput::update after prepare_examples; supported: [n,2] u32 (pos, ins);
 * sup_rows: [n] u32; info_logits [n], bases_logits [n,5] f32.  Any pointer may be NULL. */
int hb_debug_dump_window(hb_ctx* ctx, uint32_t rid, uint32_t wid, uint8_t* bases, uint8_t* quals,
                         uint32_t* supported, uint32_t* sup_rows, float* info_logits, float* bases_logits);

/* `herro features` (src/lib.rs:50-111, src/features.rs:724-764,806-839) from the device path: for target `rid` of the
 * most recent launch (HB_FLAG_KEEP_DEBUG) writes, per window, under <out_dir>/<read_names[rid]>/ :
 *   <wid>.features.npy   u8 [2, L', 31]: plane 0 the pileup as raw ASCII (ACGT / acgt / '*' '#' / '.'), plane 1 the qualities
 *   <wid>.supported.npy  1-D records {pos: u16, ins: u8}  (SupportedPos, src/features.rs:894-898)
 *   <wid>.ids.txt        the query read ids of all overlaps that survived the filter, in final rank order (src/features.rs:569)
 * i.e. the arguments of FeaturesOutput::update.  read_names[i] = id of read i (NUL-terminated), n_reads entries.
 * The .npy headers are the ones numpy writes (v1.0, padded to 64 bytes). */
int hb_dump_features(hb_ctx* ctx, uint32_t rid, const char* out_dir, const char* const* read_names);

/* ---- device-resident replay, used by bench.py for the HBM-resident `value` -------------- */
/* Re-run all device stages of the most recent launch from its inputs already in HBM
 * (no host<->device copies), `iters` times; returns the CUDA-event milliseconds in *ms. */
int hb_replay_last_launch(hb_ctx* ctx, uint32_t iters, float* ms);

/* ---- diagnostics ------------------------------------------------------------------------- */
/* Runs the wgmma (bf16x3) contraction kernel and the fp32 SIMT one on the same random
 * [M,K]x[N,K]^T problem (M % 128 == 0, N % 128 == 0, K % 64 == 0; lda = K + lda_extra; act: 0 none,
 * 1 ReLU, 2 ReLU with split-bf16 output; res: add a residual) and reports the largest absolute
 * difference, the largest |reference| and both kernel times. */
int hb_selftest_gemm(int cuda_device, uint32_t M, uint32_t N, uint32_t K, int act, int res, uint32_t lda_extra,
                     float* max_abs_err, float* max_abs_ref, float* ms_tc, float* ms_simt);
/* Runs the position-axis stage's masked attention kernel, through the launcher the forward uses, on n_seq sequences of
 * lens[i] rows stored back to back: qkv is [sum lens][3 * heads * head_dim] fp32 (q | k | v), head_dim 32 or 64.  Writes
 * the attention output [sum lens][heads * head_dim] as the sum of its split bf16 halves, and the kernel's time in *ms
 * (may be NULL). */
int hb_selftest_pos_attention(int cuda_device, const uint32_t* lens, uint32_t n_seq, uint32_t heads, uint32_t head_dim,
                              const float* qkv, float* out, float* ms);

#ifdef __cplusplus
}
#endif
#endif /* HERRO_B200_H */

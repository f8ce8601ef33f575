/*
 * uisrnn_b200.h -- C ABI of libuisrnn_b200.so: the H100 (sm_90a) implementation of UIS-RNN's
 * predict() hot path (beam search over GRU hypotheses).
 *
 * The reference (google/uis-rnn) has NO native / FFI layer (SURVEY.md 2.2): its only boundary
 * is the Python API.  This header is the seam a maintainer would bind (ctypes stub in
 * INTEGRATION.md); each entry point names the reference code it replaces.  All paths are
 * relative to /root/reference.
 *
 * Conventions
 *   - return 0 on success, negative uis_status on failure; message via uis_last_error()
 *     (thread-local).  Nothing throws across the ABI.
 *   - a uis_model is bound to one CUDA device; calls on one handle must be serialised by the
 *     caller; different handles may be used from different threads/processes.
 *   - caller owns every input/output buffer; the library owns the handle and its workspace.
 *   - all device work is ordered on the `stream` argument (a cudaStream_t, NULL = default
 *     stream).  The *_device entry point does not synchronise; the host-buffer entry point
 *     returns after the labels have landed in the caller's host buffers.
 */
#ifndef UISRNN_B200_H_
#define UISRNN_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define UIS_ABI_VERSION 7

typedef enum uis_status {
  UIS_OK = 0,
  UIS_ERR_INVALID = -1,     /* bad argument (shape, NULL, beam_size < 1, ...)                  */
  UIS_ERR_UNSUPPORTED = -2, /* shape / option the sm_90a kernels are not instantiated for      */
  UIS_ERR_CUDA = -3,        /* a CUDA runtime call failed; uis_last_error() has the string     */
  UIS_ERR_OVERFLOW = -4,    /* a hypothesis opened more than `kcap` clusters; retry with more  */
  UIS_ERR_NOMEM = -5,
  UIS_ERR_CAPACITY = -6     /* look_ahead >= 2: a beam step's candidate tree exhausted the device-memory arena
                               of the spill kernel (budget: UISRNN_B200_TREE_SPILL_MB)                   */
} uis_status;

typedef struct uis_model uis_model; /* opaque */

/* Inference options = the reference's inference_args (uisrnn/arguments.py:172-193). */
typedef struct uis_predict_opts {
  int32_t beam_size;      /* --beam_size      (arguments.py:175-180), 1..128 (1..32 when look_ahead >= 2) */
  int32_t look_ahead;     /* --look_ahead     (arguments.py:181-185), >= 1                     */
  int32_t test_iteration; /* --test_iteration (arguments.py:186-193), >= 1                     */
  int32_t kcap;           /* max clusters per hypothesis held on device; 0 = default (32; 16
                             when look_ahead >= 2 or on the tensor-core engine; beam_size > 32:
                             the largest of 32, 16, 8, 4 whose tables fit shared memory)        */
  int32_t n_ctas;         /* persistent CTAs to launch; 0 = one per SM                         */
  int32_t lanes;          /* utterances advanced together per CTA (share each weight pass);
                             0 = auto (FFMA engine: 2 when U >= 2 * CTAs, else 1, max 4;
                             tensor-core engine: up to columns / 8 = 6, max 8)                  */
  int32_t cluster;        /* CTAs per utterance (latency modes for few utterances; default shape,
                             depth 1, look_ahead 1): 0 = auto (32 when U * 32 <= CTAs, else 4 or 2 when
                             U * cluster <= CTAs), -1 = off, 2 / 4 / 8 = thread-block cluster (k-split of the
                             streamed weights), 32 = stationary-weights group (weights resident in the
                             shared memory of 32 CTAs, products split by rows, cooperative launch)         */
  int32_t engine;         /* matrix engine of the look_ahead-1 beam kernel: 0 = auto (tensor cores
                             when some CTA gets more than one utterance), 1 = fp32 FFMA kernels,
                             2 = wgmma tensor-core pass (fp16 hi/lo split operands, fp32-grade;
                             depth 1, hidden/dim multiples of 128; kcap defaults to 16)          */
} uis_predict_opts;

/* Optional per-call debug / parity taps.  Any pointer may be NULL.  All are HOST buffers
 * the library fills before uis_predict*() returns (it synchronises the stream if any tap is set).
 * Taps do not change the plan: a traced call runs the kernel the same call without taps runs (engine,
 * lanes, cluster or stationary-weights mode) and returns the same labels. */
typedef struct uis_debug_taps {
  int32_t trace_utt;       /* utterance index to trace step by step, -1 = none                 */
  int32_t trace_capacity;  /* rows available in step_winners / step_scores                     */
  int32_t* step_winners;   /* [trace_capacity][1+look_ahead]: (parent beam, cluster...) rows,
                              ranked order, all steps concatenated -- what uisrnn.py:551-556
                              unravels                                                         */
  float* step_scores;      /* [trace_capacity] neg_likelihood of each new hypothesis           */
  int64_t* step_offsets;   /* [steps+1] row offsets per beam step                              */
  float* final_scores;     /* [U][beam_size] final neg_likelihood per hypothesis (+inf pad)    */
  int32_t* final_k;        /* [U] clusters in the best hypothesis                              */
  float* best_mean;        /* [kcap][D]  mean_set   of the best hypothesis of `trace_utt`      */
  float* best_hidden;      /* [kcap][depth][H] hidden_set of the best hypothesis of `trace_utt` */
  int32_t* best_blocks;    /* [kcap]     block_counts of the best hypothesis of `trace_utt`    */
} uis_debug_taps;

/* Work counters of the last uis_predict*() call on this handle (for bench.py's accounting). */
typedef struct uis_stats {
  int64_t utterances;
  int64_t frames;          /* un-tiled input rows                                              */
  int64_t beam_steps;      /* sum over utterances of test_iteration * N / look_ahead (ceil)    */
  int64_t gru_columns;     /* GRU+MLP evaluations actually performed                           */
  int64_t weight_passes;   /* full passes over (W_hh, W1, W2) streamed by all CTAs             */
  int64_t candidates;      /* scored (hypothesis, cluster) candidates                          */
  int64_t kernel_launches; /* CUDA kernels launched by the call                                */
  int32_t ctas;            /* persistent CTAs used                                             */
  int32_t max_k;           /* largest cluster count seen in any hypothesis                     */
  float prepass_ms;        /* device time of the input-projection GEMM (CUDA events on `stream`) */
  float beam_ms;           /* device time of the persistent beam-search kernel                 */
  int32_t lanes;           /* lanes per CTA used                                               */
  int32_t cluster;   /* CTAs per utterance the last call used: 1 = none, 2/4/8 = cluster, 32 = stationary-weights group */
  int32_t engine;          /* 1 = FFMA kernels, 2 = tensor-core pass                            */
  int32_t tc_columns;      /* tensor-core pass: columns per weight pass (0 otherwise)           */
  int64_t phase_cycles[10]; /* SM cycles summed over CTAs: [0] re-pack (P4), [1] gather, [2] GRU pass,
                               [3] W1 pass, [4] W2 pass, [5] advance/back-track, [6] frame landing
                               (P0), [7] scoring (P1), [8] ranking (P2), [9] column/slot assignment (P3) */
  int64_t tc_cycles[4];     /* tensor-core pass, SM cycles of consumer thread 0 summed over CTAs: waiting for [0] a
                               weight box not yet landed (TMA), [1] MMAs to complete; [2] staging the B operands;
                               [3] inside passes */
  /* host-buffer entry point (uis_predict) only, ABI 4: */
  float h2d_ms;             /* span of the chunked host->device copies on the copy stream                              */
  float pipeline_ms;        /* compute stream: first cast kernel -> start of the beam kernel (casts + input projections,
                               overlapped with the copies)                                                             */
  float host_ms;            /* wall time inside uis_predict()                                                          */
  int32_t chunks;           /* staging chunks the float64 rows travelled in                                            */
  int32_t groups;           /* every predict and score entry point: groups of whole utterances the list ran in (1: at
                               once; > 1: it did not fit the device at once); the other fields add up over the groups */
  int32_t staged;           /* 1: the inputs were pageable and went through the library's pinned staging ring (host
                               copy threads), 0: copied straight from the caller's (pinned) buffers                     */
} uis_stats;

int uis_version(void);
const char* uis_last_error(void);

/*
 * Replaces UISRNN.__init__ / load (uisrnn/uisrnn.py:83-107, 149-170) for the inference path:
 * takes the CoreRNN parameters (uisrnn.py:35-43, PyTorch state_dict layout, row-major fp32):
 *   w_ih [3H,D]  w_hh [3H,H]  b_ih [3H]  b_hh [3H]   (gru.*_l0, gate order r,z,n)
 *   w1 [H,H] b1 [H] (linear_mean1)   w2 [D,H] b2 [D] (linear_mean2)
 *   h0 [depth,H] (rnn_init_hidden)   sigma2 [D]
 * Stacked layers (depth 2..4): w_ih = [gru.weight_ih_l0 (3H x D) | gru.weight_ih_l1 (3H x H) | ...]
 * concatenated, w_hh / b_ih / b_hh = the per-layer tensors concatenated in layer order.
 * Pointers may be host or device memory (copied, never retained).  Precomputes the per-model
 * constants CoreRNN(zeros, rnn_init_hidden) that uisrnn.py:435-439 recomputes per candidate.
 */
int uis_model_create(uis_model** out, int device, int D, int H, int depth,
                     const float* w_ih, const float* w_hh, const float* b_ih, const float* b_hh,
                     const float* w1, const float* b1, const float* w2, const float* b2,
                     const float* h0, const float* sigma2, double transition_bias,
                     double crp_alpha);
int uis_model_destroy(uis_model* m);

/* Copies the per-model constants back (host buffers, fp32): mean0 [D], hidden0 [depth][H]. */
int uis_model_constants(uis_model* m, float* mean0, float* hidden0);

/*
 * Replaces UISRNN.predict / predict_single / parallel_predict (uisrnn/uisrnn.py:479-623) for a
 * list of U utterances held in HOST memory:
 *   seqs[u]      -> row-major float64 [n_frames[u], D]   (the ndarray the reference validates at
 *                   uisrnn.py:511-521; cast to fp32 on the device, = uisrnn.py:525-526)
 *   labels_out[u]-> int32 [n_frames[u]]  = beam_set[0].trace[-N:] (uisrnn.py:561)
 * Host->device copies, the beam search and the device->host copy of the labels all happen
 * inside the call.  Utterances are independent; they are scheduled longest-first over
 * persistent CTAs.
 * Lists larger than the device (every predict and score entry point): when the per-frame workspace of the whole list
 * does not fit the free device memory, the call runs consecutive groups of whole utterances one after the other on
 * `stream`, each planned on its own, and writes every output where the whole call would.  An utterance longer than the
 * budget is a group of its own.  The environment variable UISRNN_B200_MAX_ROWS (frames, >= 1) sets the budget instead.
 * Debug taps keep a call in one group.
 */
int uis_predict(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                const uis_predict_opts* opts, int32_t* const* labels_out,
                const uis_debug_taps* taps, void* stream);

/*
 * Same search with inputs already resident in HBM:
 *   x_dev      fp32 [frame_offsets[U], D] (all utterances concatenated), device memory
 *   frame_offsets  HOST int64 [U+1]
 *   labels_dev int32 [frame_offsets[U]], device memory
 * Asynchronous on `stream` unless taps != NULL.
 */
int uis_predict_device(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                       const uis_predict_opts* opts, int32_t* labels_dev,
                       const uis_debug_taps* taps, void* stream);

/*
 * ABI 5: the same searches with a bound on the number of speakers (clusters) per utterance.  Not in the reference,
 * whose only knob is crp_alpha.  The three extra arguments, any of which may be NULL:
 *   max_speakers [U] HOST int32: 0 = no bound, else >= 1.  A candidate that would take its hypothesis past
 *                    max_speakers clusters scores +inf (it is never generated), so every label is < max_speakers
 *                    and, with kcap >= max_speakers, UIS_ERR_OVERFLOW cannot occur for that utterance.  Ranking and
 *                    tie-breaking are those of the unbounded search.
 *   min_speakers [U] HOST int32: 0 = no bound, else <= max_speakers when that is set.  Applied at the end only: the
 *                    labels come from the best-ranked final hypothesis with at least min_speakers clusters, or from
 *                    rank 0 when the final beam holds none (speakers_out then reports fewer than min_speakers).
 *   speakers_out [U] int32 (HOST for uis_predict_bounded, DEVICE for uis_predict_device_bounded): clusters of the
 *                    returned hypothesis, 0 for an empty or failed utterance.
 * "Speakers" counts clusters over the whole tiled decode (test_iteration copies): with test_iteration > 1 the
 * returned last copy may use fewer distinct ids.  Any other value is UIS_ERR_INVALID.  Both bounds NULL (or 0)
 * decode exactly as uis_predict / uis_predict_device, which are these calls with three NULLs.
 * Workspace: a call with bounds holds 8 * U more device bytes, and uis_predict_bounded with speakers_out 4 * U more,
 * beyond uis_predict_workspace_bytes().
 */
int uis_predict_bounded(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                        const uis_predict_opts* opts, int32_t* const* labels_out, const uis_debug_taps* taps, void* stream,
                        const int32_t* max_speakers, const int32_t* min_speakers, int32_t* speakers_out);
int uis_predict_device_bounded(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                               const uis_predict_opts* opts, int32_t* labels_dev, const uis_debug_taps* taps, void* stream,
                               const int32_t* max_speakers, const int32_t* min_speakers, int32_t* speakers_dev);

/*
 * ABI 6: the N best hypotheses of every utterance, with their scores.  Not in the reference, which returns rank 0's
 * labels only.  Each call takes the bounded call's arguments (speaker bounds as above; the cluster counts come in
 * `out`) plus
 *   n_best       1 <= n_best <= beam_size, else UIS_ERR_INVALID.
 *   out          where the hypotheses go (HOST buffers for uis_predict_nbest, DEVICE buffers for
 *                uis_predict_device_nbest; the label member the other entry point uses is ignored).
 * Hypothesis j < n_best of an utterance is the j-th final rank (in rank order) with at least min_speakers clusters;
 * when no final rank has that many, it is rank 0 alone.  So hypothesis 0 is what uis_predict_bounded returns.  Its
 * score is the neg_likelihood accumulated over the whole tiled decode (BeamState.neg_likelihood, the value
 * uis_debug_taps.final_scores shows).  Entries past count[u] hold labels -1, score +inf and 0 clusters; an empty or
 * failed utterance returns no hypothesis.  With test_iteration > 1 two hypotheses may differ only in an earlier
 * copy and so carry the same labels (the last copy's); they are not merged.
 * uis_predict_bounded / uis_predict_device_bounded are n_best = 1 calls of the same search.
 * Workspace: beyond uis_predict_workspace_bytes(), uis_predict_nbest holds 4 * (n_best - 1) * rows more label bytes
 * and 4 * (2 * n_best + 1) * U bytes for the outputs (its group planner counts both).
 */
typedef struct uis_nbest_out {
  int32_t* const* labels_out;  /* host entry: labels_out[u] -> int32 [n_best][n_frames[u]]                        */
  int32_t* labels_dev;         /* device entry: int32 [n_best][frame_offsets[U]], plane 0 = uis_predict_device's labels */
  float* scores;               /* [U][n_best]  neg_likelihood, +inf where absent                                   */
  int32_t* speakers;           /* [U][n_best]  clusters, 0 where absent (may be NULL)                              */
  int32_t* count;              /* [U]          hypotheses returned (may be NULL)                                   */
} uis_nbest_out;

int uis_predict_nbest(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                      const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                      const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                      const uis_nbest_out* out);
int uis_predict_device_nbest(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                             const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                             const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                             const uis_nbest_out* out);

/*
 * ABI 7: the score of given labellings.  Not in the reference, where the same quantity exists only inside the search
 * (BeamState.neg_likelihood, uisrnn.py:388-453).  The score of utterance u is the neg_likelihood of the trace that
 * assigns frame t to cluster labels[u][t]: per frame loss_t = fl32(f64(mse_t) - pen_t), with mse_t the Gaussian term
 * of the frame against its cluster's running mean before that frame (mean0 for a new cluster; +inf by the first-column
 * rule) and pen_t the transition / ddCRP term of the trace so far; the score is the fp32 running sum of loss_t in frame
 * order.  That is the arithmetic of the search, so a hypothesis the FFMA beam kernel kept (engine 1, no cluster mode)
 * scores exactly the value its N-best entry reports.  Lower is better.  test_iteration is not applied: the sequence
 * is scored once, as given (tile both the rows and the labels to score a tiled decode).  An empty utterance scores 0.
 *   labels       canonical int32 ids: 0, 1, 2, ... in order of first appearance (the ids a trace holds); anything
 *                else is UIS_ERR_INVALID, and uis_last_error() names the utterance and the frame.  Any number of
 *                clusters per utterance (no kcap).
 *   scores_out   [U] float32 neg_likelihood.
 *   frame_out    per-frame increments loss_t (may be NULL); summed in fp32 in frame order they give the score bit for
 *                bit.
 * uis_score: host buffers (seqs[u] float64 [n_frames[u], D] as in uis_predict, labels[u] int32 [n_frames[u]],
 * frame_out[u] float32 [n_frames[u]]); returns when the scores have landed.  uis_score_device: device buffers in the
 * layout of uis_predict_device (x_dev fp32 [frame_offsets[U], D], labels_dev int32 [frame_offsets[U]], scores_dev [U],
 * frame_dev [frame_offsets[U]]; frame_offsets on the host).  It copies the labels back to plan the chains, which
 * synchronises `stream` once at the start of the call; the kernels are then enqueued without waiting, group after group
 * when the list runs in groups.
 * Work: one GRU + MLP column per frame that is not the first of its cluster, in the FFMA weight pass of the beam
 * kernels (every kernel shape and depth).  Workspace: the handle's cache, about (12 H + 4 D + 24) bytes per frame; a
 * list that does not fit the device is scored in groups of whole utterances (see uis_predict).  uis_get_stats after a
 * score call fills utterances, frames, gru_columns, weight_passes, kernel_launches, ctas, max_k (most clusters in one
 * utterance), prepass_ms, beam_ms (the chain kernel), engine = 1 and, for uis_score, the host-path fields; the rest
 * is zero.
 */
int uis_score(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
              const int32_t* const* labels, float* scores_out, float* const* frame_out, void* stream);
int uis_score_device(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                     const int32_t* labels_dev, float* scores_dev, float* frame_dev, void* stream);

/*
 * Decoding-parameter sweeps (same ABI version 7; additive).  Not in the reference, which decodes with the model's
 * crp_alpha (--crp_alpha) and transition_bias only.  One call decodes or scores a list under `count` (crp_alpha,
 * transition_bias) pairs: config c gives exactly what the plain call returns for a model created with pair c.  The
 * input rows cross the bus once and their input projection runs once; the kernels run U * count independent jobs,
 * job j = utterance j % U under config j / U (the configs of one utterance are scheduled side by side).
 *   params       count >= 1, U * count <= INT_MAX, every crp_alpha finite and > 0, every transition_bias finite and in
 *                (0, 1); anything else is UIS_ERR_INVALID and uis_last_error() names the pair.  Host arrays, read
 *                during the call only.
 * uis_predict_sweep / uis_predict_device_sweep take the arguments of uis_predict_nbest / uis_predict_device_nbest
 * (speaker bounds per utterance, the same for every config) and write config-major outputs, config c's block being
 * what the N-best call writes:
 *   host labels    labels_out[u] -> int32 [count][n_best][n_frames[u]]
 *   device labels  labels_dev    -> int32 [count][n_best][frame_offsets[U]]
 *   scores, speakers [count][U][n_best];  count [count][U]
 * uis_score_sweep / uis_score_device_sweep take the arguments of uis_score / uis_score_device: scores [count][U];
 * per-frame increments frame_out[u] -> float32 [count][n_frames[u]] (host) or frame_dev -> [count][frame_offsets[U]]
 * (device).  The chain kernel and the first-visit kernel run once; the reduce kernel runs once per config.
 * Debug taps index jobs: trace_utt = c * U + u, final_scores [count * U][beam_size], final_k [count * U].
 * uis_get_stats after a sweep: utterances = jobs (U * count), frames = distinct input rows; the work counters cover
 * every job (a score sweep's gru_columns equal a plain score call's).  Every sweep runs a list that does not fit the
 * device in groups of whole utterances, each with all its configs.
 * Synchronisation: the log tables of a sweep are built on the host and cached in the handle.  A sweep whose pairs (or
 * longest tiled decode) differ from the previous sweep's rewrites them in place, and first synchronises the DEVICE
 * (cudaDeviceSynchronize: an earlier call on any stream may still read them), so uis_predict_device_sweep /
 * uis_score_device_sweep block in that case; a sweep that repeats the previous sweep's pairs enqueues without waiting.
 * The tables of the model's own pair, which the plain entry points use, are kept apart and never rewritten by a sweep.
 */
typedef struct uis_decode_params {
  int32_t count;
  const double* crp_alpha;        /* [count] */
  const double* transition_bias;  /* [count] */
} uis_decode_params;

int uis_predict_sweep(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                      const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                      const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                      const uis_nbest_out* out, const uis_decode_params* params);
int uis_predict_device_sweep(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                             const uis_predict_opts* opts, const uis_debug_taps* taps, void* stream,
                             const int32_t* max_speakers, const int32_t* min_speakers, int32_t n_best,
                             const uis_nbest_out* out, const uis_decode_params* params);
int uis_score_sweep(uis_model* m, const double* const* seqs, const int64_t* n_frames, int U,
                    const int32_t* const* labels, float* scores_out, float* const* frame_out, void* stream,
                    const uis_decode_params* params);
int uis_score_device_sweep(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                           const int32_t* labels_dev, float* scores_dev, float* frame_dev, void* stream,
                           const uis_decode_params* params);

/*
 * Scoring labellings held on the device as arbitrary ids (same ABI version 7; additive).  uis_score_device_sweep with
 *   ids_dev      int64 [frame_offsets[U]] device memory: any values per frame.  A labelling is taken up to renaming:
 *                frame t of utterance u belongs to cluster c, c = the number of distinct ids of u first seen before
 *                ids_dev[t]'s first appearance (what canonical labels hold), so no input is an invalid labelling.
 *   labels_dev   int32 [frame_offsets[U]] device memory, may be NULL: receives those canonical labels.
 * The other arguments and the outputs are those of uis_score_device_sweep; frame_offsets[0] must be 0, the list
 * holds fewer than 2^31 - 1 frames, x_dev is 16-byte aligned (the rows are read with 16-byte loads) and ids_dev 8-byte
 * aligned; anything else is UIS_ERR_INVALID.  The renaming and the chain plan run on the device (sorts and scans on `stream`),
 * so the call reads nothing back: it enqueues its work on `stream` and returns, except where a sweep rewrites its log
 * tables (see above) or the handle's workspace grows (cudaMalloc / cudaFree).  A list run in groups stays so: its
 * groups are cut from the host frame_offsets, each is renamed and planned on the device on its own (renaming is per
 * utterance, so its ids rename as in the whole call), and the workspace is sized for the largest group before the
 * first is enqueued.  The scores are those
 * uis_score_device_sweep gives for the canonical labels, bit for bit.  uis_get_stats fills the fields a score call
 * fills, max_k from the device plan.
 *
 * Every entry point of a handle orders its device work after the previous call's: each call records an event on its
 * stream at its end, and the next call's stream waits for it (cudaStreamWaitEvent; the host does not block).  So calls
 * on one handle from different streams do not overwrite the workspace under each other's kernels.
 */
int uis_score_device_ids(uis_model* m, const float* x_dev, const int64_t* frame_offsets, int U,
                         const int64_t* ids_dev, float* scores_dev, float* frame_dev, int32_t* labels_dev,
                         void* stream, const uis_decode_params* params);

/* Device bytes uis_predict_device() will hold for this problem (workspace is cached in the handle). */
size_t uis_predict_workspace_bytes(uis_model* m, const int64_t* frame_offsets, int U,
                                   const uis_predict_opts* opts);

int uis_get_stats(uis_model* m, uis_stats* out);

/* ------------------------------------------------------------------------------------------------
 * Training: one iteration of UISRNN.fit_concatenated (uisrnn/uisrnn.py:252-295) on the device.
 * Parameters are 4 * depth + 6 tensors, in this order, row-major fp32 (PyTorch layouts); depth 1:
 *   0 gru.weight_ih_l0 [3H,D]  1 gru.weight_hh_l0 [3H,H]  2 gru.bias_ih_l0 [3H]  3 gru.bias_hh_l0 [3H]
 *   4 linear_mean1.weight [H,H] 5 linear_mean1.bias [H]   6 linear_mean2.weight [D,H] 7 linear_mean2.bias [D]
 *   8 rnn_init_hidden [H]       9 sigma2 [D]
 * depth > 1: the four gru tensors of layer 0, then of layer 1 (weight_ih_l1 is [3H,H]), ..., then linear_mean1/2,
 * rnn_init_hidden [depth,H], sigma2.
 * (all but the last two = the "rnn parameters" group that is norm-clipped, uisrnn.py:120-133, 292.)
 */
typedef struct uis_trainer uis_trainer; /* opaque; owns parameters, gradients and Adam state */

typedef struct uis_train_hparams {          /* training_args, uisrnn/arguments.py:105-169 */
  float learning_rate;                      /* --learning_rate                                   */
  float sigma_alpha, sigma_beta;            /* --sigma_alpha / --sigma_beta                      */
  float regularization_weight;              /* --regularization_weight                           */
  float grad_max_norm;                      /* --grad_max_norm                                   */
  int32_t train_sigma2;                     /* 1 if sigma2 is estimated (model_args.sigma2 None) */
  /* ABI 4: stacked GRU layers (model_args, uisrnn/arguments.py:55-64; nn.GRU(num_layers, dropout), uisrnn.py:35-43) */
  int32_t rnn_depth;                        /* --rnn_depth, 1..4 (0 = 1)                         */
  float rnn_dropout;                        /* --rnn_dropout: applied to the output sequence of every layer but the
                                               last, in every training iteration (train mode), when rnn_depth > 1   */
  int64_t dropout_seed;                     /* seed of the dropout masks: keep(i) is a pure function of
                                               (seed, iteration, layer, element) -- see uis_train.cu dropout_hash   */
} uis_train_hparams;

/* params: 4 * hp->rnn_depth + 6 host (or device) pointers, copied.  Adam state starts at zero (a fresh optimiser per
 * fit_concatenated call, uisrnn.py:235-236). */
int uis_trainer_create(uis_trainer** out, int device, int D, int H, const float* const* params,
                       const uis_train_hparams* hp);
int uis_trainer_destroy(uis_trainer* t);

/* One iteration on one batch = what utils.pack_sequence builds (utils.py:237-246): x_host fp32
 * [L][B][D] zero-padded, time-major, row 0 all zeros; lengths[B] (incl. the zero row) sorted
 * descending with lengths[0] == L; any B >= 1 (the recurrence runs in groups of 32 columns).  mode 0: forward + backward + clip + Adam + clamp;
 * mode 1: forward + backward only (for gradient checks); mode 2: data-parallel shard (see below).  losses_out[3] (host, may be NULL) =
 * negative log likelihood, sigma2 prior, regularisation -- the three numbers uisrnn.py:297-310 logs.
 * With losses_out == NULL the call only enqueues work on `stream` (the host batch has been staged
 * when it returns); read the losses later with uis_trainer_losses(). */
int uis_trainer_step(uis_trainer* t, const float* x_host, const int32_t* lengths, int B, int L, int mode,
                     float* losses_out, void* stream);

/* what = 0: current parameters, 1: gradients of the last step.  out: 4 * depth + 6 host pointers (NULL = skip). */
int uis_trainer_get(uis_trainer* t, int what, float* const* out);

/* Losses of the last `count` (<= 4096) steps, oldest first: out[count][3] host floats.  Synchronises. */
int uis_trainer_losses(uis_trainer* t, int count, float* out);

/*
 * Training set resident on the device (SURVEY.md 8(f) f1; replaces the per-iteration host work of
 * utils.pack_sequence, utils.py:204-250, and the num_permutations-fold float64 copy of
 * utils.resize_sequence, utils.py:172-201).  rows: host float64 [n_rows][D] = the concatenated training
 * sequence (cast to fp32 on the device); index: host int32 [n_index] = the row indices of every
 * sub-sequence back to back; offsets: host int64 [n_sub + 1].  uis_trainer_step_corpus() then runs one
 * iteration on the batch whose columns are sub-sequences chosen[0..B) (the caller keeps the reference's RNG
 * draw and passes the ids in pack_sequence's column order: lengths descending); the batch tensor is
 * gathered on the device, zero frame first, zero padded.
 */
int uis_trainer_set_corpus(uis_trainer* t, const double* rows, int64_t n_rows, const int32_t* index, int64_t n_index,
                           const int64_t* offsets, int32_t n_sub);
int uis_trainer_step_corpus(uis_trainer* t, const int32_t* chosen, int B, int mode, float* losses_out, void* stream);

/*
 * Training set read in place from device memory (same ABI version 7; additive).  Instead of a float64 host copy,
 *   row_addr  device array of n_rows row addresses: row r is D elements of `dtype` in unit element stride starting at
 *             row_addr[r], aligned to the element size (no wider alignment is assumed; rows may overlap or repeat).
 *   dtype     one of uis_dtype.
 * index, offsets and n_sub are those of uis_trainer_set_corpus and are checked the same way on the host.  Null
 * pointers, an unknown dtype, inconsistent sizes or an index out of range give UIS_ERR_INVALID before any device work.
 * The trainer keeps no copy of the rows: every later uis_trainer_step_corpus gathers its batch from row_addr and
 * the rows it points to, converting each element to fp32 (float64 rounds to nearest, as uis_trainer_set_corpus's
 * cast does; float16 and bfloat16 convert exactly).  So the table and the rows must stay allocated and unchanged
 * until the next uis_trainer_set_corpus* call or uis_trainer_destroy, and a step reads what they hold when its
 * gather runs on its stream.  The trainer's initialisation (uis_trainer_create) and the index upload run on the legacy
 * default stream; `stream` is made to wait for them on an event, so steps on any stream, non-blocking ones included,
 * start after them, and the call does not wait for earlier work on `stream`.  An fp32 corpus of an earlier
 * uis_trainer_set_corpus is freed (cudaFree, which may synchronise the device).
 */
typedef enum uis_dtype {
  UIS_DTYPE_F32 = 0,
  UIS_DTYPE_F16 = 1,
  UIS_DTYPE_BF16 = 2,
  UIS_DTYPE_F64 = 3
} uis_dtype;

int uis_trainer_set_corpus_device(uis_trainer* t, const void* const* row_addr, int32_t dtype, int64_t n_rows,
                                  const int32_t* index, int64_t n_index, const int64_t* offsets, int32_t n_sub,
                                  void* stream);

/*
 * Data-parallel fit() (optional; SURVEY.md 8(e)): every rank runs uis_trainer_step(mode = 2) on its
 * shard of the mini-batch (forward + backward with UN-normalised gradients), exports
 *   [gradients of all parameters but sigma2 | per-dimension squared-residual sums | per-dimension counts | row count]
 * (uis_trainer_comm_size() floats) into a caller-owned DEVICE buffer, all-reduces(sum) it (NCCL over
 * NVLink: one collective per iteration), and hands it back: uis_trainer_comm_apply() normalises by the
 * global row count, forms the sigma2 gradient and the three losses from the global statistics, adds the
 * regulariser, clips and takes the Adam step -- identically on every rank.  A rank that holds no column of
 * an iteration (a mini-batch narrower than the world) runs no step and exports nothing: it contributes a
 * zero buffer to the sum and calls uis_trainer_comm_apply() all the same, which it may do before its
 * first uis_trainer_step().
 */
int64_t uis_trainer_comm_size(uis_trainer* t);
int uis_trainer_comm_export(uis_trainer* t, float* dev_buf, void* stream);
int uis_trainer_comm_apply(uis_trainer* t, const float* dev_buf, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* UISRNN_B200_H_ */

/*
 * mosh2.h -- C-ABI of libmosh2.so, the H100 (sm_90a) MoSh++ Stage-II pose solver.
 *
 * The reference has no FFI: its Stage-II plug-in point is a Python callable,
 *     MoSh.mosh_stageii(self, mosh_stageii_func)          src/moshpp/mosh_head.py:268-301
 * invoked as mosh_stageii_func(mocap_fname, cfg, markers_latent, latent_labels, betas,
 * marker_meta, v_template_fname) (mosh_head.py:280-286; reference implementation
 * src/moshpp/chmosh.py:458-741).  moshpp_b200/chmosh.py keeps that signature and drives this
 * library through ctypes; INTEGRATION.md shows the binding a reference maintainer would add.
 *
 * Conventions: plain pointers and sizes only; every host buffer is caller-owned, C-contiguous,
 * float64 / int32 / uint8; the library owns all device memory behind the opaque handles; every
 * entry point returns 0 or a negative MOSH2_E_* code and never throws across the ABI;
 * mosh2_last_error() returns a thread-local message.  One model handle per GPU; calls on one
 * handle / job must be serialised by the caller, different handles are independent.
 */
#ifndef MOSH2_H_
#define MOSH2_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MOSH2_VERSION 107

enum {
    MOSH2_OK = 0,
    MOSH2_E_INVALID = -1,   /* bad argument / inconsistent sizes            */
    MOSH2_E_CUDA = -2,      /* CUDA runtime error (message in last_error)   */
    MOSH2_E_NO_DEVICE = -3, /* no usable sm_90 device                       */
    MOSH2_E_TOO_LARGE = -4  /* model does not fit the kernel (shared memory, tree depth > 16, > 254 joints) */
};

enum { MOSH2_F32 = 0, MOSH2_F64 = 1 };

/* per-frame status bits written to mosh2_result.status */
enum {
    MOSH2_ST_SOLVED = 1,       /* both dog-legs of the frame terminated by the reference's stop rules */
    MOSH2_ST_SKIPPED = 2,      /* no visible marker: frame skipped (chmosh.py:586-588)                  */
    MOSH2_ST_HAS_VELO = 4,     /* the velocity term was active (third processed frame on, chmosh.py:624) */
    MOSH2_ST_HAS_EXTRAP = 8,   /* the DMPL extrapolation term was active (chmosh.py:694-697)            */
    MOSH2_ST_GN_FALLBACK = 16, /* a Gauss-Newton system was not positive definite; Cauchy step used     */
    MOSH2_ST_MAXITER = 32,     /* a dog-leg hit maxiter                                                 */
    MOSH2_ST_SHORT_WARMUP = 64 /* chunked schedule: the chunk of this frame found fewer solved warm-up frames than
                                  asked for (a long marker drop-out in front of it); rerun the range sequentially
                                  if reference-exact continuity across the gap matters                          */
};

/* Constants of one (body model, betas, latent markers) triple, as laid out by
 * moshpp_b200/pack.py:build_pack (what chmosh.py:488-514,548-579 sets up before the frame loop;
 * models/smpl_fast_derivatives.py:52-241; transformed_lm.py:59-113; prior/gmm_prior_ch.py:107-134).
 * "slot" = 3*marker + t, t = 0..2 the three attachment vertices of a marker. */
typedef struct mosh2_model_desc {
    int32_t n_joints, n_markers, body_dof, p_red, n_hand_red, n_hand_full, n_dmpl;
    int32_t kw;               /* skinning weights kept per slot, 1..8 (SMPL-family models: 4) */
    const int32_t *parents;   /* [n_joints], -1 for the root; the tree may be at most 16 levels deep */
    const int32_t *w_joint;   /* [3M*kw] skinning joint ids, -1 padded                       */
    const double *hand_comps; /* [n_hand_red * n_hand_full]  selected_components             */
    const double *hands_mean; /* [n_hand_full]                                               */
    const double *v0;         /* [3M*3]  shaped template rows                                */
    const double *sd;         /* [3M*3*n_dmpl] DMPL directions of the slots                  */
    const double *pd;         /* [(n_joints-1) * 9M * 9] pose-blend slabs                    */
    const double *w_val;      /* [3M*kw]                                                     */
    const double *j0;         /* [n_joints*3]                                                */
    const double *jd;         /* [n_joints*3*n_dmpl]                                         */
    const double *coefs;      /* [M*3] marker attachment coefficients                        */
    int32_t prior_k, prior_d, prior_off; /* max-mixture prior on pose[prior_off : prior_off+prior_d] ...          */
    const int32_t *prior_ids;            /* ... or, if not NULL, on pose[prior_ids[0..prior_d)] (animal models)      */
    const double *prior_means;   /* [K*D]                                                    */
    const double *prior_Q;       /* [K*D*D]  0.5 * inv(cov_k)                                */
    const double *prior_neglogw; /* [K]                                                      */
    int32_t n_free1, n_free2;    /* free variables of Step 1 / Step 2 (chmosh.py:645-649,676-699) */
    const int32_t *free1, *free2; /* indices into x = [trans(3) | pose(p_red) | dmpl(n_dmpl)] */
    int32_t finger_lo, finger_hi; /* reduced-pose ids penalised by poseH in Step 2            */
    /* optimize_face (SMPL-X; chmosh.py:560-566,685-689): the last n_expr of the n_dmpl linear coefficients are
     * expression coefficients (sd / jd hold their directions after the DMPL ones); [face_lo, face_hi) are the
     * reduced-pose ids of the jaw, penalised by poseF in Step 2 */
    int32_t n_expr, face_lo, face_hi;
    /* animal_horse (chmosh.py:572-573,615-617; prior/horse_body_prior.py:56-71): besides the pose prior (here: prior_k = 1,
     * Q = P P^T, -log w = 0) a joint-angle term r_i = 2 wt_pose exp(2 s_i pose[jangles_ids[i]]); its SSE is reported in
     * the poseH column of mosh2_result.errs (animal models have no finger term).  n_jangles <= 16. */
    int32_t n_jangles;
    const int32_t *jangles_ids;
    const double *jangles_signs;
} mosh2_model_desc;

/* Stage-II weights and dog-leg options (support_data/conf/moshpp_conf.yaml:95-125,
 * chmosh.py:460,596-609,651-653,669-671,697,703-705). */
typedef struct mosh2_options {
    double wt_data, wt_poseB, wt_poseH, wt_velo, wt_dmpl, wt_annealing, wt_extrap_dmpl;
    double num_train_markers;
    double delta_0, e3_first, e3;
    int32_t maxiter;
    int32_t optimize_fingers, optimize_dynamics;
    double wt_poseF, wt_expr;  /* moshpp_conf.yaml: stageii_wt_poseF (annealed), stageii_wt_expr */
    int32_t optimize_face;
} mosh2_options;

/* Outputs, one row per input frame (rows of skipped frames are zero). */
typedef struct mosh2_result {
    double *fullpose;    /* [F * 3*n_joints]            chmosh.py:719   */
    double *pose;        /* [F * p_red]   reduced pose (debug)          */
    double *trans;       /* [F * 3]                      chmosh.py:720   */
    double *dmpls;       /* [F * n_dmpl] or NULL: DMPL, then expression coefficients   chmosh.py:722,724 */
    double *markers_sim; /* [F * M * 3]                  chmosh.py:716   */
    double *errs;        /* [F * 8] SSE of data,poseB,velo,poseH,dmpl,extrap_dmpl,poseF,expr  chmosh.py:712-714 */
    int32_t *status;     /* [F] MOSH2_ST_* bits                           */
    int32_t *counters;   /* [F * 4] dog-leg iterations, residual evals, Jacobian builds, minimisations */
} mosh2_result;

typedef struct mosh2_model mosh2_model;
typedef struct mosh2_job mosh2_job;

int mosh2_version(void);
const char *mosh2_last_error(void);
int mosh2_device_count(void);

void mosh2_default_options(mosh2_options *opt);

/* Job buffers (device and pinned host memory) are recycled between jobs; this returns the cached blocks to the driver. */
void mosh2_release_cached_memory(void);

/* Uploads the constants to `device` (both f32 and f64 copies). */
int mosh2_model_create(const mosh2_model_desc *desc, int device, mosh2_model **out);
void mosh2_model_destroy(mosh2_model *m);

/* Parallel-in-time schedule of a job (DESIGN.md section 4).  The reference solves the frames of a sequence one after
 * the other (chmosh.py:584-724); chunk_len <= 0 does exactly that in one thread block.  chunk_len > 0 cuts the
 * sequence into chunks solved concurrently; every chunk starts early enough to solve chunk_warmup frames (frames with
 * at least one visible marker) before its first emitted frame, from the reference's own cold start.  The last
 * warmup_full of those run the full per-frame schedule, the earlier ones a single linearisation of the Step-2 problem
 * (warmup_full < 0 or >= chunk_warmup: all of them run the full schedule).  first_extra > 0: the first chunk of every
 * sequence -- which has no warm-up to solve -- emits chunk_len + first_extra frames, so that with first_extra = the cost
 * of a warm-up all chunks of a sequence finish together and no chunk starts closer to the sequence start than a warm-up.
 * A chunk whose walk-back does reach the first frame of its sequence solves all those frames with the full schedule: it
 * is then the reference's own recursion from its own start, and its rows equal the sequential pass exactly. */
typedef struct mosh2_schedule {
    int32_t chunk_len, chunk_warmup, warmup_full, first_extra;
} mosh2_schedule;

/* A job = device buffers for one sequence of n_frames frames. */
int mosh2_job_create(mosh2_model *m, const mosh2_options *opt, int32_t n_frames, const mosh2_schedule *sched,
                     int32_t precision, mosh2_job **out);
/* The same for n_seq sequences of ONE subject (one model) solved by one launch: the job's frame axis holds the sequences
 * back to back (n_frames = sum of frame_counts), chunks never straddle a sequence boundary and every sequence starts
 * from its own cold start.  All per-frame buffers (obs, vis, results) are indexed by the concatenated frame axis. */
int mosh2_job_create_batch(mosh2_model *m, const mosh2_options *opt, int32_t n_seq, const int32_t *frame_counts,
                           const mosh2_schedule *sched, int32_t precision, mosh2_job **out);
/* The same for sequences of SEVERAL subjects: sequence q is solved with models[model_of_seq[q]].  The frame axis and every
 * other job call are as for mosh2_job_create_batch (mosh2_job_linearize refuses a multi-model job).  All models must be on one
 * device and have the same kernel shape -- equal n_joints, n_markers, body_dof, p_red, n_hand_red, n_hand_full, n_dmpl, kw,
 * n_free1, n_free2, finger range, face range, n_expr, n_jangles, prior_k, prior_d and hand-block structure of hand_comps --
 * so that one workspace plan serves the whole launch; their tables (shape, latent markers, attachment, prior, ...) may
 * differ, e.g. the male and female model of one family.  A mismatch returns MOSH2_E_INVALID and mosh2_last_error names the
 * first field that differs.  The models must outlive the job (as the model of any job must). */
int mosh2_job_create_multi(mosh2_model *const *models, int32_t n_models, const mosh2_options *opt, int32_t n_seq,
                           const int32_t *frame_counts, const int32_t *model_of_seq, const mosh2_schedule *sched,
                           int32_t precision, mosh2_job **out);
/* obs [F*M*3] metres in latent-label order, vis [F*M] 0/1.  Async on the job's stream. */
int mosh2_job_upload(mosh2_job *j, const double *obs, const uint8_t *vis);
/* Mocap input adapter on the device -- what the reference does per frame in Python between the capture file and the frame
 * loop (tools/mocap_interface.py:186,223-225,254-279 MocapSession / markers_asdict; chmosh.py:582-594).  `markers`: the raw
 * marker table of the file, host memory, [n_file_frames][n_cols][3] float64 in file units; `col_of_marker` [M]: the file
 * column that carries latent marker i's label after the label clean-up (-1: the file has no such label); job frame f is
 * file frame frame_start + f * frame_step; `unit_per_metre` 1000 / 100 / 1 (mocap.unit); `rot3x3`: optional row-major
 * rotation applied before the unit conversion (mocap.rotate), NULL for none.  A sample is missing when a coordinate is NaN
 * or all three are exactly zero.  The table goes through pinned staging to the device, one kernel writes the job's
 * observations (metres, compute precision) and visibility.  Async on the job's stream; replaces mosh2_job_upload. */
int mosh2_job_upload_markers(mosh2_job *j, const double *markers, int32_t n_file_frames, int32_t n_cols, const int32_t *col_of_marker,
                             int32_t frame_start, int32_t frame_step, double unit_per_metre, const double *rot3x3);
/* ... for frames [frame0, frame0 + n) of the job's frame axis only (one capture of a batch job, mosh2_job_create_batch):
 * job frame frame0 + k is file frame frame_start + k * frame_step of this capture's table.  Every call stages its own rows
 * (pinned host memory that is not reused before the call's copy and kernel have finished), so the uploads of a subject's
 * captures can be issued back to back without waiting; the caller's buffers may be freed when the call returns.  Async on
 * the job's stream. */
int mosh2_job_upload_markers_range(mosh2_job *j, int32_t frame0, int32_t n, const double *markers, int32_t n_file_frames, int32_t n_cols,
                                   const int32_t *col_of_marker, int32_t frame_start, int32_t frame_step, double unit_per_metre,
                                   const double *rot3x3);
/* ---- Stage I building block (chmosh.py:83-455; SURVEY.md 8(f-2)) ------------------------------------------------------------
 * Linearise mode: the frames of the job are INDEPENDENT problems (the twelve frames of Stage I), each evaluated by one
 * thread block at a state the caller gives -- x [F][3 + p_red + n_dmpl] = trans | reduced pose | linear coefficients.  The
 * frame's own terms are data, the pose prior (+ joint-angle term) and, with step == 2, the finger term, (optimize_face)
 * the jaw and expression terms and (optimize_dynamics of the job's options, at the job's wt_dmpl) the DMPL term, under opt's
 * wt_data / wt_poseB / wt_poseH / wt_poseF / wt_expr taken as they are (Stage I's annealed weights; no visibility
 * scaling) and opt's optimize_fingers; every other option is the job's (opt may be NULL: the job's weights).  step 1 / 2 picks the
 * free-variable list free1 / free2 of the model description (n columns).  Outputs (host, float64, any pointer may be NULL):
 *   errs [F][8] SSE per term, markers_sim [F][M][3], r [F][3M] weighted data residual (sim - obs) wt_data (0 where invisible),
 *   vp [F][3M][3] posed attachment vertices; with build != 0 also A [F][n][n], g [F][n] (normal equations of the frame's own
 *   terms, g = -J^T r) and J [F][3M][n] (the weighted data rows d r / d x_free).
 * With the shape directions (or, with optimize_face and a given shape, the expression directions) as the model's linear
 * block these are all per-frame quantities the joint shape / latent-marker solve needs (moshpp_b200/stagei.py).  Jobs of
 * one-frame chunks only (chunk_len = 1).  A float32 job rounds x to float32 and computes in float32; its outputs are widened
 * to the float64 buffers.  Synchronous. */
typedef struct mosh2_lin_out {
    double *errs, *markers_sim, *r, *vp, *A, *g, *J;
} mosh2_lin_out;
int mosh2_job_linearize(mosh2_job *j, const mosh2_options *opt, int32_t step, int32_t build, const double *x, const mosh2_lin_out *out);
/* The same from DEVICE memory (e.g. the receive buffer of an NCCL scatter): d_obs [F*M*3] float32 (obs_f64 = 0) or
 * float64 (obs_f64 = 1) on the job's device, d_vis [F*M]; converted to the job's precision on the device.  The
 * copy is ordered after the work already queued on `producer_stream` (a cudaStream_t, may be NULL = legacy stream). */
int mosh2_job_upload_device(mosh2_job *j, const void *d_obs, int32_t obs_f64, const uint8_t *d_vis, void *producer_stream);
/* ... for frames [frame0, frame0 + n) of the job's frame axis only (one sequence of a batch job) */
int mosh2_job_upload_device_range(mosh2_job *j, int32_t frame0, int32_t n, const void *d_obs, int32_t obs_f64,
                                  const uint8_t *d_vis, void *producer_stream);
int mosh2_job_launch(mosh2_job *j);                 /* async; all chunks; clears the result buffers first */
/* Boundary check of the chunked schedule.  Every chunk that does not start at the beginning of its sequence reports the
 * state x = [trans | pose | dmpl] it reached on its LAST warm-up frame and that frame's index (or -1); the emitted result
 * of the same frame was produced by an earlier chunk further along its own history.  Their difference measures what the
 * warm-up left of the cold start, chunk by chunk.  x [n_chunks * (3 + p_red + n_dmpl)], frames [n_chunks]; syncs. */
int mosh2_job_warm_states(mosh2_job *j, double *x, int32_t *frames);
/* The same comparison done on the device: out [n_chunks * 4] = per chunk max |warm-up state - emitted row| over the pose
 * coefficients [0, body_ids), the remaining pose coefficients, the translation, the dmpl / expression coefficients
 * (zeros for chunks that start their sequence).  Queued behind the last launch on the job's stream; syncs. */
int mosh2_job_boundary_deltas(mosh2_job *j, int32_t body_ids, float *out);
/* Re-solves the listed chunks only (e.g. those that failed the boundary check); the rows of all other frames keep the
 * values of the previous launch.  chunk_warmup >= 0: with that warm-up, from a cold start.  chunk_warmup < 0: RESUME --
 * no warm-up; the chunk continues the recursion from the rows the previous launch emitted for the last two solved frames
 * in front of it, exactly as the previous chunk would have gone on (boundary repair); the repair of a chunk stops early once
 * two consecutive re-solved frames lie within merge_tol (rad; translation in 0.1 m) of the rows they replace -- the two
 * trajectories have merged and the remaining rows of the chunk stand (merge_tol = 0: re-solve the whole chunk).
 * root_turns (NULL: 0 for every chunk): per listed chunk, full turns added to the angle of the root its cold start finds (the
 * first-frame alignment returns an angle in [0, pi]).  The sequential pass tracks the root as a free parameter from the first
 * frame on, so after the body has turned past pi its axis-angle root lies beyond pi; a chunk whose cold start lies behind such
 * a crossing must start on that branch, u (theta + 2 pi turns), to solve the sequential pass's problem.  async */
int mosh2_job_relaunch_chunks(mosh2_job *j, int32_t n, const int32_t *chunk_ids, int32_t chunk_warmup, int32_t warmup_full,
                              double merge_tol, const int32_t *root_turns);
int mosh2_job_download(mosh2_job *j, const mosh2_result *res); /* async D2H + stream sync */
int mosh2_job_sync(mosh2_job *j);
/* Results as ONE packed float32 device row per frame, for device-side consumers (NCCL gather): row f =
 * [fullpose 3*n_joints | trans 3 | dmpls n_dmpl | errs 8 | status 1 | jacobian builds 1] (status / builds stored as
 * float values).  d_rows [F * mosh2_job_row_width()] on the job's device; async on the job's stream + stream sync. */
int mosh2_job_row_width(mosh2_job *j);
int mosh2_job_download_device(mosh2_job *j, float *d_rows);
/* device time of the last launch (CUDA events on the job's stream), ms; valid after a sync */
int mosh2_job_kernel_ms(mosh2_job *j, float *ms);
/* device time from the start of `first`'s last launch to the end of `last`'s last launch (jobs of one device that were
 * launched on their own streams at the same time: the span of the whole group is the maximum over all pairs), ms */
int mosh2_job_span_ms(mosh2_job *first, mosh2_job *last, float *ms);
int mosh2_job_num_chunks(mosh2_job *j);
/* out [n_chunks * 2]: first emitted frame and end of the emitted range of every chunk (job frame axis) */
int mosh2_job_chunk_ranges(mosh2_job *j, int32_t *out);
/* work done by the last launch: out8 = {dog-leg iterations, residual evaluations, Jacobian / normal-equation builds,
 * minimisations} over ALL processed frames (warm-up included), then the same four over the EMITTED frames only */
int mosh2_job_totals(mosh2_job *j, int32_t *out8);
void mosh2_job_destroy(mosh2_job *j);

/* upload + launch + download in one call (the call the Python wrapper makes). */
int mosh2_solve(mosh2_model *m, const mosh2_options *opt, int32_t n_frames, const double *obs,
                const uint8_t *vis, const mosh2_schedule *sched, int32_t precision, const mosh2_result *res);

/* ---- Stage-I surface term (SURVEY.md 8(f-2)) --------------------------------------------------------------------------
 * Distance of samples to a triangle mesh with derivatives -- replaces the reference's only native code,
 *   scan2mesh/mesh_distance/sample2meshdist.h:67-207 (plane / edge / vertex distance and gradients under the three
 *   robustifiers), sample2meshdist.pyx:55-103 (`somedistance`: the loop over samples) and the nearest (triangle, part) query
 *   of psbody.mesh's AABB tree (mesh_distance_main.py:346-376).
 * kind: 0 distance, 1 squared distance, 2 Geman-McClure(sigma) of the squared distance.  part: 0 the triangle's plane
 * (signed distance), 1..3 its edges ab / bc / ca, 4..6 its vertices a / b / c.  nearest_tri / nearest_part: both NULL =
 * searched on the device (brute force over all triangles, float32), or both given (what `somedistance` takes).
 * Output arrays may be NULL.  d_tri holds d value / d (a, b, c) of the sample's triangle, 9 numbers per sample. */
typedef struct mosh2_mesh_distance_out {
    double *value;     /* [S]     f(distance)                  */
    int32_t *tri;      /* [S]     nearest triangle             */
    int32_t *part;     /* [S]     nearest part of that triangle */
    double *d_sample;  /* [S * 3] d value / d sample           */
    double *d_tri;     /* [S * 9] d value / d (a, b, c)        */
} mosh2_mesh_distance_out;
int mosh2_mesh_distance(int32_t device, int32_t kind, double sigma, int32_t n_samples, const double *samples, int32_t n_verts,
                        const double *verts, int32_t n_tris, const int32_t *tris, const int32_t *nearest_tri,
                        const int32_t *nearest_part, const mosh2_mesh_distance_out *out, float *kernel_ms);

#ifdef __cplusplus
}
#endif
#endif /* MOSH2_H_ */

/* myo_b200.h -- C-ABI of the B200-native batched musculoskeletal simulator (libmyo_b200.so).
 *
 * Drop-in boundary for ONE hot path of MyoSuite: `env.step` of
 *   myosuite/envs/myo/base_v0.py:82-118  (BaseV0.step)
 * for thousands of parallel envs.  The reference has no FFI seam of its own on this path; what the
 * library semantically replaces is the MuJoCo C API the reference reaches through pybind11:
 *   mj_step      myosuite/robot/robot.py:861
 *   mj_forward   myosuite/robot/robot.py:607,1002 ; envs/env_base.py:91-92
 *   mj_resetData myosuite/robot/robot.py:999
 *   MjSpec.from_file().compile()  myosuite/envs/env_base.py:70-72,96-106
 * plus the per-step Python glue that must run on the device to keep envs resident in HBM:
 *   sigmoid action remap            base_v0.py:86-94
 *   3CC-r fatigue                   envs/myo/fatigue.py:38-76,82-99
 *   frame_skip substeps             robot/robot.py:901-905
 *   obs / reward / done (pose task) envs/myo/myobase/pose_v0.py:100-140
 *   random reset + target sampling  envs/myo/myobase/pose_v0.py:140-170,250-253
 *
 * Conventions: every function returns 0 on success, <0 on error (text via myo_last_error(), thread
 * local).  No exceptions cross the ABI, no torch types appear in it.  All per-env arrays are
 * CALLER-OWNED device buffers (e.g. torch CUDA tensors passed by data_ptr()), contiguous,
 * row-major [n_env, width], on the batch's device, and must outlive the batch.  A batch is
 * single-stream and not re-entrant; distinct batches (one per GPU) are independent; a model is
 * immutable and shareable.  `stream` arguments are `cudaStream_t` passed as void* (NULL = default).
 */
#ifndef MYO_B200_H
#define MYO_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct myo_model myo_model;
typedef struct myo_batch myo_batch;

enum { MYO_TASK_NONE = 0, MYO_TASK_POSE = 1, MYO_TASK_WALK = 2, MYO_TASK_HOLD = 3, MYO_TASK_REACH = 4 };
enum { MYO_COND_NONE = 0, MYO_COND_FATIGUE = 2 };   /* sarcopenia / reafferentation are host-side model edits */

/* model dimensions (mirrors the mjModel sizes the reference reads: env.unwrapped.mj_model.{nq,nv,nu,na}) */
typedef struct {
  int32_t nq, nv, nu, na, nbody, njnt, ntendon, nM;
  int32_t npair;       /* collision candidate pairs evaluated on the device */
  int32_t nta;         /* actuated tendons */
  int32_t maxcon;      /* contact capacity per env */
  int32_t maxefc;      /* constraint-row capacity per env */
  int32_t smem_bytes_per_env;
  int32_t reserved[3];
} myo_dims;

/* task / stepping configuration (registry kwargs of the reference, envs/myo/myobase/__init__.py) */
typedef struct {
  int32_t task;              /* MYO_TASK_* */
  int32_t frame_skip;        /* physics substeps per env step (base_v0.py:27 default 10) */
  int32_t max_episode_steps; /* TimeLimit truncation (registry max_episode_steps) */
  int32_t normalize_act;     /* sigmoid remap of muscle actions (base_v0.py:86-94) */
  int32_t muscle_condition;  /* MYO_COND_* */
  int32_t auto_reset;        /* 1: envs that finish are reset inside the step kernel */
  int32_t reset_random;      /* reset_type="random": pose qpos ~ U(jnt_range); walk keyframe row 0/1 of init_qpos + N(0,0.02) (walk_v0.py:321-337); hold goal/size sampling. 0 = init_qpos */
  int32_t maxcon;            /* 0 = library default */
  int32_t reaf_dst, reaf_src;/* reafferentation (base_v0.py:104-108): ctrl[dst] = ctrl[src]; ctrl[src] = 0 ; dst == src = off */
  int32_t barrier_mode;      /* CTA phase barriers: 0 = before every phase (default), 1 = once per substep, 2 = none, >2 = bit mask of the 8 phases that start with a barrier (tuning knob) */
  int32_t reserved_i;        /* lockstep groups per CTA (tuning knob; 0/1 = the whole CTA is one group) */
  int32_t fatigue_reset;     /* fatigue state at reset (fatigue.py:82-99): 0 = MA 0, MR 1, MF 0 ; 1 = fatigue_reset_random (u1, u2 ~ U(0,1): MA = u1 u2, MR = u1 (1 - u2), MF = 1 - u1) ; 2 = fatigue_reset_vec (MF = vec, MR = 1 - vec, MA = 0) */
  double pose_thd;           /* pose_v0.py:43 */
  double weights[8];         /* reward weights in the task's own key order (pose_v0.py:18-23, walk_v0.py:205-211, obj_hold_v0.py:17-21; reach_v0.py:18-22 as reach, bonus, act_reg, penalty) */
  double solver_tolerance;   /* scaled-gradient stop of the Newton solver; 0 = library default (1e-10) */
  int32_t task_i[16];        /* task-specific indices, filled by the host mirror (vec_env.py): WALK body/joint ids, HOLD object ids, REACH [ntip, tip body x ntip] */
  double task_d[24];         /* task-specific constants: WALK targets / thresholds / torso quaternion offset, HOLD object site, REACH tip-site offsets [3 x ntip] then far_th */
  double reserved[2];        /* [0] != 0 with the phase-cycle tap bound: record the barrier wait before each phase instead of its work (profiling) */
  /* REACH reward shape: reach = c_off - d - c_vel |qvel dt| ; act_reg = -c_act |act|/na ; bonus thresholds near and 2 near with near = ntip near_per_tip.
   * {c_off, c_vel, c_act, near_per_tip}; all zero = reach_v0.py:120-160 (0, 0, 1, 0.0125).  The leg stand task (walk_v0.py:104-140) is (10, 10, 100, 0.05). */
  double reach_shape[4];
  /* REACH reset, when hi > lo: for every joint j, qpos[jnt_qposadr[j]] = clip(init_qpos[.] + U(lo, hi), jnt_range[j]) (walk_v0.py:142-186) */
  double joint_random[2];
} myo_task_cfg;

/* caller-owned device buffers; nullable ones are marked.  f64 state, f32 I/O like the reference
 * (obs cast to float32 in envs/obs_vec_dict.py:83, action space float32 in envs/env_base.py:155). */
typedef struct {
  const float* action;       /* [n, nu]  in  */
  double* qpos;              /* [n, nq]  in/out */
  double* qvel;              /* [n, nv]  in/out */
  double* act;               /* [n, na]  in/out */
  double* qacc_warmstart;    /* [n, nv]  in/out (mjData.qacc_warmstart) */
  double* time;              /* [n]      in/out */
  double* fatigue;           /* [n, 3, nu] MA,MR,MF (nullable unless MYO_COND_FATIGUE) */
  double* target;            /* [n, nq]  pose target_jnt_value, in/out */
  const double* target_range;/* [nq, 2]  per-qpos target sampling range (pose), model-level, in */
  const double* init_qpos;   /* [nq]     reset pose, in ([2,nq] for the walk task with reset_random: the two candidate keyframes) */
  const double* init_qvel;   /* [nv]     reset velocity (nullable = zeros), in ([2,nv] alongside a [2,nq] init_qpos) */
  double* env_prm;           /* [n, 8]   per-env model overrides (HOLD: goal site pos[3], object geom size[3]); nullable */
  int32_t* step_count;       /* [n] */
  int64_t* episode_count;    /* [n]  also the Philox stream counter */
  float* obs;                /* [n, obs_dim] out */
  float* reward;             /* [n] out (rwd_dense) */
  uint8_t* done;             /* [n] out (terminated) */
  uint8_t* truncated;        /* [n] out (TimeLimit) */
  float* ep_return;          /* [n] running return of the current episode */
  float* last_return;        /* [n] return of the most recently finished episode */
  /* parity taps, all nullable: values of the LAST substep's forward pass (pre-integration state) */
  double* tap_qacc;          /* [n, nv] */
  double* tap_actuator_force;/* [n, nu] */
  double* tap_ten_length;    /* [n, nta] actuator_length order */
  double* tap_qfrc_smooth;   /* [n, nv] */
  int32_t* tap_ncon;         /* [n, 4]: ncon, nefc, newton iterations, overflow flag */
  int32_t* tap_contact_pair; /* [n, maxcon] program pair index of each contact, -1 padded */
  double* tap_contact_dist;  /* [n, maxcon] */
  double* tap_moment;        /* [n, nnz] structural non-zeros of the tendon moment */
  double* tap_qM;            /* [n, nM] */
  long long* tap_phase_cycles; /* [n, 20] SM-clock cycles per phase over the call (profiling aid; 8-11 solver parts, 12,13: max ncon / nefc, 14,15: Newton iterations / dense ones, 16: cooperative collision, 17: load..substeps) */
  const double* fatigue_reset_vec; /* [nu] nullable unless cfg.fatigue_reset == 2: the reference's fatigue_reset_vec (base_v0.py:29,48; fatigue.py:90-94) */
  int32_t* overflow;         /* [n] nullable: sticky flag, set when a substep of this env dropped contacts (more than maxcon, or more ellipsoid candidates than the list holds); cleared by the env's reset */
} myo_buffers;

const char* myo_last_error(void);
int myo_version(void);

/* Model from the packed blob produced by myosuite_b200.blob.pack (host arrays; copied).
 * Replaces: MjSpec.from_file(path).compile() + the model upload.  */
int myo_model_from_blob(const int32_t* I, int64_t nI, const double* D, int64_t nD, myo_model** out);
int myo_model_dims(const myo_model* m, const myo_task_cfg* cfg_or_null, myo_dims* out);
void myo_model_destroy(myo_model* m);

/* Batch of n_env envs of one model on one device. */
int myo_batch_create(const myo_model* m, int device, int n_env, const myo_task_cfg* cfg, myo_batch** out);
int myo_batch_bind(myo_batch* b, const myo_buffers* bufs);
void myo_batch_destroy(myo_batch* b);
int myo_batch_obs_dim(const myo_batch* b);

/* Reset envs whose mask byte is non-zero (mask == NULL: all).  Per-env Philox streams keyed
 * (seed, env_offset + env, episode_count).  Replaces env.reset() (pose_v0.py:174-257, robot.py:996-1002). */
int myo_batch_reset(myo_batch* b, const uint8_t* mask_dev_or_null, uint64_t seed, int64_t env_offset, void* stream);

/* One control step for every env: action->ctrl, [fatigue], frame_skip x (forward + Euler), obs,
 * reward, done, TimeLimit, optional auto-reset.  Asynchronous on `stream`.
 * Replaces BaseV0.step (base_v0.py:82-118) for the whole batch. */
int myo_batch_step(myo_batch* b, void* stream);

/* obs / reward / done of the CURRENT state without advancing it.
 * Replaces env.forward() (envs/env_base.py:393-432). */
int myo_batch_observe(myo_batch* b, void* stream);

/* Parity tap: ONE forward pass (mj_forward) on the bound qpos/qvel/act with ctrl := action taken
 * verbatim (no sigmoid), writing the tap_* buffers; state is not advanced.  If n_substeps > 0 the
 * state IS advanced by that many mj_step's with the same ctrl (taps hold the last forward). */
int myo_batch_forward_debug(myo_batch* b, const double* ctrl_dev /* [n, nu] */, int n_substeps, void* stream);

/* number of kernel launches issued by this batch so far (bench.py's gpu_launches claim) */
int64_t myo_batch_launch_count(const myo_batch* b);

/* Read-only queries of how env steps are launched (for tests of the product kernels at their real launch shapes).
 * launch_info writes the first min(n, 8) of: use_w14 (1: the launch_bounds(448) kernel, 0: launch_bounds(320)), warps_per_cta,
 * grid, rounds of warps each CTA walks, regroup (1: load-sorted slot -> env map), balanced (1: env e on CTA e % grid when not
 * regrouped, 0: contiguous groups of warps), smem_bytes, perm_slots (entries of the slot -> env map, 0 without regroup).
 * debug_perm copies the slot -> env map of the last env step to HOST memory (n >= perm_slots entries; slot
 * cta + grid*(round*warps_per_cta + warp), -1 = idle slot); it synchronises the device and fails when regroup is off or no step has run. */
int myo_batch_launch_info(const myo_batch* b, int32_t* out, int n);
int myo_batch_debug_perm(const myo_batch* b, int32_t* host_out, int n);

/* Unit-test hook for the dense solver the Newton and integrator phases use: solves H x = b for `count` independent SPD systems
 * (H_host: count x n(n+1)/2 packed lower triangles, row-major; x_host: count x n, rhs in / solution out; HOST pointers), one
 * warp per system (row-in-registers / column-through-shared-memory L D L' for n <= 32, bordered register Cholesky for 32 < n <= 36, shared-memory
 * fallback above).  `mode` is ignored (kept for ABI stability).  n <= 64. */
int myo_debug_chol_solve(int device, const double* H_host, double* x_host, int n, int count, int mode);

#ifdef __cplusplus
}
#endif
#endif

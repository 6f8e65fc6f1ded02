/* llq.h -- C-ABI of the batched legged-quadruped rollout engine ("llq").
 *
 * This is the drop-in boundary for the hot path named in BASELINE.json: the
 * TLeague actor's env.reset()/env.step() on the reference's PyBullet envs.
 * The reference has no FFI of its own for this path (it is pure Python over the
 * pybullet wheel), so every entry point cites the reference Python interface it
 * replaces.  Citations are relative to /root/reference/src/lifelike/sim_envs/pybullet_envs/:
 *   LR  = legged_robot/legged_robot.py
 *   PLE = primitive_level_env/primitive_level_env.py
 *   ML  = primitive_level_env/motion_lib.py
 *   CPE = create_pybullet_envs.py
 *
 * Two shared libraries implement this header with identical semantics:
 *   oracle/libllq_cpu.so                                  fp64 CPU restatement (test oracle only)
 *   lifelike_agility_and_play_b200/csrc/libllq_cuda.so    fp32 sm_90a CUDA engine (the product)
 *
 * Conventions: plain C types only; all array arguments are caller-owned;
 * every function returns 0 on success and a negative LLQ_E* code on failure,
 * never aborts; llq_last_error() gives a human-readable message for the last
 * failure on the calling thread.  A handle is single-owner and not re-entrant;
 * several handles (one per GPU) may coexist in one process.
 */
#ifndef LLQ_H
#define LLQ_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LLQ_ABI_VERSION 4

/* per-env sizes (PMC env, reference PLE:102-124 with the shipped prop_type) */
#define LLQ_STATE_DIM   37   /* base_pos3 base_orn4(xyzw) base_lin_vel3 base_ang_vel3 joint_pos12 joint_vel12 (LR:86-106) */
#define LLQ_ACTION_DIM  12   /* residual joint-position targets (PLE:198-200) */
#define LLQ_PROP_DIM    33   /* joint_pos12 joint_vel12 ang_vel_loc3 lin_vel_loc3 e_g3 (PLE:247-260) */
#define LLQ_OBS_DIM     207  /* prop 3x33 | prop_a 3x12 | future 4x18 (PLE:117-121,276-297) */
#define LLQ_MOCAP_FRAME 19   /* x y z qx qy qz qw + 12 joint angles (ML:88-96) */
#define LLQ_OBS_DIM_EPMC 916 /* prop 99 | prop_a 36 | percep_2d 25x13 | percep_1d 128 | percep_front 25x13 | target 3
                                (max_game_elements/playground_env.py:129-144) */
#define LLQ_ENV_PMC  0       /* PrimitiveLevelEnv  (primitive_level_env.py) */
#define LLQ_ENV_EPMC 1       /* PlayGroundEnv, element_id 0 = flat-ground joystick task, the shipped script default
                                (max_game_elements/playground_env.py, train_scripts/example_epmc_train.sh:100) */
#define LLQ_OBS_DIM_SEPMC 965 /* per agent: prop 99 | prop_a 36 | percept_2d 325 | percept_1d 128 | percept_front 325 | percept_vec 5 |
                                 oppo_info 15 | oppo_info_cheat 15 | flag_info 7 | flag_info_cheat 7 | with_flag 2 | control_spd 1
                                 (max_game/chase_tag_game_env.py:111-124) */
#define LLQ_ENV_SEPMC 2      /* ChaseTagGameEnv in the empty arena of the shipped config (max_game/chase_tag_game_env.py,
                                train_scripts/example_sepmc_train.sh:113-116).  n_envs counts ROBOTS and must be even: robots 2p and
                                2p+1 form env-pair p; actions / obs / reward / done are per robot (done is the pair's, on both rows). */
#define LLQ_AUX_DIM  18      /* columns of LLQ_F_AUX, the EPMC / SEPMC bookkeeping; slots: */
/* shared by EPMC and SEPMC */
#define LLQ_AUX_COUNTER        0   /* env steps of the episode */
#define LLQ_AUX_TOTAL_SPD      7   /* sum of the per-step speeds */
#define LLQ_AUX_MAX_SPD        8   /* largest per-step speed */
#define LLQ_AUX_PUSH_COUNT     9   /* push randomiser sub-step counter (PR:56-87) */
#define LLQ_AUX_PUSH_F        10   /* last applied push force x; y and z in slots 11 and 12 */
#define LLQ_AUX_FOOT_FRICTION 13   /* per-episode foot lateral friction (PGE:209) */
#define LLQ_AUX_PUSH_DRAWS    14   /* push-randomiser draws taken (SEPMC: the pair's) */
#define LLQ_AUX_YAW_ACCUM_DEG 16   /* running reset yaw: the reference mutates its module-level init-state dict (PGE:181-189; SEPMC: the pair's) */
/* EPMC */
#define LLQ_AUX_CMD_FREQ           1   /* cmd_vary_freq (PGE:170,223) */
#define LLQ_AUX_TARGET_X           2
#define LLQ_AUX_TARGET_Y           3
#define LLQ_AUX_TARGET_SPD         4
#define LLQ_AUX_TARGET_ANGLE       5
#define LLQ_AUX_LAST_POS_DIFF_LEN  6
#define LLQ_AUX_CMD_DRAWS         15   /* joystick-command draws taken */
#define LLQ_AUX_INIT_POS_DIFF_LEN 17   /* elements 1-3 (PGE:192-195) */
/* SEPMC */
#define LLQ_AUX_WITH_FLAG     1
#define LLQ_AUX_FLAG_X        2
#define LLQ_AUX_FLAG_Y        3
#define LLQ_AUX_CONTROL_SPD   4
#define LLQ_AUX_OPPO_VISIBLE  5
#define LLQ_AUX_SWITCH_FLAG   6
#define LLQ_AUX_FLAG_DRAWS   15
#define LLQ_AUX_FLAG_TOUCH   17   /* this robot's body touched the flag in the last sub-step: the stale manifold reset() sees (CTG:302,573) */
#define LLQ_NUM_FEET    4

/* error codes */
#define LLQ_OK            0
#define LLQ_EINVAL      (-1)
#define LLQ_ENOMEM      (-2)
#define LLQ_ECUDA       (-3)
#define LLQ_ESTATE      (-4)  /* call order violated (e.g. step before load_model / load_mocap / reset) */
#define LLQ_EUNSUPPORTED (-5)

/* pointer-space flags for llq_step_ex / llq_reset_ex */
#define LLQ_IO_HOST    0   /* pointers are host memory (pageable or pinned); copies happen inside the call */
#define LLQ_IO_DEVICE  1   /* pointers are device memory on the handle's GPU; no host round trip, no sync */
#define LLQ_IO_PINNED  2   /* pointers are page-locked host memory (llq_host_alloc / cudaHostAlloc / cudaHostRegister): the copies
                              go straight between the caller's buffers and the device, no staging memcpy; synchronous like HOST */

/* field ids for llq_get_field / llq_set_field (host pointers, row-major, [n_envs, width]) */
#define LLQ_F_STATE       0  /* float   [N,37]  robot state, pybullet base-inertial-frame convention (LR:86-106) */
#define LLQ_F_CLIP        1  /* int32   [N]     sampled mocap clip id (ML:59-63) */
#define LLQ_F_TIME        2  /* double  [N]     env clock PLE.time (PLE:208-210,271) */
#define LLQ_F_REWARD_SUM  3  /* float   [N]     PLE.reward_sum (PLE:231) */
#define LLQ_F_EPISODE_STEPS 4 /* int32  [N]     PLE._episode_steps (PLE:197) */
#define LLQ_MAX_SPHERES   32 /* collision spheres of the robot: 4 feet, 4 knee wheels, 4 hips, 4 thighs, 8 shank, 8 trunk corners */
#define LLQ_MAX_CONTACTS  8  /* manifold points kept per robot and sub-step (sphere order); counter LLQ_CNT_DROPPED counts what was dropped */
#define LLQ_MAX_LIMIT_ROWS 8 /* joint-limit rows kept per robot and sub-step (joint order) */
#define LLQ_F_WARMSTART   5  /* float   [N,32]  previous sub-step's normal impulse per collision sphere (contact warm start) */
#define LLQ_F_OBS         6  /* float   [N,207] last observation (carries the 3-frame prop / action history) */
#define LLQ_F_KIN_STATE   7  /* float   [N,37]  kinematic (mocap) robot state (PLE:217-218) -- get only */
#define LLQ_F_SAMPLE_PROB 8  /* double  [n_clips] prioritized sampling probabilities (PLE:239-240) */
#define LLQ_F_AVG_REWARD  9  /* double  [n_clips] PLE._avg_reward_sum (PLE:236) */
#define LLQ_F_EPISODE_ID  10 /* int64   [N]     per-env episode counter (RNG stream position).  SEPMC: robot 0's id keys every
                                                   draw of its pair, and a reset writes robot 0's id + 1 to both robots; unequal ids
                                                   in a pair are accepted, robot 1's is ignored */
#define LLQ_F_FOOT_POS    11 /* float   [N,12]  world positions of the 4 foot links after the last step (LR:199-205) -- get only */
#define LLQ_F_AUX         13 /* double  [N,18]  EPMC bookkeeping (LLQ_AUX_DIM): counters, joystick target, push randomiser, friction */
#define LLQ_F_OB_ID       14 /* int32   [N]     PMC hurdle: index of the active plate within the clip's plate list (PLE:179,264-265) */
#define LLQ_MAX_BOXES     36 /* static boxes of one EPMC corridor: 2 walls + up to 32 cubes / 18 hurdles / 18 bars (BSE:205-243) */
#define LLQ_F_BOXES       15 /* float   [N,36,6] centre xyz, half extents xyz of the env's static boxes (walls first) -- get only */
#define LLQ_F_NBOX        16 /* int32   [N]      number of valid boxes */
#define LLQ_F_DECISION_MARGIN 12 /* float [N]   CPU oracle only, get only: smallest distance to a discontinuous branch taken during
                                   the last step: min(|q-limit|) over joints [rad], min(|dist-contact_breaking|) over the collision spheres [m], and -- where a
                                   sphere touches two statics at once -- the depth difference that decides which one owns its manifold point [m];
                                   under knee_contacts = 1, where a leg's foot and knee wheel both touch, their depth difference (the deeper one is kept) [m].
                                   Parity tests use it to tell rounding noise from a flipped joint-limit / contact decision. */

typedef struct llq_config {
  int32_t struct_size;        /* = sizeof(llq_config), for ABI checking */
  int32_t n_envs;             /* environments stepped in lock-step by this handle */
  int32_t device;             /* CUDA device ordinal (ignored by the CPU oracle) */
  int32_t substeps;           /* physics sub-steps per env step: int(policy_step/time_step) = 10 (PLE:52) */
  int32_t solver_iters;       /* PGS iterations, numSolverIterations=10 (LR:261) */
  int32_t auto_reset;         /* 1: envs that finish are re-sampled inside llq_step (vector-env convention) */
  int32_t num_threads;        /* CPU oracle: OpenMP threads over envs (0 = all cores); ignored by CUDA */
  int32_t element_id;         /* EPMC (PGE:199-206): 0 flat joystick arena, 1 hurdles, 2 'holes' (bars to pass under), 3 cubes (easy) */
  int64_t global_env_offset;  /* global id of env 0 (RNG streams are keyed by global id => result independent of sharding) */
  uint64_t seed;
  double sim_dt;              /* 1/sim_freq = 0.002 (PLE:49) */
  double kp, kd, max_tau;     /* PD gains and torque clip (LR:138-141; train cfg 50, 0.5, 18) */
  double gravity_z;           /* -9.80665 (LR:260) */
  double ground_friction;     /* plane.urdf lateral_friction 0.9 (legged_robot/data/urdf/plane.urdf:5) */
  double foot_friction;       /* foot_lateral_friction 0.5 (LR:304-308) */
  double contact_erp;         /* Bullet m_erp2 as set by pybullet */
  double joint_erp;           /* Bullet m_erp (joint-limit rows) */
  double linear_slop;         /* Bullet m_linearSlop as set by pybullet (1e-5) */
  double warmstart;           /* Bullet m_warmstartingFactor as set by pybullet (0.1) */
  double contact_breaking;    /* relative contact breaking threshold: 0.02 * sphere radius */
  double lin_damping;         /* btMultiBody m_linearDamping 0.04 */
  double ang_damping;         /* btMultiBody m_angularDamping 0.04 */
  double max_coord_vel;       /* btMultiBody m_maxCoordinateVelocity 100 */
  double max_applied_impulse; /* btMultiBody m_maxAppliedImpulse 1000 (joint-limit rows) */
  double w_joint_pos, w_joint_vel, w_end_effector, w_root_pose, w_root_vel; /* reward weights (PLE:352-370) */
  double prioritized_sample_factor; /* (PLE:136,239) */
  double policy_dt;           /* 1/control_freq = 0.02 (PLE:47) -- used for MotionLib margin / max_steps (ML:35,45) */
  /* ---- environmental level (LLQ_ENV_EPMC); PGE = max_game_elements/playground_env.py, PR = randomizer/push_randomizer.py */
  int32_t env_kind;           /* LLQ_ENV_PMC / LLQ_ENV_EPMC */
  int32_t max_steps;          /* episode length cap, 1000 (PGE:66,364) */
  int32_t cmd_freq_lo, cmd_freq_hi;   /* cmd_vary_freq ~ randint(lo, hi) (PGE:170,223) */
  int32_t push_start_count;   /* -start_time // time_step  = -250 (PR:53)   -- computed by the host with Python float floor division */
  int32_t push_interval_steps;/* interval_time // time_step = 499  (PR:46) */
  int32_t push_duration_steps;/* duration_time // time_step = 100  (PR:45) */
  int32_t push_enabled;       /* 'disturb_force_config' present (PGE:155-158) */
  double friction_lo, friction_hi;    /* per-episode foot lateral friction ~ U (PGE:209) */
  double push_h_lo, push_h_hi, push_v_lo, push_v_hi;   /* horizontal / vertical push force ranges (PR:89-99) */
  double target_spd_lo, target_spd_hi;                 /* target_spd_range (PGE:317) */
  /* EPMC elements 1-3: corridor of max_game_elements/bullet_static_entities.py (BSE) */
  double wall_width_lo, wall_width_hi;                 /* PGE:160: [0.02, 0.5]  (BSE:171) */
  double wall_gap_lo, wall_gap_hi;                     /* PGE:161: [1.0, 20.0]  (BSE:174) */
  double hole_gap_lo, hole_gap_hi;                     /* hole_config min/max_gap_height (BSE:372-373; shipped 0.25, 0.25) */
  /* ---- which collision shapes of the robot touch the statics (the reference loads every link with its geometry, LR:212-217):
     0 = the four foot spheres only;
     1 = + the knee wheels (link_*W, cylinders r = 0.028 / 0.036 on the thigh links, as spheres), ONE contact per leg = the deeper
         of {foot, knee wheel} -- the round-1 model, kept selectable;
     2 = (default) every collision sphere of the model blob, each with its own manifold point: feet, knee wheels, hips, thighs,
         shanks, trunk-box corners, against ground, arena walls and corridor boxes (at most LLQ_MAX_CONTACTS per robot).
     Without the knee wheels the shipped Bullet-trained policy falls in 57 % of its episodes (tools/statistical_pin.py, DESIGN.md 6). */
  int32_t knee_contacts;
  int32_t reserved1;
  double link_friction;       /* lateral friction of links without a changeDynamics() call: Bullet's default 0.5 */
  double auxiliary_radius;    /* EPMC elements 1-3: radius of the two auxiliary cylinders the reference lays along the front / back top
                                 edges of every hurdle and cube and along the bottom edges of every bar (BSE:43-104, 360-362, 418-420,
                                 451-453; env_randomize_config['auxiliary_radius'], shipped 0.02).  They collide with the robot and are
                                 invisible to rays.  0 = none. */
} llq_config;

typedef struct llq_engine* llq_handle;

/* ABI / build info: returns LLQ_ABI_VERSION; *is_cuda = 1 for the CUDA engine, 0 for the CPU oracle. */
int llq_abi_version(int* is_cuda);

/* Fill cfg with the reference's training configuration (train_scripts/example_pmc_train.sh:67-79,
 * PLE:27-43 defaults, Bullet/pybullet solver defaults of SURVEY appendix A). */
int llq_default_config(llq_config* cfg);

/* Replaces: PrimitiveLevelEnv.__init__ (PLE:27-148) -- allocate an engine for cfg->n_envs environments. */
int llq_create(const llq_config* cfg, llq_handle* out);

/* Replaces: PrimitiveLevelEnv.close (PLE:428-431). */
int llq_destroy(llq_handle h);

/* Observation row width of this handle: LLQ_OBS_DIM (PMC) or LLQ_OBS_DIM_EPMC. */
int llq_obs_dim(llq_handle h);

/* EPMC only. Replaces LeggedRobot.get_init_states_info (LR:115-117): the 37-float state every episode starts from
 * (utils/constants.py:103-116 STATES_INFO_12_RUN_0) before the random yaw and z = 0.5 of PGE:181-189 are applied. */
int llq_set_init_state(llq_handle h, const double* state37);

/* Replaces: LeggedRobot._init_dynamic_model / loadURDF (LR:207-264).  blob: float64 table produced by
 * model/compile_model.py, layout in llq_model_layout.h. */
int llq_load_model(llq_handle h, const double* blob, int64_t n_doubles);

/* Replaces: MotionLib._open_all_mocap_datas (ML:19-46).  frames: [total_frames,19] float64 (clips back to
 * back, file order = sorted names), clip_offsets: [n_clips+1] prefix offsets, frame_dt = "FrameDuration".
 * Every clip needs at least margin + 3 frames (margin = ceil(policy_dt / frame_dt) + 1 / frame_dt + 2).
 * Clip limit (CUDA engine): the reset kernel keeps the prioritized clip table in shared memory, 8 B per clip beside its static
 * tables, so n_clips <= (cudaDevAttrMaxSharedMemoryPerBlockOptin - static shared memory of the reset kernel) / 8: 26,814 clips on an
 * H100.  A larger table is refused with LLQ_EINVAL and a message naming the limit; the handle keeps its previous table.  The CPU
 * oracle has no limit. */
int llq_load_mocap(llq_handle h, const double* frames, const int32_t* clip_offsets, int32_t n_clips, double frame_dt);

/* Replaces: MotionLib.obstacles_info + PrimitiveLevelEnv._create_obstacle / _update_obstacle (ML:38-42, PLE:173-193,262-268,
 * utils/obstacle.py:6-33) -- set_obstacle=True.  table: [total,4] float64 rows (apex time [s], x, y, yaw) of every clip's
 * hurdle plates back to back, offsets: [n_clips+1]; half extents of the plate (PLE:184: 0.025, 0.5, obstacle_height).
 * An episode ends when the robot touches the active plate (PLE:341-346).  Contact is evaluated on the poses of the last
 * sub-step (what getContactPoints reports after stepSimulation) with detection proxies: foot / wheel / hip spheres and the
 * body box corners -- a coarse stand-in for Bullet's exact link shapes; the plate exerts no force (the episode ends anyway).
 * Must be called after llq_load_mocap. */
int llq_load_obstacles(llq_handle h, const double* table, const int32_t* offsets, int32_t n_clips, double half_x, double half_y,
                       double half_z);

/* Replaces: PrimitiveLevelEnv.reset (PLE:150-171) for every env with mask[i] != 0 (mask == NULL: all).
 * Clip ~ prioritized_sample_probability, phase ~ U(0,1) (ML:48-63), drawn from Philox4x32-10 keyed by
 * (seed, global env id, episode counter).  obs (nullable): [N,207] host buffer receiving the reset obs. */
int llq_reset(llq_handle h, const uint8_t* mask, float* obs);

/* Deterministic variant used by tests and by the gym adaptor's "reset to clip/time": same as llq_reset but
 * clip[i] / time[i] are given instead of sampled (ML:50-57 with sampled_time = time[i]). */
int llq_reset_to(llq_handle h, const uint8_t* mask, const int32_t* clip, const double* time, float* obs);

/* Replaces: PrimitiveLevelEnv.step (PLE:195-245) for all envs, minus the real-time sleep (PLE:241-244).
 * actions [N,12] -> obs [N,207], reward [N], done [N].  Host pointers; H2D/D2H copies are inside the call. */
int llq_step(llq_handle h, const float* actions, float* obs, float* reward, uint8_t* done);

/* Same, with explicit pointer space, observation row stride (floats, >= 207; lets the engine write straight
 * into a [T,N,ld] trajectory slab) and, for LLQ_IO_DEVICE, the CUDA stream (cudaStream_t as void*, NULL =
 * the handle's own stream) on which the step is enqueued without synchronising. Any of obs/reward/done may be
 * NULL. */
int llq_step_ex(llq_handle h, const float* actions, float* obs, int64_t obs_ld, float* reward, uint8_t* done,
                int io_mode, void* stream);

/* State access for parity tests and checkpoint/resume (replaces LR.get_states_info / set_states_info,
 * LR:62-113, and the env bookkeeping fields).  Host pointers. */
int llq_get_field(llq_handle h, int field, void* dst);
int llq_set_field(llq_handle h, int field, const void* src);

/* counters: out[LLQ_CNT_*] below, n <= 8. */
#define LLQ_CNT_ENV_STEPS     0   /* env steps */
#define LLQ_CNT_EPISODES      1   /* episodes finished */
#define LLQ_CNT_CONTACT_ROWS  2   /* contact rows solved */
#define LLQ_CNT_LIMIT_ROWS    3   /* joint-limit rows solved */
#define LLQ_CNT_LAUNCHES      4   /* kernel launches issued by the engine (CUDA) / 0 (CPU) */
#define LLQ_CNT_DROPPED       5   /* manifold points / limit rows dropped by the LLQ_MAX_CONTACTS / LLQ_MAX_LIMIT_ROWS caps */
int llq_get_counters(llq_handle h, int64_t* out, int32_t n);

/* Per-kernel device timing of the most recent llq_step*: out[0] = fused step kernel ms, out[1] = reset/table kernel ms
 * (CUDA events on the launching stream; valid after llq_sync).  Enabled by llq_set_option(h, "profile", 1).
 * Other options: "record" = 1: the step kernel also writes action 12 | reward | done behind the observation of the slab row it is handed
 * (obs_ld >= observation width + 14; SURVEY 8e: no column copies after the step), 2: into the slab row before it (the [T+1, N, ld]
 * layout of parallel/rollout.py).  The CPU oracle returns LLQ_EUNSUPPORTED. */
int llq_set_option(llq_handle h, const char* name, double value);
int llq_get_timing(llq_handle h, double* out, int32_t n);

/* Page-locked host buffers for LLQ_IO_PINNED (plain malloc/free in the CPU oracle). */
int llq_host_alloc(void** out, int64_t bytes);
int llq_host_free(void* p);

/* Block until all work enqueued by this handle has finished (no-op for the CPU oracle). */
int llq_sync(llq_handle h);

const char* llq_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* LLQ_H */

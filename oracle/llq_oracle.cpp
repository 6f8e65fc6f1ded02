// llq_oracle.cpp -- CPU restatement ("oracle") of the reference env.step() hot path.
//
//  *** TEST INFRASTRUCTURE ONLY ***  Only tests/, __graft_entry__.smoke() and bench.py's
//  cpu_baseline / --impl reference legs may load libllq_cpu.so.  The product path
//  (lifelike_agility_and_play_b200/) never links, imports or calls anything in oracle/.
//
//  PARITY STATUS: the *environment logic* (mocap interpolation, observation, reward,
//  termination, clocks, sampling) is pinned against the reference's own Python code run in
//  this container (tests/golden/gen_golden_from_reference.py imports MotionLib /
//  PrimitiveLevelEnv from /root/reference with pybullet replaced by a shim).  The *physics*
//  (Bullet btMultiBody step) is "parity unpinned": PyBullet/Bullet3 is an un-vendored,
//  un-pinned dependency (setup.py:20) that is absent from /root/reference and from this
//  image, and the reference's tests hold no golden vectors (SURVEY.md 4, 8c).  The physics
//  below restates Bullet's published algorithm as listed in SURVEY.md appendix A.
//
//  fp64 throughout; one environment at a time; OpenMP over environments.
//  Citations: LR/PLE/ML/CPE as in include/llq.h.
//
//  Formulation (deliberately different from the CUDA engine so that the two cross-check):
//  generic kinematic tree read from the model blob (23 links, fixed joints kept as 0-dof
//  links like Bullet without URDF_MERGE_FIXED_LINKS), spatial quantities in each link's
//  inertial (CoM, principal-axes) frame, dense 6x6 articulated inertias, generalized
//  velocity (omega_world, v_world, qdot) exactly as btMultiBody stores it.
#include "../include/llq.h"
#include "../include/llq_model_layout.h"

#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>
#ifdef _OPENMP
#include <omp.h>
#endif

namespace {

thread_local std::string g_err;
int fail(int code, const std::string& msg) { g_err = msg; return code; }

// ------------------------------------------------------------------ small linear algebra
struct V3 { double x, y, z; };
struct M3 { double m[3][3]; };
inline V3 operator+(V3 a, V3 b) { return {a.x + b.x, a.y + b.y, a.z + b.z}; }
inline V3 operator-(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
inline V3 operator*(double s, V3 a) { return {s * a.x, s * a.y, s * a.z}; }
inline double dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
inline V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
inline double norm(V3 a) { return std::sqrt(dot(a, a)); }
inline V3 mul(const M3& A, V3 v) {
  return {A.m[0][0] * v.x + A.m[0][1] * v.y + A.m[0][2] * v.z, A.m[1][0] * v.x + A.m[1][1] * v.y + A.m[1][2] * v.z,
          A.m[2][0] * v.x + A.m[2][1] * v.y + A.m[2][2] * v.z};
}
inline V3 tmul(const M3& A, V3 v) {  // A^T v
  return {A.m[0][0] * v.x + A.m[1][0] * v.y + A.m[2][0] * v.z, A.m[0][1] * v.x + A.m[1][1] * v.y + A.m[2][1] * v.z,
          A.m[0][2] * v.x + A.m[1][2] * v.y + A.m[2][2] * v.z};
}
inline M3 mul(const M3& A, const M3& B) {
  M3 C;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C.m[i][j] = A.m[i][0] * B.m[0][j] + A.m[i][1] * B.m[1][j] + A.m[i][2] * B.m[2][j];
  return C;
}
inline M3 transpose(const M3& A) {
  M3 C;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C.m[i][j] = A.m[j][i];
  return C;
}
inline M3 ident() { return {{{1, 0, 0}, {0, 1, 0}, {0, 0, 1}}}; }
inline M3 from9(const double* p) {
  M3 A;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) A.m[i][j] = p[3 * i + j];
  return A;
}
inline M3 axis_angle(V3 a, double q) {  // Rodrigues, |a| = 1
  double c = std::cos(q), s = std::sin(q), t = 1 - c;
  return {{{t * a.x * a.x + c, t * a.x * a.y - s * a.z, t * a.x * a.z + s * a.y},
           {t * a.x * a.y + s * a.z, t * a.y * a.y + c, t * a.y * a.z - s * a.x},
           {t * a.x * a.z - s * a.y, t * a.y * a.z + s * a.x, t * a.z * a.z + c}}};
}

// quaternions are (x, y, z, w), scalar last, as scipy / pybullet (SURVEY A.4)
struct Q4 { double x, y, z, w; };
inline Q4 qnormalize(Q4 q) {
  double n = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
  return {q.x / n, q.y / n, q.z / n, q.w / n};
}
inline Q4 qmul(Q4 a, Q4 b) {  // Hamilton product; scipy R1*R2 == qmul(q1, q2)
  return {a.w * b.x + a.x * b.w + a.y * b.z - a.z * b.y, a.w * b.y - a.x * b.z + a.y * b.w + a.z * b.x,
          a.w * b.z + a.x * b.y - a.y * b.x + a.z * b.w, a.w * b.w - a.x * b.x - a.y * b.y - a.z * b.z};
}
inline Q4 qconj(Q4 q) { return {-q.x, -q.y, -q.z, q.w}; }
inline M3 qmat(Q4 q) {  // scipy Rotation.from_quat(q).as_matrix(), q unit
  double x = q.x, y = q.y, z = q.z, w = q.w;
  return {{{1 - 2 * (y * y + z * z), 2 * (x * y - z * w), 2 * (x * z + y * w)},
           {2 * (x * y + z * w), 1 - 2 * (x * x + z * z), 2 * (y * z - x * w)},
           {2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)}}};
}
// scipy Rotation.as_rotvec: angle in [0, pi]
inline V3 q_rotvec(Q4 q) {
  if (q.w < 0) q = {-q.x, -q.y, -q.z, -q.w};
  double s = std::sqrt(q.x * q.x + q.y * q.y + q.z * q.z);
  double angle = 2 * std::atan2(s, q.w);
  double scale;
  if (angle <= 1e-3) {
    double a2 = angle * angle;
    scale = 2 + a2 / 12 + 7 * a2 * a2 / 2880;
  } else {
    scale = angle / std::sin(angle / 2);
  }
  return {scale * q.x, scale * q.y, scale * q.z};
}
// scipy Rotation.from_rotvec
inline Q4 rotvec_q(V3 r) {
  double angle = norm(r), scale;
  if (angle <= 1e-3) {
    double a2 = angle * angle;
    scale = 0.5 - a2 / 48 + a2 * a2 / 3840;
  } else {
    scale = std::sin(angle / 2) / angle;
  }
  return {scale * r.x, scale * r.y, scale * r.z, std::cos(angle / 2)};
}

// ------------------------------------------------------------------ 6-vectors / 6x6 (angular first)
struct S6 { double v[6]; };
struct M6 { double m[6][6]; };
inline S6 s6(V3 a, V3 l) { return {{a.x, a.y, a.z, l.x, l.y, l.z}}; }
inline V3 ang(const S6& s) { return {s.v[0], s.v[1], s.v[2]}; }
inline V3 lin(const S6& s) { return {s.v[3], s.v[4], s.v[5]}; }
inline double dot6(const S6& a, const S6& b) {
  double r = 0;
  for (int i = 0; i < 6; i++) r += a.v[i] * b.v[i];
  return r;
}
inline S6 mul6(const M6& A, const S6& x) {
  S6 y;
  for (int i = 0; i < 6; i++) {
    double r = 0;
    for (int j = 0; j < 6; j++) r += A.m[i][j] * x.v[j];
    y.v[i] = r;
  }
  return y;
}
inline S6 tmul6(const M6& A, const S6& x) {  // A^T x
  S6 y;
  for (int i = 0; i < 6; i++) {
    double r = 0;
    for (int j = 0; j < 6; j++) r += A.m[j][i] * x.v[j];
    y.v[i] = r;
  }
  return y;
}
// motion transform parent(CoM frame) -> child(CoM frame): ang_c = R ang_p ; lin_c = R lin_p - r x (R ang_p)
inline M6 motion_xform(const M3& R, V3 r) {
  M6 X;
  std::memset(&X, 0, sizeof(X));
  M3 rx = {{{0, -r.z, r.y}, {r.z, 0, -r.x}, {-r.y, r.x, 0}}};
  M3 rxR = mul(rx, R);
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) {
      X.m[i][j] = R.m[i][j];
      X.m[i + 3][j + 3] = R.m[i][j];
      X.m[i + 3][j] = -rxR.m[i][j];
    }
  return X;
}
// solve A x = b for symmetric positive definite 6x6 (Cholesky)
inline bool chol6(const M6& A, double L[6][6]) {
  for (int i = 0; i < 6; i++)
    for (int j = 0; j <= i; j++) {
      double s = A.m[i][j];
      for (int k = 0; k < j; k++) s -= L[i][k] * L[j][k];
      if (i == j) {
        if (!(s > 0)) return false;
        L[i][i] = std::sqrt(s);
      } else {
        L[i][j] = s / L[j][j];
      }
    }
  return true;
}
inline S6 chol6_solve(const double L[6][6], const S6& b) {
  double y[6];
  for (int i = 0; i < 6; i++) {
    double s = b.v[i];
    for (int k = 0; k < i; k++) s -= L[i][k] * y[k];
    y[i] = s / L[i][i];
  }
  S6 x;
  for (int i = 5; i >= 0; i--) {
    double s = y[i];
    for (int k = i + 1; k < 6; k++) s -= L[k][i] * x.v[k];
    x.v[i] = s / L[i][i];
  }
  return x;
}

// ------------------------------------------------------------------ Philox4x32-10 (counter-based RNG)
inline void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
  for (int r = 0; r < 10; r++) {
    uint64_t p0 = (uint64_t)0xD2511F53u * c[0], p1 = (uint64_t)0xCD9E8D57u * c[2];
    uint32_t n0 = (uint32_t)(p1 >> 32) ^ c[1] ^ k0, n1 = (uint32_t)p1;
    uint32_t n2 = (uint32_t)(p0 >> 32) ^ c[3] ^ k1, n3 = (uint32_t)p0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}
// two uniforms in (0,1) for (seed, global env id, episode counter)
inline void reset_uniforms(uint64_t seed, int64_t gid, int64_t episode, double* u_clip, double* u_phase) {
  uint32_t c[4] = {(uint32_t)gid, (uint32_t)((uint64_t)gid >> 32), (uint32_t)episode, (uint32_t)((uint64_t)episode >> 32)};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  *u_clip = ((double)c[0] + 0.5) * (1.0 / 4294967296.0);
  *u_phase = ((double)c[1] + 0.5) * (1.0 / 4294967296.0);
}

// four uniforms of stream `stream` (1 = EPMC reset, 2 = push randomiser, 3 = joystick command), draw `index`
inline void stream_uniforms(uint64_t seed, int64_t gid, int64_t episode, uint32_t stream, uint32_t index, double u[4]) {
  uint32_t c[4] = {(uint32_t)gid, ((uint32_t)((uint64_t)gid >> 32) & 0x00FFFFFFu) | (stream << 24), (uint32_t)episode, index};
  philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32));
  for (int i = 0; i < 4; i++) u[i] = ((double)c[i] + 0.5) * (1.0 / 4294967296.0);
}

// ------------------------------------------------------------------ model
struct LinkM {
  int parent, jtype, dof;
  V3 jxyz; M3 jrot; V3 axis;
  double mass; V3 com; M3 Rin; V3 idiag;
  double lower, upper, jdamp; bool haslim;
};
struct SphereM { int link; V3 c; double r, mu; };
struct ProxyM { int link; V3 c; double r; int kind; };
struct Model {
  std::vector<LinkM> links;
  std::vector<SphereM> spheres;
  std::vector<ProxyM> proxies;   // detection-only spheres for the hurdle plate (llq_load_obstacles)
  int ndof = 0;
  std::vector<int> dof_link;  // dof -> link
};

constexpr int MAXL = 32;   // max links
constexpr int MAXD = 6 + 16;

struct Env {
  double pos[3], quat[4], linv[3], angv[3], q[12], qd[12];
  double kin[LLQ_STATE_DIM];
  double time; int clip; double reward_sum; int episode_steps; int64_t episode;
  int frame_id; double frame_frac;
  double warm[LLQ_MAX_SPHERES];
  double prop_hist[3][LLQ_PROP_DIM]; double act_hist[3][LLQ_ACTION_DIM];
  double foot_pos[12];
  double margin;   // LLQ_F_DECISION_MARGIN
  double foot_mu;  // per-episode foot lateral friction (PGE:209; PMC: cfg.foot_friction)
  // EPMC bookkeeping (PGE:146-179, PR:40-54)
  int counter, cmd_freq; double tgt_x, tgt_y, target_spd, target_angle, last_pos_diff_len, total_spd, max_spd;
  int push_count, push_draws, cmd_draws; double push_f[3];
  int ob_id;      // active hurdle plate (PLE:179,264-265)
  // EPMC elements 1-3: static boxes of the corridor (walls first), centre + half extents; PGE:192-195
  int n_boxes; double boxes[LLQ_MAX_BOXES][6]; double init_pos_diff_len;
  int n_cyl; double cyl[2 * LLQ_MAX_BOXES][5];   // auxiliary edge cylinders (BSE:43-104): axis point x, y, z | radius | length along y
  // SEPMC (CTG): per-robot copies of the pair's game state
  int with_flag, switch_flag, visible, flag_draws, touch; double flag_x, flag_y, fix_spd;
  double yaw_accum_deg;   // PGE:181-189 mutates the shared init-state dict: every reset's yaw is applied on top of the previous ones
  float obs[LLQ_OBS_DIM_SEPMC];
};

}  // namespace

struct llq_engine {
  llq_config cfg;
  Model model; bool has_model = false;
  std::vector<double> frames; std::vector<int32_t> clip_off; int n_clips = 0; double frame_dt = 0; bool has_mocap = false;
  int frame_rate = 0, margin = 0;
  std::vector<double> max_steps, sample_prob, avg_reward;
  std::vector<Env> envs; bool was_reset = false;
  double init_state[LLQ_STATE_DIM]; bool has_init_state = false;
  std::vector<double> ob_table; std::vector<int32_t> ob_off; double ob_half[3] = {0, 0, 0}; bool has_obstacles = false;
  int obs_dim() const { return cfg.env_kind == LLQ_ENV_EPMC ? LLQ_OBS_DIM_EPMC : (cfg.env_kind == LLQ_ENV_SEPMC ? LLQ_OBS_DIM_SEPMC : LLQ_OBS_DIM); }
  int64_t counters[8] = {0, 0, 0, 0, 0, 0, 0, 0};
};

namespace {

// ------------------------------------------------------------------ kinematics of the tree
struct Kin {
  M3 Rl[MAXL]; V3 pl[MAXL];   // link frames in world
  M3 Rc[MAXL]; V3 pc[MAXL];   // inertial (CoM) frames in world
};
void kinematics(const Model& md, const double pos[3], const double quat[4], const double* q, Kin& k) {
  Q4 qb = qnormalize({quat[0], quat[1], quat[2], quat[3]});
  M3 Rb = qmat(qb);
  const LinkM& b = md.links[0];
  k.Rl[0] = mul(Rb, transpose(b.Rin));           // base state is the pose of the base inertial frame (SURVEY A.1)
  k.pl[0] = V3{pos[0], pos[1], pos[2]} - mul(k.Rl[0], b.com);
  k.Rc[0] = Rb; k.pc[0] = {pos[0], pos[1], pos[2]};
  for (size_t i = 1; i < md.links.size(); i++) {
    const LinkM& l = md.links[i];
    M3 R = mul(k.Rl[l.parent], l.jrot);
    if (l.jtype == 1) R = mul(R, axis_angle(l.axis, q[l.dof]));
    k.Rl[i] = R;
    k.pl[i] = k.pl[l.parent] + mul(k.Rl[l.parent], l.jxyz);
    k.Rc[i] = mul(R, l.Rin);
    k.pc[i] = k.pl[i] + mul(R, l.com);
  }
}

// ------------------------------------------------------------------ articulated-body algorithm (Bullet layout)
struct AbaCache {
  M6 X[MAXL];        // motion transform parent CoM frame -> link CoM frame
  S6 S[MAXL];        // joint motion subspace (revolute) in link CoM frame
  S6 U[MAXL]; double Dinv[MAXL];
  double L0[6][6];   // Cholesky factor of the base articulated inertia
  M3 Rb;
};

// Forward dynamics: returns generalized acceleration (omegadot_world, vdot_world, qdd) in acc[6+ndof].
// ext_f / ext_n: optional per-link external force / torque about the CoM, world frame (may be null).
bool aba(const llq_engine& E, const Kin& k, const double* gv /*omega_w, v_w, qd*/, const double* tau,
         const V3* ext_f, const V3* ext_n, double* acc, AbaCache& c) {
  const Model& md = E.model;
  const int n = (int)md.links.size();
  const double kl = E.cfg.lin_damping, ka = E.cfg.ang_damping;
  S6 v[MAXL], cor[MAXL], Z[MAXL], a[MAXL]; M6 IA[MAXL]; double u[MAXL];
  V3 g = {0, 0, E.cfg.gravity_z};
  c.Rb = k.Rc[0];
  for (int i = 0; i < n; i++) {
    const LinkM& l = md.links[i];
    if (i == 0) {
      v[0] = s6(tmul(k.Rc[0], V3{gv[0], gv[1], gv[2]}), tmul(k.Rc[0], V3{gv[3], gv[4], gv[5]}));
      std::memset(&cor[0], 0, sizeof(S6));
    } else {
      M3 R = mul(transpose(k.Rc[i]), k.Rc[l.parent]);
      V3 r = tmul(k.Rc[i], k.pc[i] - k.pc[l.parent]);
      c.X[i] = motion_xform(R, r);
      v[i] = mul6(c.X[i], v[l.parent]);
      if (l.jtype == 1) {
        V3 sa = tmul(l.Rin, l.axis);
        V3 d = tmul(l.Rin, l.com);           // joint pivot (link origin) -> CoM, inertial coords
        c.S[i] = s6(sa, cross(sa, d));
        double qd = gv[6 + l.dof];
        S6 vj;
        for (int t = 0; t < 6; t++) vj.v[t] = c.S[i].v[t] * qd;
        for (int t = 0; t < 6; t++) v[i].v[t] += vj.v[t];
        // velocity-product acceleration  c = v x vj  (motion cross product)
        V3 w = ang(v[i]), vl = lin(v[i]), wj = ang(vj), vjl = lin(vj);
        cor[i] = s6(cross(w, wj), cross(w, vjl) + cross(vl, wj));
      } else {
        std::memset(&cor[i], 0, sizeof(S6));
      }
    }
    // zero-acceleration (bias) force, Bullet order: -external, +damping, +gyroscopic
    V3 w = ang(v[i]), vl = lin(v[i]);
    V3 Iw = {l.idiag.x * w.x, l.idiag.y * w.y, l.idiag.z * w.z};
    V3 f_ext = l.mass * g;
    V3 n_ext = {0, 0, 0};
    if (ext_f) f_ext = f_ext + ext_f[i];
    if (ext_n) n_ext = n_ext + ext_n[i];
    V3 zn = (-1.0) * tmul(k.Rc[i], n_ext), zf = (-1.0) * tmul(k.Rc[i], f_ext);
    zn = zn + (ka + ka * norm(w)) * Iw;
    zf = zf + (l.mass * (kl + kl * norm(vl))) * vl;
    zn = zn + cross(w, Iw);
    zf = zf + l.mass * cross(w, vl);
    Z[i] = s6(zn, zf);
    std::memset(&IA[i], 0, sizeof(M6));
    IA[i].m[0][0] = l.idiag.x; IA[i].m[1][1] = l.idiag.y; IA[i].m[2][2] = l.idiag.z;
    IA[i].m[3][3] = IA[i].m[4][4] = IA[i].m[5][5] = l.mass;
  }
  for (int i = n - 1; i >= 1; i--) {
    const LinkM& l = md.links[i];
    M6 Ia = IA[i]; S6 pa = Z[i];
    if (l.jtype == 1) {
      c.U[i] = mul6(IA[i], c.S[i]);
      double D = dot6(c.S[i], c.U[i]);
      if (!(D > 0)) return false;
      c.Dinv[i] = 1.0 / D;
      u[i] = tau[l.dof] - dot6(c.S[i], Z[i]);
      for (int r = 0; r < 6; r++)
        for (int s = 0; s < 6; s++) Ia.m[r][s] -= c.U[i].v[r] * c.U[i].v[s] * c.Dinv[i];
      S6 Iac = mul6(Ia, cor[i]);
      for (int t = 0; t < 6; t++) pa.v[t] += Iac.v[t] + c.U[i].v[t] * (u[i] * c.Dinv[i]);
    }
    // IA[parent] += X^T Ia X ; Z[parent] += X^T pa
    const M6& X = c.X[i];
    M6 T;
    for (int r = 0; r < 6; r++)
      for (int s = 0; s < 6; s++) {
        double acc2 = 0;
        for (int t = 0; t < 6; t++) acc2 += Ia.m[r][t] * X.m[t][s];
        T.m[r][s] = acc2;
      }
    for (int r = 0; r < 6; r++)
      for (int s = 0; s < 6; s++) {
        double acc2 = 0;
        for (int t = 0; t < 6; t++) acc2 += X.m[t][r] * T.m[t][s];
        IA[l.parent].m[r][s] += acc2;
      }
    S6 zp = tmul6(X, pa);
    for (int t = 0; t < 6; t++) Z[l.parent].v[t] += zp.v[t];
  }
  if (!chol6(IA[0], c.L0)) return false;
  S6 mz;
  for (int t = 0; t < 6; t++) mz.v[t] = -Z[0].v[t];
  a[0] = chol6_solve(c.L0, mz);
  for (int i = 1; i < n; i++) {
    const LinkM& l = md.links[i];
    a[i] = mul6(c.X[i], a[l.parent]);
    for (int t = 0; t < 6; t++) a[i].v[t] += cor[i].v[t];
    if (l.jtype == 1) {
      double qdd = (u[i] - dot6(c.U[i], a[i])) * c.Dinv[i];
      acc[6 + l.dof] = qdd;
      for (int t = 0; t < 6; t++) a[i].v[t] += c.S[i].v[t] * qdd;
    }
  }
  // base acceleration back to world; classical linear acceleration = spatial + omega x v
  V3 wb = ang(v[0]), vb = lin(v[0]);
  V3 od = mul(k.Rc[0], ang(a[0]));
  V3 vd = mul(k.Rc[0], lin(a[0]) + cross(wb, vb));
  acc[0] = od.x; acc[1] = od.y; acc[2] = od.z; acc[3] = vd.x; acc[4] = vd.y; acc[5] = vd.z;
  return true;
}

// Response of the generalized velocity to a unit generalized impulse F (torque_w, force_w on the base CoM, joint
// torques): out = M^-1 F, using the quantities cached by aba() (Bullet: calcAccelerationDeltasMultiDof).
void aba_delta(const Model& md, const AbaCache& c, const double* F, double* out) {
  const int n = (int)md.links.size();
  S6 Z[MAXL], a[MAXL]; double u[MAXL];
  for (int i = 0; i < n; i++) std::memset(&Z[i], 0, sizeof(S6));
  Z[0] = s6((-1.0) * tmul(c.Rb, V3{F[0], F[1], F[2]}), (-1.0) * tmul(c.Rb, V3{F[3], F[4], F[5]}));
  for (int i = n - 1; i >= 1; i--) {
    const LinkM& l = md.links[i];
    S6 pa = Z[i];
    if (l.jtype == 1) {
      u[i] = F[6 + l.dof] - dot6(c.S[i], Z[i]);
      for (int t = 0; t < 6; t++) pa.v[t] += c.U[i].v[t] * (u[i] * c.Dinv[i]);
    }
    S6 zp = tmul6(c.X[i], pa);
    for (int t = 0; t < 6; t++) Z[l.parent].v[t] += zp.v[t];
  }
  S6 mz;
  for (int t = 0; t < 6; t++) mz.v[t] = -Z[0].v[t];
  a[0] = chol6_solve(c.L0, mz);
  for (int i = 1; i < n; i++) {
    const LinkM& l = md.links[i];
    a[i] = mul6(c.X[i], a[l.parent]);
    if (l.jtype == 1) {
      double qdd = (u[i] - dot6(c.U[i], a[i])) * c.Dinv[i];
      out[6 + l.dof] = qdd;
      for (int t = 0; t < 6; t++) a[i].v[t] += c.S[i].v[t] * qdd;
    }
  }
  V3 od = mul(c.Rb, ang(a[0])), vd = mul(c.Rb, lin(a[0]));
  out[0] = od.x; out[1] = od.y; out[2] = od.z; out[3] = vd.x; out[4] = vd.y; out[5] = vd.z;
}

// Jacobian row of "velocity of world point P fixed on link li, along world direction d" w.r.t. (omega_w, v_w, qd)
void point_jacobian(const Model& md, const Kin& k, int li, V3 P, V3 d, double* J) {
  for (int t = 0; t < 6 + md.ndof; t++) J[t] = 0;
  V3 rb = P - k.pc[0];
  V3 jw = cross(rb, d);
  J[0] = jw.x; J[1] = jw.y; J[2] = jw.z; J[3] = d.x; J[4] = d.y; J[5] = d.z;
  for (int i = li; i > 0; i = md.links[i].parent) {
    const LinkM& l = md.links[i];
    if (l.jtype != 1) continue;
    V3 aw = mul(k.Rl[i], l.axis);
    J[6 + l.dof] = dot(cross(aw, P - k.pl[i]), d);
  }
}

// btPlaneSpace1
void plane_space(V3 n, V3& p, V3& q) {
  if (std::fabs(n.z) > 0.7071067811865475244008443621048490) {
    double a = n.y * n.y + n.z * n.z, kk = 1.0 / std::sqrt(a);
    p = {0, -n.z * kk, n.y * kk};
    q = {a * kk, -n.x * p.z, n.x * p.y};
  } else {
    double a = n.x * n.x + n.y * n.y, kk = 1.0 / std::sqrt(a);
    p = {-n.y * kk, n.x * kk, 0};
    q = {-n.z * p.y, n.z * p.x, a * kk};
  }
}

struct Row {
  double J[MAXD], W[MAXD];
  double rhs, invd, lam, lo, hi;
};

inline double clampd(double v, double lo, double hi) { return std::max(lo, std::min(v, hi)); }

// One Bullet stepSimulation() with numSubSteps=1 (SURVEY A.2) for one robot on the infinite plane z=0.
// tau: motor torques (12).  Returns false if the dynamics became singular / non-finite.
bool physics_substep(llq_engine& E, Env& e, const double* tau, int64_t* n_contact_rows, int64_t* n_limit_rows,
                     const double* push_local = nullptr) {
  const Model& md = E.model;
  const llq_config& cf = E.cfg;
  const int nd = 6 + md.ndof;
  const double dt = cf.sim_dt;
  Kin k;
  kinematics(md, e.pos, e.quat, e.q, k);

  // (a) collision detection on pre-step poses: foot spheres vs plane z = 0
  struct Contact { int link, sphere; V3 P, n; double dist, mu; };
  Contact contacts[LLQ_MAX_SPHERES]; int nc = 0;
  // static half-spaces the feet can touch: the ground, plus (SEPMC) the inner faces of the four arena walls (BSG:863-902:
  // 5 x 0.01 x 2 boxes centred at +-2.5).  One contact per foot: the deepest half-space (DESIGN.md 5).
  const int n_planes = cf.env_kind == LLQ_ENV_SEPMC ? 5 : 1;
  const V3 pn[5] = {{0, 0, 1}, {-1, 0, 0}, {1, 0, 0}, {0, -1, 0}, {0, 1, 0}};
  const double pd[5] = {0.0, -2.495, -2.495, -2.495, -2.495};
  for (size_t s = 0; s < md.spheres.size(); s++) {
    const SphereM& sp = md.spheres[s];
    V3 cw = k.pl[sp.link] + mul(k.Rl[sp.link], sp.c);
    double dist = 1e30, second = 1e30; V3 nrm = pn[0];      // second: runner-up among the statics (the sphere keeps ONE manifold point)
    const bool statics = s < 4 || cf.knee_contacts == 2;           // legacy sets: only the feet touch walls and boxes
    for (int pi = 0; pi < (statics ? n_planes : 1); pi++) {
      double dpi = dot(pn[pi], cw) - pd[pi] - sp.r;
      if (dpi < dist) { second = dist; dist = dpi; nrm = pn[pi]; } else second = std::min(second, dpi);
    }
    // EPMC corridor: sphere vs every static box (walls, hurdles, bars, cubes), then the auxiliary edge cylinders below; one contact
    // per sphere, the deepest.  Under knee_contacts 0 / 1 only the feet meet walls, boxes and cylinders; under 2 every sphere does.
    for (int b = 0; b < (statics ? e.n_boxes : 0); b++) {
      const double* bx = e.boxes[b];
      const double p[3] = {cw.x - bx[0], cw.y - bx[1], cw.z - bx[2]};
      double c[3]; bool inside = true;
      for (int a = 0; a < 3; a++) { c[a] = clampd(p[a], -bx[3 + a], bx[3 + a]); if (c[a] != p[a]) inside = false; }
      double db; V3 nb;
      if (!inside) {
        const V3 v = {p[0] - c[0], p[1] - c[1], p[2] - c[2]};
        const double len = norm(v);
        db = len - sp.r; nb = (1.0 / len) * v;
      } else {                                  // centre inside the box: leave through the nearest face
        int ax = 0; double best = 1e30, sg = 1.0;
        for (int a = 0; a < 3; a++) {
          const double dp = bx[3 + a] - p[a], dm = bx[3 + a] + p[a];
          if (dp < best) { best = dp; ax = a; sg = 1.0; }
          if (dm < best) { best = dm; ax = a; sg = -1.0; }
        }
        db = -best - sp.r; nb = V3{ax == 0 ? sg : 0.0, ax == 1 ? sg : 0.0, ax == 2 ? sg : 0.0};
      }
      if (db < dist) { second = dist; dist = db; nrm = nb; } else second = std::min(second, db);
    }
    // auxiliary edge cylinders (static bodies of their own in the reference; here they compete for the sphere's one manifold point)
    for (int c = 0; c < (statics ? e.n_cyl : 0); c++) {
      const double* cy = e.cyl[c];
      if (std::fabs(cw.y - cy[1]) > 0.5 * cy[4]) continue;          // beside the cylinder's length (its flat ends lie in the walls)
      const double dx = cw.x - cy[0], dz = cw.z - cy[2], len = std::sqrt(dx * dx + dz * dz);
      if (!(len > 0)) continue;
      const double dc = len - cy[3] - sp.r;
      if (dc < dist) { second = dist; dist = dc; nrm = V3{dx / len, 0.0, dz / len}; } else second = std::min(second, dc);
    }
    e.margin = std::min(e.margin, std::fabs(dist - cf.contact_breaking));
    if (second < cf.contact_breaking) e.margin = std::min(e.margin, second - dist);   // which static is the deepest: also a branch of the step
    if (dist < cf.contact_breaking) {
      contacts[nc++] = {sp.link, (int)s, cw - sp.r * nrm, nrm, dist, cf.ground_friction * (s < 4 ? e.foot_mu : sp.mu)};
    } else {
      e.warm[s] = 0.0;  // manifold point removed
    }
  }

  if (cf.knee_contacts == 1 && md.spheres.size() == 8) {
    // legacy rule (llq_config.knee_contacts = 1): one contact per leg, the deeper of {foot, knee wheel}
    Contact kept[LLQ_MAX_SPHERES]; int nk = 0;
    for (int leg = 0; leg < 4; leg++) {
      int best = -1;
      for (int ci = 0; ci < nc; ci++)
        if (contacts[ci].sphere == leg || contacts[ci].sphere == 4 + leg) {
          if (best >= 0) e.margin = std::min(e.margin, std::fabs(contacts[ci].dist - contacts[best].dist));   // which of the two wins
          if (best < 0 || contacts[ci].dist < contacts[best].dist) best = ci;
        }
      for (int ci = 0; ci < nc; ci++)
        if ((contacts[ci].sphere == leg || contacts[ci].sphere == 4 + leg) && ci != best) e.warm[contacts[ci].sphere] = 0.0;
      if (best >= 0) kept[nk++] = contacts[best];
    }
    nc = nk;
    for (int ci = 0; ci < nc; ci++) contacts[ci] = kept[ci];
  }
  // both engines keep at most LLQ_MAX_CONTACTS manifold points per robot (sphere order) and LLQ_MAX_LIMIT_ROWS limit rows (joint order);
  // anything beyond that is a heap of a robot whose episode ends with this step (counter [5] counts the dropped rows)
  for (int ci = LLQ_MAX_CONTACTS; ci < nc; ci++) e.warm[contacts[ci].sphere] = 0.0;
  if (nc > LLQ_MAX_CONTACTS) {
    const int64_t dropped = nc - LLQ_MAX_CONTACTS;
#pragma omp atomic
    E.counters[LLQ_CNT_DROPPED] += dropped;
    nc = LLQ_MAX_CONTACTS;
  }
  // (b) joint damping (pybullet applyJointDamping) + motor torque, forward dynamics, velocity prediction
  double gv[MAXD], tt[16], acc[MAXD];
  for (int t = 0; t < 3; t++) { gv[t] = e.angv[t]; gv[3 + t] = e.linv[t]; }
  for (int j = 0; j < md.ndof; j++) {
    gv[6 + j] = e.qd[j];
    tt[j] = tau[j] - md.links[md.dof_link[j]].jdamp * e.qd[j];
  }
  AbaCache c;
  V3 extf[MAXL];
  if (push_local) {
    // applyExternalForce(linkIndex=0, LINK_FRAME) (PR:73-77): pybullet link 0 = first child link (FR hip); force and position
    // are expressed in that link's inertial frame; position (0,0,0) = its CoM => pure force, no torque (SURVEY A.2.4)
    for (size_t i = 0; i < md.links.size(); i++) extf[i] = V3{0, 0, 0};
    extf[1] = mul(k.Rc[1], V3{push_local[0], push_local[1], push_local[2]});
  }
  if (!aba(E, k, gv, tt, push_local ? extf : nullptr, nullptr, acc, c)) return false;
  for (int t = 0; t < nd; t++) gv[t] = clampd(gv[t] + acc[t] * dt, -cf.max_coord_vel, cf.max_coord_vel);

  // (c) constraint rows
  std::vector<Row> lim, nrm, fr;
  for (int j = 0; j < md.ndof; j++) {
    const LinkM& l = md.links[md.dof_link[j]];
    if (!l.haslim) continue;
    for (int side = 0; side < 2; side++) {
      double pen = side == 0 ? e.q[j] - l.lower : l.upper - e.q[j];
      e.margin = std::min(e.margin, std::fabs(pen));
      if (pen > 0) continue;                       // btMultiBodyJointLimitConstraint: row only when violated
      e.margin = std::min(e.margin, std::fabs(pen + 0.04));   // the split-impulse threshold below switches the positional term
      double dir = side == 0 ? 1.0 : -1.0;
      Row r; std::memset(&r, 0, sizeof(r));
      r.J[6 + j] = dir;
      aba_delta(md, c, r.J, r.W);
      double denom = 0, rel = 0;
      for (int t = 0; t < nd; t++) { denom += r.J[t] * r.W[t]; rel += r.J[t] * gv[t]; }
      r.invd = 1.0 / denom;
      // split-impulse quirk: positional term only while the violation is shallower than 0.04 (m_splitImpulsePenetrationThreshold)
      double poserr = pen > -0.04 ? -pen * cf.joint_erp / dt : 0.0;
      r.rhs = (poserr - rel) * r.invd;
      r.lo = 0; r.hi = cf.max_applied_impulse; r.lam = 0;
      if ((int)lim.size() < LLQ_MAX_LIMIT_ROWS) lim.push_back(r);
      else {
#pragma omp atomic
        E.counters[LLQ_CNT_DROPPED] += 1;
      }
    }
  }
  for (int ci = 0; ci < nc; ci++) {
    const Contact& ct = contacts[ci];
    V3 nrml = ct.n, t1, t2;
    plane_space(nrml, t1, t2);
    V3 dirs[3] = {nrml, t1, t2};
    for (int d = 0; d < 3; d++) {
      Row r; std::memset(&r, 0, sizeof(r));
      point_jacobian(md, k, ct.link, ct.P, dirs[d], r.J);
      aba_delta(md, c, r.J, r.W);
      double denom = 0, rel = 0;
      for (int t = 0; t < nd; t++) { denom += r.J[t] * r.W[t]; rel += r.J[t] * gv[t]; }
      r.invd = 1.0 / denom;
      if (d == 0) {
        double pen = ct.dist + cf.linear_slop;
        double poserr = 0, velerr = -rel;
        if (pen > 0) velerr -= pen / dt; else poserr = -pen * cf.contact_erp / dt;
        r.rhs = (poserr + velerr) * r.invd;
        r.lo = 0; r.hi = 1e10;
        r.lam = cf.warmstart * e.warm[ct.sphere];
        nrm.push_back(r);
      } else {
        r.rhs = -rel * r.invd;
        r.lam = 0;
        fr.push_back(r);
      }
    }
  }
  *n_contact_rows += (int64_t)nrm.size() * 3;
  *n_limit_rows += (int64_t)lim.size();

  // (d) projected Gauss-Seidel on delta velocities
  double dv[MAXD];
  for (int t = 0; t < nd; t++) dv[t] = 0;
  for (auto& r : nrm)
    if (r.lam != 0)
      for (int t = 0; t < nd; t++) dv[t] += r.W[t] * r.lam;   // warm start
  auto solve_row = [&](Row& r) {
    double jd = 0;
    for (int t = 0; t < nd; t++) jd += r.J[t] * dv[t];
    double dl = r.rhs - jd * r.invd;
    double sum = r.lam + dl;
    if (sum < r.lo) { dl = r.lo - r.lam; r.lam = r.lo; }
    else if (sum > r.hi) { dl = r.hi - r.lam; r.lam = r.hi; }
    else r.lam = sum;
    for (int t = 0; t < nd; t++) dv[t] += r.W[t] * dl;
  };
  for (int it = 0; it < cf.solver_iters; it++) {
    for (auto& r : lim) solve_row(r);
    for (auto& r : nrm) solve_row(r);
    for (size_t ci = 0; ci < nrm.size(); ci++) {   // implicit cone friction on the row pair (t1, t2)
      Row& a = fr[2 * ci]; Row& b = fr[2 * ci + 1];
      double limit = contacts[ci].mu * nrm[ci].lam;
      double ja = 0, jb = 0;
      for (int t = 0; t < nd; t++) { ja += a.J[t] * dv[t]; jb += b.J[t] * dv[t]; }
      double sa = a.lam + (a.rhs - ja * a.invd), sb = b.lam + (b.rhs - jb * b.invd);
      double r2 = sa * sa + sb * sb;
      if (r2 >= limit * limit && r2 > 0) {
        double sc = limit / std::sqrt(r2);
        sa *= sc; sb *= sc;
      }
      double da = sa - a.lam, db = sb - b.lam;
      a.lam = sa; b.lam = sb;
      for (int t = 0; t < nd; t++) dv[t] += a.W[t] * da + b.W[t] * db;
    }
  }
  for (int t = 0; t < nd; t++) gv[t] = clampd(gv[t] + dv[t], -cf.max_coord_vel, cf.max_coord_vel);
  for (int ci = 0; ci < nc; ci++) e.warm[contacts[ci].sphere] = nrm[ci].lam;

  // (e) integrate (btMultiBody::stepPositionsMultiDof): explicit positions from the new velocities
  for (int t = 0; t < 3; t++) { e.angv[t] = gv[t]; e.linv[t] = gv[3 + t]; e.pos[t] += gv[3 + t] * dt; }
  {
    V3 w = {gv[0], gv[1], gv[2]};
    double fa = norm(w);
    V3 ax;
    if (fa < 0.001) ax = (0.5 * dt - dt * dt * dt * 0.020833333333 * fa * fa) * w;
    else ax = (std::sin(0.5 * fa * dt) / fa) * w;
    Q4 dq = {ax.x, ax.y, ax.z, std::cos(fa * dt * 0.5)};
    Q4 qn = qnormalize(qmul(dq, Q4{e.quat[0], e.quat[1], e.quat[2], e.quat[3]}));
    e.quat[0] = qn.x; e.quat[1] = qn.y; e.quat[2] = qn.z; e.quat[3] = qn.w;
  }
  for (int j = 0; j < md.ndof; j++) { e.qd[j] = gv[6 + j]; e.q[j] += gv[6 + j] * dt; }
  for (int t = 0; t < nd; t++)
    if (!std::isfinite(gv[t])) return false;
  return true;
}

// ------------------------------------------------------------------ MotionLib restatement (ML:11-172)
inline const double* frame_ptr(const llq_engine& E, int clip, int f) {
  return &E.frames[(size_t)(E.clip_off[clip] + f) * LLQ_MOCAP_FRAME];
}
// ML:88-166 _get_states_info_by_interpolation -> 37 doubles in LLQ_F_STATE order
void mocap_state(const llq_engine& E, const double* fc, const double* fn, double frac, double* st) {
  const double dt = E.frame_dt;
  for (int i = 0; i < 3; i++) {
    st[i] = fc[i] + frac * (fn[i] - fc[i]);          // ML:118-124
    st[7 + i] = (fn[i] - fc[i]) / dt;                // ML:137-140
  }
  Q4 qc = qnormalize({fc[3], fc[4], fc[5], fc[6]}), qn = qnormalize({fn[3], fn[4], fn[5], fn[6]});
  V3 rv = q_rotvec(qmul(qconj(qc), qn));             // scipy Slerp: rotvec of R_c^-1 R_n
  Q4 qi = qmul(qc, rotvec_q(frac * rv));             // ML:127-134
  st[3] = qi.x; st[4] = qi.y; st[5] = qi.z; st[6] = qi.w;
  V3 rw = q_rotvec(qmul(qn, qconj(qc)));             // ML:143-149
  double angle = norm(rw);
  V3 axis = (1.0 / (angle + 1e-8)) * rw;
  st[10] = axis.x * angle / dt; st[11] = axis.y * angle / dt; st[12] = axis.z * angle / dt;
  for (int j = 0; j < 12; j++) {                     // ML:152-160
    st[13 + j] = fc[7 + j] + frac * (fn[7 + j] - fc[7 + j]);
    st[25 + j] = (fn[7 + j] - fc[7 + j]) / dt;
  }
}
const double kTimeFuture[4] = {1. / 30., 1. / 15., 1. / 3., 1.};  // ML:44

void foot_positions(const llq_engine& E, const double* st, double* out12) {
  Kin k;
  kinematics(E.model, st, st + 3, st + 13, k);
  for (size_t s = 0; s < E.model.spheres.size() && s < 4; s++) {
    int li = E.model.spheres[s].link;
    out12[3 * s] = k.pc[li].x; out12[3 * s + 1] = k.pc[li].y; out12[3 * s + 2] = k.pc[li].z;  // getLinkState()[0]
  }
}

inline void pack_state(const Env& e, double* st) {
  for (int i = 0; i < 3; i++) { st[i] = e.pos[i]; st[7 + i] = e.linv[i]; st[10 + i] = e.angv[i]; }
  for (int i = 0; i < 4; i++) st[3 + i] = e.quat[i];
  for (int j = 0; j < 12; j++) { st[13 + j] = e.q[j]; st[25 + j] = e.qd[j]; }
}
inline void unpack_state(Env& e, const double* st) {
  for (int i = 0; i < 3; i++) { e.pos[i] = st[i]; e.linv[i] = st[7 + i]; e.angv[i] = st[10 + i]; }
  for (int i = 0; i < 4; i++) e.quat[i] = st[3 + i];
  for (int j = 0; j < 12; j++) { e.q[j] = st[13 + j]; e.qd[j] = st[25 + j]; }
}

// PLE:247-260 with the shipped prop_type order
void make_prop(const double* st, double* prop) {
  M3 R = qmat(qnormalize({st[3], st[4], st[5], st[6]}));
  for (int j = 0; j < 12; j++) { prop[j] = st[13 + j]; prop[12 + j] = st[25 + j]; }
  V3 wl = tmul(R, V3{st[10], st[11], st[12]}), vl = tmul(R, V3{st[7], st[8], st[9]});
  prop[24] = wl.x; prop[25] = wl.y; prop[26] = wl.z;
  prop[27] = vl.x; prop[28] = vl.y; prop[29] = vl.z;
  prop[30] = R.m[2][0]; prop[31] = R.m[2][1]; prop[32] = R.m[2][2];
}

// PLE:299-317 + ML:75-86
void make_future(const llq_engine& E, const Env& e, const double* st, double* fut72) {
  Q4 qb = qnormalize({st[3], st[4], st[5], st[6]});
  M3 Rb = qmat(qb);
  for (int i = 0; i < 4; i++) {
    double t = E.frame_dt * e.frame_frac + kTimeFuture[i];           // ML:80
    int fid = (int)std::floor(t / E.frame_dt);                        // ML:81
    double ffrac = t / E.frame_dt - fid;                              // ML:82
    double fs[LLQ_STATE_DIM];
    mocap_state(E, frame_ptr(E, e.clip, e.frame_id + fid), frame_ptr(E, e.clip, e.frame_id + fid + 1), ffrac, fs);
    Q4 qi = qnormalize({fs[3], fs[4], fs[5], fs[6]});
    Q4 qd = qmul(qconj(qb), qi);                                      // PLE:307
    V3 rv = q_rotvec(qnormalize(qd));
    double angle = norm(rv);
    V3 axis = (1.0 / (angle + 1e-8)) * rv;                            // PLE:19-23
    V3 dp = tmul(Rb, V3{fs[0] - st[0], fs[1] - st[1], fs[2] - st[2]}); // PLE:310-311
    double* o = fut72 + 18 * i;
    o[0] = dp.x; o[1] = dp.y; o[2] = dp.z;
    o[3] = axis.x * angle; o[4] = axis.y * angle; o[5] = axis.z * angle;
    for (int j = 0; j < 12; j++) o[6 + j] = fs[13 + j];
  }
}

void write_obs(const llq_engine& E, Env& e, const double* st) {
  double fut[72];
  make_future(E, e, st, fut);
  int o = 0;
  for (int h = 0; h < 3; h++)
    for (int t = 0; t < LLQ_PROP_DIM; t++) e.obs[o++] = (float)e.prop_hist[h][t];
  for (int h = 0; h < 3; h++)
    for (int t = 0; t < LLQ_ACTION_DIM; t++) e.obs[o++] = (float)e.act_hist[h][t];
  for (int t = 0; t < 72; t++) e.obs[o++] = (float)fut[t];
}

void motion_set_time(const llq_engine& E, Env& e, double t) {  // ML:65-67
  e.frame_id = (int)std::floor(t / E.frame_dt);
  e.frame_frac = (t - e.frame_id * E.frame_dt) / E.frame_dt;
  // A cursor past the clip's playable range (a finished env stepped on without a reset, a clock set through llq_set_field) stays on
  // the last cursor whose 1 s future window (122 frames) lies inside the clip -- the reference raises IndexError there; both engines
  // clamp.  The final step of an episode legitimately runs up to 2.4 frames past the "ended" threshold nf - margin - 1.
  const int last = E.clip_off[e.clip + 1] - E.clip_off[e.clip] - E.margin + 2;
  if (e.frame_id > last) { e.frame_id = last; e.frame_frac = 0.0; }
  if (e.frame_id < 0) { e.frame_id = 0; e.frame_frac = 0.0; }
}

// PLE:150-171 with (clip, sampled_time) given
void reset_env(llq_engine& E, Env& e, int clip, double sampled_time) {
  e.clip = clip;
  e.time = sampled_time;
  motion_set_time(E, e, sampled_time);                                   // ML:52-53 (same arithmetic as ML:65-67)
  mocap_state(E, frame_ptr(E, clip, e.frame_id), frame_ptr(E, clip, e.frame_id + 1), e.frame_frac, e.kin);
  unpack_state(e, e.kin);                                                // PLE:162-163
  e.reward_sum = 0; e.episode_steps = 0;
  e.ob_id = 0;                                                                           // PLE:179
  e.foot_mu = E.cfg.foot_friction;
  for (int s = 0; s < LLQ_MAX_SPHERES; s++) e.warm[s] = 0;
  double prop[LLQ_PROP_DIM];
  make_prop(e.kin, prop);
  for (int h = 0; h < 3; h++) {                                          // PLE:282-290
    std::memcpy(e.prop_hist[h], prop, sizeof(prop));
    for (int t = 0; t < 12; t++) e.act_hist[h][t] = 0;
  }
  foot_positions(E, e.kin, e.foot_pos);
  write_obs(E, e, e.kin);
}

void sample_reset(llq_engine& E, Env& e, int64_t gid) {
  double u1, u2;
  reset_uniforms(E.cfg.seed, gid, e.episode, &u1, &u2);
  e.episode++;
  // np.random.choice(p): cdf = cumsum(p); cdf /= cdf[-1]; searchsorted(cdf, u, side='right')   (ML:60)
  double tot = 0;
  for (int c = 0; c < E.n_clips; c++) tot += E.sample_prob[c];
  double acc = 0; int clip = E.n_clips - 1;
  for (int c = 0; c < E.n_clips; c++) {
    acc += E.sample_prob[c];
    if (acc / tot > u1) { clip = c; break; }
  }
  int nf = E.clip_off[clip + 1] - E.clip_off[clip];
  double duration = E.frame_dt * (nf - E.margin - 1);                    // ML:50
  reset_env(E, e, clip, u2 * duration);                                  // ML:51
}

// Robot (detection proxies) vs the active hurdle plate: box [hx, hy, hz] centred at (x, y, 0), yawed (OBS:27-33, PLE:184-193).
bool obstacle_hit(const llq_engine& E, const Env& e) {
  if (!E.has_obstacles) return false;
  int n_ob = E.ob_off[e.clip + 1] - E.ob_off[e.clip];
  if (n_ob == 0) return false;                                  // MotionLib.obstacle is None for this clip (OBS:17-18)
  const double* ob = &E.ob_table[(size_t)(E.ob_off[e.clip] + e.ob_id) * 4];
  Kin k;
  kinematics(E.model, e.pos, e.quat, e.q, k);
  double cy = std::cos(ob[3]), sy = std::sin(ob[3]);
  for (const ProxyM& p : E.model.proxies) {
    if (p.kind > 3) continue;   // handles (kind 4) only serve SEPMC visibility
    V3 w = k.pl[p.link] + mul(k.Rl[p.link], p.c);
    double dx = w.x - ob[1], dy = w.y - ob[2], dz = w.z;
    double bx = cy * dx + sy * dy, by = -sy * dx + cy * dy;    // into the plate frame
    double qx = bx - clampd(bx, -E.ob_half[0], E.ob_half[0]), qy = by - clampd(by, -E.ob_half[1], E.ob_half[1]),
           qz = dz - clampd(dz, -E.ob_half[2], E.ob_half[2]);
    double dist = std::sqrt(qx * qx + qy * qy + qz * qz) - p.r;
    if (dist < E.cfg.contact_breaking) return true;
  }
  return false;
}

// PLE:195-245 for one env; returns reward, sets *done
double step_env(llq_engine& E, Env& e, const float* action, bool* done, int64_t* ncr, int64_t* nlr) {
  const llq_config& cf = E.cfg;
  e.episode_steps += 1;
  e.margin = 1e30;
  double act[12], tgt[12], tau[12];
  for (int j = 0; j < 12; j++) { act[j] = (double)action[j]; tgt[j] = e.q[j] + act[j]; }   // PLE:198-200
  bool ok = true, ob_hit = false;
  for (int s = 0; s < cf.substeps; s++) {
    for (int j = 0; j < 12; j++) {                                                          // LR:126-141
      double tg = clampd(tgt[j], -3.0, 3.0);
      double t = cf.kp * (tg - e.q[j]) + cf.kd * (0.0 - e.qd[j]);
      tau[j] = clampd(t, -cf.max_tau, cf.max_tau);
    }
    // getContactPoints (PLE:343) reports the manifolds of the last stepSimulation, which were built on that sub-step's
    // pre-step poses, with the plate where _update_obstacle left it at the end of the previous policy step
    if (s == cf.substeps - 1) ob_hit = obstacle_hit(E, e);
    if (ok) ok = physics_substep(E, e, tau, ncr, nlr);                                       // PLE:206
    motion_set_time(E, e, e.time);                                                           // PLE:208
    e.time += cf.sim_dt;                                                                     // PLE:210
  }
  if (E.has_obstacles) {                                                                     // PLE:224-225, 262-268
    int n_ob = E.ob_off[e.clip + 1] - E.ob_off[e.clip];
    while (e.ob_id < n_ob - 1 && e.time > E.ob_table[(size_t)(E.ob_off[e.clip] + e.ob_id) * 4] + 0.5) e.ob_id++;
  }
  // PLE:217-222
  mocap_state(E, frame_ptr(E, e.clip, e.frame_id), frame_ptr(E, e.clip, e.frame_id + 1), e.frame_frac, e.kin);
  double st[LLQ_STATE_DIM];
  pack_state(e, st);
  // PLE:276-297 history update
  double prop[LLQ_PROP_DIM];
  make_prop(st, prop);
  std::memmove(e.prop_hist[0], e.prop_hist[1], 2 * sizeof(e.prop_hist[0]));
  std::memcpy(e.prop_hist[2], prop, sizeof(prop));
  std::memmove(e.act_hist[0], e.act_hist[1], 2 * sizeof(e.act_hist[0]));
  std::memcpy(e.act_hist[2], act, sizeof(act));
  write_obs(E, e, st);
  // reward PLE:350-426
  double sw = cf.w_joint_pos + cf.w_joint_vel + cf.w_end_effector + cf.w_root_pose + cf.w_root_vel;
  double djp = 0, djv = 0;
  for (int j = 0; j < 12; j++) {
    double a = st[13 + j] - e.kin[13 + j], b = st[25 + j] - e.kin[25 + j];
    djp += a * a; djv += b * b;
  }
  double fd[12], fk[12], dee = 0;
  foot_positions(E, st, fd);
  foot_positions(E, e.kin, fk);
  for (int t = 0; t < 12; t++) { dee += (fd[t] - fk[t]) * (fd[t] - fk[t]); e.foot_pos[t] = fd[t]; }
  double dp = 0, dvl = 0, dva = 0;
  for (int t = 0; t < 3; t++) {
    dp += (st[t] - e.kin[t]) * (st[t] - e.kin[t]);
    dvl += (st[7 + t] - e.kin[7 + t]) * (st[7 + t] - e.kin[7 + t]);
    dva += (st[10 + t] - e.kin[10 + t]) * (st[10 + t] - e.kin[10 + t]);
  }
  Q4 q1 = qnormalize({st[3], st[4], st[5], st[6]}), q2 = qnormalize({e.kin[3], e.kin[4], e.kin[5], e.kin[6]});
  double angle = norm(q_rotvec(qnormalize(qmul(q2, qconj(q1)))));                           // PLE:410-411
  double r = (cf.w_joint_pos / sw) * std::exp(-1.0 * djp) + (cf.w_joint_vel / sw) * std::exp(-0.1 * djv) +
             (cf.w_end_effector / sw) * std::exp(-40.0 * dee) +
             (cf.w_root_pose / sw) * std::exp(-20.0 * dp - 10.0 * angle * angle) +
             (cf.w_root_vel / sw) * std::exp(-2.0 * dvl - 0.2 * dva);
  // termination PLE:337-348
  M3 R = qmat(q1);
  double left_z = R.m[0][2] * R.m[1][0] - R.m[1][2] * R.m[0][0];                             // LR:171-172
  bool fall = left_z > std::sin(45.0 * M_PI / 180.0) || left_z < std::sin(-45.0 * M_PI / 180.0) ||
              R.m[2][2] < std::cos(60.0 * M_PI / 180.0);                                     // LR:173-178
  int nf = E.clip_off[e.clip + 1] - E.clip_off[e.clip];
  bool ended = e.frame_id >= nf - E.margin - 1;                                              // ML:168-172
  bool diff = std::fabs(angle) > 1.0 || dp > 1.0;                                            // PLE:319-335
  *done = fall || ended || diff || ob_hit || !ok;                                            // PLE:347
  if (!ok || !std::isfinite(r)) { r = 0.0; *done = true; }
  e.reward_sum += r;                  // after the zeroing: a NaN reward must not poison the sum and, through it, the clip table
  return r;
}


// ================================================================== EPMC (PlayGroundEnv, element_id 0: flat joystick task)
// PGE = max_game_elements/playground_env.py, PR = randomizer/push_randomizer.py
void epmc_randomize_push(llq_engine& E, Env& e, int64_t gid) {   // PR:89-99
  double u[4];
  stream_uniforms(E.cfg.seed, gid, e.episode - 1, 2, (uint32_t)e.push_draws++, u);   // e.episode was advanced by epmc_reset
  double theta = 2.0 * M_PI * u[0];
  double h = E.cfg.push_h_lo + u[1] * (E.cfg.push_h_hi - E.cfg.push_h_lo);
  double v = E.cfg.push_v_lo + u[2] * (E.cfg.push_v_hi - E.cfg.push_v_lo);
  e.push_f[0] = h * std::cos(theta); e.push_f[1] = h * std::sin(theta); e.push_f[2] = v;
}

// PGE:374-447 on the flat 200 x 200 ground slab (top face z = 0) -- the only static body of element 0 besides the
// degenerate target marker (BSE:106-131 gives its collision box zero extents).
struct Box { V3 lo, hi; };
double ray_boxes(const Box* bs, int nb, V3 a, V3 b);

// EPMC corridor (elements 1-3), BSE = max_game_elements/bullet_static_entities.py: reset() -> _generate_random_width_walls
// (BSE:170-210) then _create_hurdles / _create_holes / _create_cubes(easy=True) (BSE:212-263, 308-470).  Draws come from
// Philox stream 5 in the order the reference consumes them.
struct TerrainRng {
  const llq_config& cf; int64_t gid, ep; int k = 0; double u[4] = {0, 0, 0, 0};
  double next() {
    if (k % 4 == 0) stream_uniforms(cf.seed, gid, ep, 5, (uint32_t)(k / 4), u);
    return u[k++ % 4];
  }
  double uniform(double lo, double hi) { return lo + next() * (hi - lo); }
  int randint(int lo, int hi) { return lo + (int)std::floor(next() * (hi - lo)); }
};
void add_box(Env& e, double cx, double cy, double cz, double lx, double ly, double lz) {
  if (e.n_boxes >= LLQ_MAX_BOXES) return;
  double* b = e.boxes[e.n_boxes++];
  b[0] = cx; b[1] = cy; b[2] = cz; b[3] = lx / 2; b[4] = ly / 2; b[5] = lz / 2;
}
// _create_auxiliary_obj (BSE:43-104): one cylinder of radius `ra` along y at each of the box's two x faces, on its top (flag = 1:
// hurdles BSE:360-362, cubes BSE:451-453) or bottom (flag = -1: bars BSE:418-420) edge
void add_aux_cylinders(Env& e, const double* b, double ra, double flag) {
  for (int side = -1; side <= 1; side += 2) {
    if (e.n_cyl >= 2 * LLQ_MAX_BOXES) return;
    double* c = e.cyl[e.n_cyl++];
    c[0] = b[0] + side * b[3]; c[1] = b[1]; c[2] = b[2] + flag * b[5]; c[3] = ra; c[4] = 2.0 * b[4];
  }
}
void epmc_generate_terrain(const llq_engine& E, Env& e, int64_t gid) {
  const llq_config& cf = E.cfg;
  TerrainRng R{cf, gid, e.episode - 1, 0, {0, 0, 0, 0}};
  e.n_boxes = 0;
  const double width = R.uniform(cf.wall_width_lo, cf.wall_width_hi), gap = R.uniform(cf.wall_gap_lo, cf.wall_gap_hi);   // BSE:171-174
  add_box(e, 5.0, gap / 2.0 + width / 2.0, 1.0, 200.0, width, 2.0);                                // BSE:207-210
  add_box(e, 5.0, -(gap / 2.0 + width / 2.0), 1.0, 200.0, width, 2.0);
  double cur = 0.0;
  if (cf.element_id == 1 || cf.element_id == 2) {                                                   // BSE:226-248
    const int n = R.randint(1, 10);
    for (int pass = 0; pass < 2; pass++) {
      for (int i = 0; i < n; i++) {
        if (cf.element_id == 1) {                                                                   // _generate_one_hurdle (BSE:308-363)
          const double h = R.uniform(0.05, 0.15), d = R.uniform(1.0, 3.0);
          add_box(e, cur + d / 2, 0.0, h / 2, 0.1, gap, h);
          cur += d + 0.1;
        } else {                                                                                    // _generate_one_hole (BSE:365-423)
          const double d = R.uniform(1.0, 3.0), g = R.uniform(cf.hole_gap_lo, cf.hole_gap_hi);
          add_box(e, cur + d / 2, 0.0, 0.3 / 2 + g, 0.1, gap, 0.3);
          cur += d + 0.1;
        }
      }
      if (pass == 0) { e.tgt_x = cur + R.uniform(-1.0, 1.0); e.tgt_y = 0.0; }
    }
  } else {                                                                                          // _create_cubes(easy=True) (BSE:212-224, 425-500)
    const int ns = R.randint(1, 5);
    for (int pass = 0; pass < 2; pass++) {
      for (int i = 0; i < ns; i++) {
        cur += R.uniform(0.0, 1.0);
        add_box(e, 1.75 + cur, 0.0, 0.25 / 2, 0.5, gap, 0.25);
        add_box(e, 1.0 + cur, 0.0, 0.1 / 2, 0.5, gap, 0.1);
        cur += 1.75 + 0.25;
        add_box(e, cur + 0.5, 0.0, 0.25 / 2, 0.5, gap, 0.25);
        add_box(e, cur + 1.25, 0.0, 0.1 / 2, 0.5, gap, 0.1);
        cur += 3.0;
      }
      if (pass == 0) { e.tgt_x = cur + R.uniform(-3.0, 3.0); e.tgt_y = 0.0; }
    }
  }
  e.n_cyl = 0;
  if (cf.auxiliary_radius > 0)
    for (int b = 2; b < e.n_boxes; b++) add_aux_cylinders(e, e.boxes[b], cf.auxiliary_radius, cf.element_id == 2 ? -1.0 : 1.0);
}
// perception against the ground slab + the corridor's boxes (PGE:374-447)
void epmc_drill_terrain(const Env& e, const double* st, float* percep) {
  Box bx[LLQ_MAX_BOXES + 1];
  bx[0] = {{-100, -100, -10}, {100, 100, 0}};
  for (int b = 0; b < e.n_boxes; b++) {
    const double* q = e.boxes[b];
    bx[1 + b] = {{q[0] - q[3], q[1] - q[4], q[2] - q[5]}, {q[0] + q[3], q[1] + q[4], q[2] + q[5]}};
  }
  const int nb = 1 + e.n_boxes;
  M3 R = qmat(qnormalize({st[3], st[4], st[5], st[6]}));
  V3 pos = {st[0], st[1], st[2]};
  const double yaw = std::atan2(R.m[1][0], R.m[0][0]);
  int k = 0;
  for (int a = 0; a < 25; a++) {
    const double gx = a == 24 ? 1.2 : -1.2 + a * (2.4 / 24.0);
    for (int b = 0; b < 13; b++) {
      const double gy = b == 12 ? 0.6 : -0.6 + b * (1.2 / 12.0);
      V3 t = mul(R, V3{gx, gy, 0.0}) + pos;
      const double f = ray_boxes(bx, nb, V3{t.x, t.y, 10.0}, V3{t.x, t.y, -10.0});
      percep[k++] = f < 0 ? 0.0f : (float)(10.0 + f * (-20.0));
    }
  }
  for (int r = 0; r < 128; r++) {
    const double ang = yaw + 2.0 * M_PI * (double)r / 128.0;
    V3 to = {pos.x + 20.0 * std::cos(ang), pos.y + 20.0 * std::sin(ang), pos.z};
    const double f = ray_boxes(bx, nb, pos, to);
    V3 hit = f < 0 ? V3{0, 0, 0} : pos + f * (to - pos);
    percep[k++] = (float)norm(hit - pos);
  }
  for (int a = 0; a < 25; a++) {
    const double y = a == 24 ? 0.25 : -0.25 + a * (0.5 / 24.0);
    for (int b = 0; b < 13; b++) {
      const double z = b == 12 ? 0.1 : -0.3 + b * (0.4 / 12.0);
      V3 from = mul(R, V3{0.0, y, z}) + pos, to = mul(R, V3{3.0, y, z}) + pos;
      const double f = ray_boxes(bx, nb, from, to);
      V3 hit = f < 0 ? to : from + f * (to - from);
      percep[k++] = (float)norm(hit - from);
    }
  }
  V3 d = tmul(R, V3{e.tgt_x - pos.x, e.tgt_y - pos.y, 0.0 - pos.z});
  const double n2 = std::sqrt(d.x * d.x + d.y * d.y);
  percep[778] = (float)(d.x / n2); percep[779] = (float)(d.y / n2); percep[780] = (float)e.target_spd;
}

void epmc_drill(const llq_engine& E, const Env& e, const double* st, float* percep /* 325 + 128 + 325 + 3 */) {
  if (E.cfg.element_id != 0) { epmc_drill_terrain(e, st, percep); return; }
  Q4 qb = qnormalize({st[3], st[4], st[5], st[6]});
  M3 R = qmat(qb);
  V3 pos = {st[0], st[1], st[2]};
  // percep_2d: rays straight down from z = 10 over a 25 x 13 grid: every ray hits the slab top => hit z = 0 (PGE:431-447)
  for (int i = 0; i < 325; i++) percep[i] = 0.0f;
  // percep_1d: 128 horizontal rays of 20 m at the base height never reach the slab (z0 > 0): miss => hit_pos = (0,0,0) =>
  // "distance" = |ray_from| = |base_pos| (PGE:49-53,388-394; SURVEY K8).  Below the surface the origin is inside the slab: miss too.
  float d1 = (float)norm(pos);
  for (int i = 0; i < 128; i++) percep[325 + i] = d1;
  // percep_front: 25 x 13 rays along body +x, 3 m, starting at body (0, y, z), y in [-.25,.25], z in [-.3,.1] (PGE:409-429)
  for (int i = 0; i < 25; i++) {
    double y = i == 24 ? 0.25 : -0.25 + i * (0.5 / 24.0);
    for (int j = 0; j < 13; j++) {
      double z = j == 12 ? 0.1 : -0.3 + j * (0.4 / 12.0);
      V3 from = mul(R, V3{0.0, y, z}) + pos;
      V3 to = mul(R, V3{3.0, y, z}) + pos;
      V3 hit = to;
      if (from.z > 0.0 && to.z < 0.0) {            // enters the slab through its top face
        double t = from.z / (from.z - to.z);
        hit = from + t * (to - from);
      }
      percep[453 + i * 13 + j] = (float)norm(hit - from);
    }
  }
  // target (PGE:396-400): unit xy of R^-1 (target - pos), then target_spd
  V3 d = tmul(R, V3{e.tgt_x - pos.x, e.tgt_y - pos.y, 0.0 - pos.z});
  double n2 = std::sqrt(d.x * d.x + d.y * d.y);
  percep[778] = (float)(d.x / n2); percep[779] = (float)(d.y / n2); percep[780] = (float)e.target_spd;
}

void epmc_write_obs(const llq_engine& E, Env& e, const double* st) {
  int o = 0;
  for (int h = 0; h < 3; h++)
    for (int t = 0; t < LLQ_PROP_DIM; t++) e.obs[o++] = (float)e.prop_hist[h][t];
  for (int h = 0; h < 3; h++)
    for (int t = 0; t < LLQ_ACTION_DIM; t++) e.obs[o++] = (float)e.act_hist[h][t];
  epmc_drill(E, e, st, e.obs + 135);
}

void epmc_reset(llq_engine& E, Env& e, int64_t gid) {   // PGE:196-249
  const llq_config& cf = E.cfg;
  double u[4];
  e.episode++;                                   // all streams of this episode are keyed by (episode - 1)
  stream_uniforms(cf.seed, gid, e.episode - 1, 1, 0, u);
  e.foot_mu = cf.friction_lo + u[0] * (cf.friction_hi - cf.friction_lo);                 // PGE:209-210
  e.push_draws = 0; e.cmd_draws = 0;
  e.push_count = cf.push_start_count;                                                    // PR:52-53
  e.push_f[0] = e.push_f[1] = e.push_f[2] = 0;
  if (cf.push_enabled) epmc_randomize_push(E, e, gid);                                   // PR:54
  e.cmd_freq = cf.cmd_freq_lo + (int)std::floor(u[2] * (cf.cmd_freq_hi - cf.cmd_freq_lo));   // np.random.randint (PGE:223)
  e.counter = 0; e.total_spd = 0; e.max_spd = 0; e.time = 0;
  e.reward_sum = 0; e.episode_steps = 0;
  // randomize_init_states (PGE:181-195): yaw about world z composed on the right of the stored tilt
  double st[LLQ_STATE_DIM];
  std::memcpy(st, E.init_state, sizeof(st));
  e.yaw_accum_deg = std::fmod(e.yaw_accum_deg + 360.0 * u[1], 360.0);
  double a = e.yaw_accum_deg * M_PI / 180.0;
  Q4 qr = {0, 0, std::sin(a / 2), std::cos(a / 2)};
  Q4 q0 = qnormalize({st[3], st[4], st[5], st[6]});
  Q4 qn = qmul(q0, qr);
  st[3] = qn.x; st[4] = qn.y; st[5] = qn.z; st[6] = qn.w;
  st[0] = 0.0; st[1] = 0.0; st[2] = 0.5;
  unpack_state(e, st);
  for (int s = 0; s < LLQ_MAX_SPHERES; s++) e.warm[s] = 0;
  e.tgt_x = 8.0; e.tgt_y = 0.0; e.n_boxes = 0; e.n_cyl = 0;                              // BSE:247-248, PGE:219
  if (cf.element_id != 0) epmc_generate_terrain(E, e, gid);                               // PGE:216-219
  e.last_pos_diff_len = std::sqrt((st[0] - e.tgt_x) * (st[0] - e.tgt_x) + (st[1] - e.tgt_y) * (st[1] - e.tgt_y));
  e.init_pos_diff_len = e.last_pos_diff_len;                                              // PGE:192-195
  double prop[LLQ_PROP_DIM];
  make_prop(st, prop);
  for (int h = 0; h < 3; h++) {
    std::memcpy(e.prop_hist[h], prop, sizeof(prop));
    for (int t = 0; t < 12; t++) e.act_hist[h][t] = 0;
  }
  foot_positions(E, st, e.foot_pos);
  epmc_write_obs(E, e, st);
}

double epmc_step(llq_engine& E, Env& e, int64_t gid, const float* action, bool* done, int64_t* ncr, int64_t* nlr) {   // PGE:301-358
  const llq_config& cf = E.cfg;
  e.episode_steps += 1;
  e.margin = 1e30;
  if (e.counter % e.cmd_freq == 0) {                                                     // PGE:302-317
    double u[4];
    stream_uniforms(cf.seed, gid, e.episode - 1, 3, (uint32_t)e.cmd_draws++, u);
    if (cf.element_id == 0) {
      e.target_angle = 2.0 * M_PI * u[0];
      e.tgt_x = e.pos[0] + std::cos(e.target_angle) * 100.0;
      e.tgt_y = e.pos[1] + std::sin(e.target_angle) * 100.0;
      e.last_pos_diff_len = std::sqrt((e.pos[0] - e.tgt_x) * (e.pos[0] - e.tgt_x) + (e.pos[1] - e.tgt_y) * (e.pos[1] - e.tgt_y));
    }
    e.target_spd = cf.target_spd_lo + u[1] * (cf.target_spd_hi - cf.target_spd_lo);
  }
  if (cf.element_id != 0) e.target_angle = std::atan2(e.tgt_y - e.pos[1], e.tgt_x - e.pos[0]);   // PGE:318-323 (plotting only)
  double act[12], tgt[12], tau[12];
  for (int j = 0; j < 12; j++) { act[j] = (double)action[j]; tgt[j] = e.q[j] + act[j]; }   // PGE:323-324
  bool ok = true;
  for (int s = 0; s < cf.substeps; s++) {
    for (int j = 0; j < 12; j++) {
      double tg = clampd(tgt[j], -3.0, 3.0);
      double t = cf.kp * (tg - e.q[j]) + cf.kd * (0.0 - e.qd[j]);
      tau[j] = clampd(t, -cf.max_tau, cf.max_tau);
    }
    const double* push = nullptr;
    if (cf.push_enabled) {                                                               // PR:56-87
      e.push_count += 1;
      if (e.push_count > 0) {
        if (e.push_count % cf.push_interval_steps == 0) { epmc_randomize_push(E, e, gid); e.push_count = 0; }
        if (e.push_count < cf.push_duration_steps) push = e.push_f;
      }
    }
    if (ok) ok = physics_substep(E, e, tau, ncr, nlr, push);                             // PGE:295-299
    e.time += cf.sim_dt;
  }
  double st[LLQ_STATE_DIM];
  pack_state(e, st);
  double prop[LLQ_PROP_DIM];
  make_prop(st, prop);
  std::memmove(e.prop_hist[0], e.prop_hist[1], 2 * sizeof(e.prop_hist[0]));
  std::memcpy(e.prop_hist[2], prop, sizeof(prop));
  std::memmove(e.act_hist[0], e.act_hist[1], 2 * sizeof(e.act_hist[0]));
  std::memcpy(e.act_hist[2], act, sizeof(act));
  foot_positions(E, st, e.foot_pos);
  epmc_write_obs(E, e, st);
  e.counter += 1;                                                                        // PGE:340
  // termination (PGE:360-372)
  Q4 q1 = qnormalize({st[3], st[4], st[5], st[6]});
  M3 R = qmat(q1);
  double left_z = R.m[0][2] * R.m[1][0] - R.m[1][2] * R.m[0][0];
  bool fall = left_z > std::sin(45.0 * M_PI / 180.0) || left_z < std::sin(-45.0 * M_PI / 180.0) || R.m[2][2] < std::cos(60.0 * M_PI / 180.0);
  double dx = e.tgt_x - st[0], dy = e.tgt_y - st[1];
  double plen = std::sqrt(dx * dx + dy * dy);
  bool reach = plen < 0.5;
  bool timeup = e.counter >= cf.max_steps;
  *done = fall || timeup || reach || !ok;
  // joystick reward (PGE:479-502)
  double ux = dx / plen, uy = dy / plen;
  double spd = std::fabs(st[7] * ux + st[8] * uy);
  e.total_spd += spd;
  if (spd > e.max_spd) e.max_spd = spd;
  double reward_vel = std::exp(-std::fabs(spd - e.target_spd));
  double yaw = std::atan2(R.m[1][0], R.m[0][0]);
  double reward_rot = std::exp((std::cos(yaw) * ux + std::sin(yaw) * uy - 1.0) * 5.0);
  double r = reward_vel * reward_rot / (double)cf.max_steps;
  if (cf.element_id != 0) {                                                              // _compute_avg_spd_reward (PGE:504-539)
    const double reward_dist = (plen - e.last_pos_diff_len) / e.init_pos_diff_len;
    e.last_pos_diff_len = plen;
    r = reward_rot / (double)cf.max_steps * 0.1 * 2.0 + (-reward_dist * 0.1);
    if (reach) r += std::exp(-std::fabs(e.total_spd / e.counter - e.target_spd));
  }
  if (!ok || !std::isfinite(r)) { r = 0.0; *done = true; }
  e.reward_sum += r;
  return r;
}


// ================================================================== SEPMC (ChaseTagGameEnv, empty arena)
// CTG = max_game/chase_tag_game_env.py, BSG = max_game/bullet_static_entities.py, PR = randomizer/push_randomizer.py
// closest hit of the segment a->b with a set of axis-aligned boxes (rayTest / rayTestBatch, mask 6 => statics only).
// Returns the hit fraction or -1.  A ray that starts inside a box does not hit that box (Bullet's convex cast).
double ray_boxes(const Box* bs, int nb, V3 a, V3 b) {
  double best = -1.0;
  V3 d = b - a;
  for (int i = 0; i < nb; i++) {
    const double lo[3] = {bs[i].lo.x, bs[i].lo.y, bs[i].lo.z}, hi[3] = {bs[i].hi.x, bs[i].hi.y, bs[i].hi.z};
    const double o[3] = {a.x, a.y, a.z}, dd[3] = {d.x, d.y, d.z};
    if (o[0] > lo[0] && o[0] < hi[0] && o[1] > lo[1] && o[1] < hi[1] && o[2] > lo[2] && o[2] < hi[2]) continue;
    double t0 = 0.0, t1 = 1.0; bool hit = true; int ax_in = -1;
    for (int ax = 0; ax < 3 && hit; ax++) {
      if (dd[ax] == 0.0) { if (o[ax] < lo[ax] || o[ax] > hi[ax]) hit = false; continue; }
      double ta = (lo[ax] - o[ax]) / dd[ax], tb = (hi[ax] - o[ax]) / dd[ax];
      if (ta > tb) std::swap(ta, tb);
      if (ta > t0) { t0 = ta; ax_in = ax; }
      t1 = std::min(t1, tb);
      if (t0 > t1) hit = false;
    }
    if (hit && ax_in >= 0 && (best < 0 || t0 < best)) best = t0;
  }
  return best;
}
void sepmc_boxes(double fx, double fy, Box* b /* 6 */) {
  b[0] = {{-100, -100, -10}, {100, 100, 0}};                       // ground slab (max_game/data/urdf/small_v3/plane.urdf)
  b[1] = {{-2.5, 2.495, 0}, {2.5, 2.505, 2}};                      // walls (BSG:895-902)
  b[2] = {{-2.5, -2.505, 0}, {2.5, -2.495, 2}};
  b[3] = {{2.495, -2.5, 0}, {2.505, 2.5, 2}};
  b[4] = {{-2.505, -2.5, 0}, {-2.495, 2.5, 2}};
  b[5] = {{fx - 0.05, fy - 0.05, 0}, {fx + 0.05, fy + 0.05, 0.5}};  // flag (CTG:163-190, 218-221)
}
double sphere_box_dist(V3 c, const Box& b) {
  double qx = c.x - clampd(c.x, b.lo.x, b.hi.x), qy = c.y - clampd(c.y, b.lo.y, b.hi.y), qz = c.z - clampd(c.z, b.lo.z, b.hi.z);
  return std::sqrt(qx * qx + qy * qy + qz * qz);
}
void proxy_positions(const llq_engine& E, const double* st, V3* out) {   // world positions of the model's proxies
  Kin k;
  kinematics(E.model, st, st + 3, st + 13, k);
  for (size_t i = 0; i < E.model.proxies.size(); i++) out[i] = k.pl[E.model.proxies[i].link] + mul(k.Rl[E.model.proxies[i].link], E.model.proxies[i].c);
}

struct PairContacts { bool tag; bool flag_touch[2]; };
// getContactPoints() of the last stepSimulation (CTG:426-456), with detection proxies: a robot's "body" links (legs + wheels,
// CTG:427) are represented by its hip and wheel spheres; any proxy of the other robot (or the flag box) counts as the other side.
PairContacts sepmc_contacts(const llq_engine& E, const Env& e0, const Env& e1) {
  const int np = (int)E.model.proxies.size();
  V3 p0[32], p1[32];
  double s0[LLQ_STATE_DIM], s1[LLQ_STATE_DIM];
  pack_state(e0, s0); pack_state(e1, s1);
  proxy_positions(E, s0, p0); proxy_positions(E, s1, p1);
  Box bx[6];
  sepmc_boxes(e0.flag_x, e0.flag_y, bx);
  PairContacts pc = {false, {false, false}};
  const double thr = E.cfg.contact_breaking;
  for (int r = 0; r < 2; r++) {
    const V3* mine = r == 0 ? p0 : p1; const V3* other = r == 0 ? p1 : p0;
    for (int i = 0; i < np; i++) {
      const ProxyM& pi = E.model.proxies[i];
      if (pi.kind != 1 && pi.kind != 2) continue;                                 // body_indices = leg + wheel links
      if (sphere_box_dist(mine[i], bx[5]) - pi.r < thr) pc.flag_touch[r] = true;
      if (r == 0)
        for (int j = 0; j < np; j++)
          if (norm(mine[i] - other[j]) - pi.r - E.model.proxies[j].r < thr) pc.tag = true;
    }
  }
  return pc;
}

void sepmc_randomize_push(llq_engine& E, Env& a, Env& b, int64_t gid, double* out3) {   // PR:89-99, one draw counter per pair
  double u[4];
  stream_uniforms(E.cfg.seed, gid, a.episode - 1, 2, (uint32_t)a.push_draws, u);
  a.push_draws += 1; b.push_draws = a.push_draws;
  double theta = 2.0 * M_PI * u[0];
  double h = E.cfg.push_h_lo + u[1] * (E.cfg.push_h_hi - E.cfg.push_h_lo);
  out3[0] = h * std::cos(theta); out3[1] = h * std::sin(theta); out3[2] = E.cfg.push_v_lo + u[2] * (E.cfg.push_v_hi - E.cfg.push_v_lo);
}

// CTG:495-596 for robot i of the pair
void sepmc_write_obs(const llq_engine&, Env* ev[2], const double st[2][LLQ_STATE_DIM], int i, const V3 prox[2][32], int with_flag_now[2]) {
  Env& e = *ev[i];
  const int j = 1 - i;
  float* o = e.obs;
  int k = 0;
  for (int h = 0; h < 3; h++) for (int t = 0; t < LLQ_PROP_DIM; t++) o[k++] = (float)e.prop_hist[h][t];
  for (int h = 0; h < 3; h++) for (int t = 0; t < LLQ_ACTION_DIM; t++) o[k++] = (float)e.act_hist[h][t];
  Box bx[6];
  sepmc_boxes(e.flag_x, e.flag_y, bx);                                   // flag where it stood during this step
  M3 R = qmat(qnormalize({st[i][3], st[i][4], st[i][5], st[i][6]}));
  V3 pos = {st[i][0], st[i][1], st[i][2]};
  double yaw = std::atan2(R.m[1][0], R.m[0][0]);
  // percept_2d (CTG:621-638): down rays over the 25 x 13 grid, value = hit z (0 on a miss)
  for (int a = 0; a < 25; a++) {
    double gx = a == 24 ? 1.2 : -1.2 + a * (2.4 / 24.0);
    for (int b = 0; b < 13; b++) {
      double gy = b == 12 ? 0.6 : -0.6 + b * (1.2 / 12.0);
      V3 t = mul(R, V3{gx, gy, 0.0}) + pos;
      double f = ray_boxes(bx, 6, V3{t.x, t.y, 10.0}, V3{t.x, t.y, -10.0});
      o[k++] = f < 0 ? 0.0f : (float)(10.0 + f * (-20.0));
    }
  }
  // percept_1d (CTG:529-537): 128 horizontal rays, 20 m; miss => hit_pos = (0,0,0)
  for (int r = 0; r < 128; r++) {
    double ang = yaw + 2.0 * M_PI * (double)r / 128.0;
    V3 to = {pos.x + 20.0 * std::cos(ang), pos.y + 20.0 * std::sin(ang), pos.z};
    double f = ray_boxes(bx, 6, pos, to);
    V3 hit = f < 0 ? V3{0, 0, 0} : pos + f * (to - pos);
    o[k++] = (float)norm(hit - pos);
  }
  // percept_front (CTG:598-619)
  for (int a = 0; a < 25; a++) {
    double y = a == 24 ? 0.25 : -0.25 + a * (0.5 / 24.0);
    for (int b = 0; b < 13; b++) {
      double z = b == 12 ? 0.1 : -0.3 + b * (0.4 / 12.0);
      V3 from = mul(R, V3{0.0, y, z}) + pos, to = mul(R, V3{3.0, y, z}) + pos;
      double f = ray_boxes(bx, 6, from, to);
      V3 hit = f < 0 ? to : from + f * (to - from);
      o[k++] = (float)norm(hit - from);
    }
  }
  // percept_vec: position(3), cos yaw, sin yaw
  o[k++] = (float)pos.x; o[k++] = (float)pos.y; o[k++] = (float)pos.z; o[k++] = (float)std::cos(yaw); o[k++] = (float)std::sin(yaw);
  // opponent (CTG:540-567)
  M3 Rj = qmat(qnormalize({st[j][3], st[j][4], st[j][5], st[j][6]}));
  double yawj = std::atan2(Rj.m[1][0], Rj.m[0][0]);
  V3 posj = {st[j][0], st[j][1], st[j][2]};
  V3 dpw = posj - pos;
  V3 dpl = tmul(R, dpw), vl = tmul(R, V3{st[j][7], st[j][8], st[j][9]}), wl = tmul(R, V3{st[j][10], st[j][11], st[j][12]});
  double oppo[15] = {(double)e.visible, posj.x, posj.y, posj.z, dpl.x, dpl.y, dpl.z, std::cos(yawj - yaw), std::sin(yawj - yaw),
                     vl.x, vl.y, vl.z, wl.x, wl.y, wl.z};
  for (int t = 0; t < 15; t++) o[k++] = e.visible ? (float)oppo[t] : 0.0f;
  for (int t = 0; t < 15; t++) o[k++] = (float)oppo[t];
  // flag (CTG:569-583): flag_visible is always true; position = where the flag stood during this step
  V3 fp = {e.flag_x, e.flag_y, 0.25};
  V3 fl = tmul(R, fp - pos);
  double flag[7] = {1.0, fp.x, fp.y, fp.z, fl.x, fl.y, fl.z};
  for (int rep = 0; rep < 2; rep++) for (int t = 0; t < 7; t++) o[k++] = (float)flag[t];
  // with_flag (CTG:596): [with_flag, with_flag[::-1]][i]  (after a possible switch in this step)
  o[k++] = (float)with_flag_now[i]; o[k++] = (float)with_flag_now[j];
  o[k++] = (float)e.fix_spd;                                                                // control_spd (CTG:364-365)
  (void)prox;
}

// visibility (CTG:472-493): clear root-to-root segment, else any clear head-handle -> {feet, wheels, handles} segment; and the
// bearing test against visible_angle = pi
void sepmc_visibility(const llq_engine& E, Env* ev[2], const double st[2][LLQ_STATE_DIM], const V3 prox[2][32]) {
  Box bx[6];
  sepmc_boxes(ev[0]->flag_x, ev[0]->flag_y, bx);
  V3 p[2] = {{st[0][0], st[0][1], st[0][2]}, {st[1][0], st[1][1], st[1][2]}};
  bool root_clear = ray_boxes(bx, 6, p[0], p[1]) < 0;
  const int np = (int)E.model.proxies.size();
  for (int i = 0; i < 2; i++) {
    bool vis = root_clear;
    if (!vis) {
      for (int h = 0; h < np && !vis; h++) {
        if (E.model.proxies[h].kind != 4) continue;
        // head point = the first handle (front handle, LR:154-156)
        for (int c = 0; c < np && !vis; c++) {
          int kd = E.model.proxies[c].kind;
          if (kd != 0 && kd != 1 && kd != 4) continue;                            // feet + wheels + handles (LR:150-152)
          if (ray_boxes(bx, 6, prox[i][h], prox[1 - i][c]) < 0) vis = true;
        }
        break;                                                                    // only the front handle
      }
    }
    M3 R = qmat(qnormalize({st[i][3], st[i][4], st[i][5], st[i][6]}));
    double yaw = std::atan2(R.m[1][0], R.m[0][0]);
    V3 d = p[1 - i] - p[i];
    double cv = (std::cos(yaw) * d.x + std::sin(yaw) * d.y) / std::sqrt(d.x * d.x + d.y * d.y);
    ev[i]->visible = (cv >= std::cos(M_PI) && vis) ? 1 : 0;
  }
}

void sepmc_finish_obs(llq_engine& E, Env* ev[2], int64_t gid, const PairContacts& pc, bool is_reset) {
  double st[2][LLQ_STATE_DIM];
  V3 prox[2][32];
  for (int i = 0; i < 2; i++) { pack_state(*ev[i], st[i]); proxy_positions(E, st[i], prox[i]); foot_positions(E, st[i], ev[i]->foot_pos); }
  sepmc_visibility(E, ev, st, prox);
  // flag switch (CTG:573-581): the robot that does NOT hold the flag touches it
  int wf[2] = {ev[0]->with_flag, ev[1]->with_flag};
  double nfx = ev[0]->flag_x, nfy = ev[0]->flag_y;
  int sw = 0;
  if (!is_reset && ((wf[0] && pc.flag_touch[1]) || (wf[1] && pc.flag_touch[0]))) {
    std::swap(wf[0], wf[1]);
    sw = 1;
    double u[4];
    stream_uniforms(E.cfg.seed, gid, ev[0]->episode - 1, 4, (uint32_t)ev[0]->flag_draws, u);
    ev[0]->flag_draws += 1; ev[1]->flag_draws = ev[0]->flag_draws;
    nfx = -2.0 + 4.0 * u[0]; nfy = -2.0 + 4.0 * u[1];                              // CTG:218-221
  }
  for (int i = 0; i < 2; i++) sepmc_write_obs(E, ev, st, i, prox, wf);
  for (int i = 0; i < 2; i++) { ev[i]->with_flag = wf[i]; ev[i]->switch_flag = sw; ev[i]->flag_x = nfx; ev[i]->flag_y = nfy; }
}

void sepmc_reset(llq_engine& E, Env& a, Env& b, int64_t gid) {   // CTG:261-304, 204-230
  const llq_config& cf = E.cfg;
  Env* ev[2] = {&a, &b};
  a.episode++; b.episode = a.episode;
  double u0[4], u1[4], u2[4];
  stream_uniforms(cf.seed, gid, a.episode - 1, 1, 0, u0);
  stream_uniforms(cf.seed, gid, a.episode - 1, 1, 1, u1);
  stream_uniforms(cf.seed, gid, a.episode - 1, 1, 2, u2);
  const double fix_spd = 0.5 + 2.5 * u0[0];                                               // CTG:262
  const int wflag = (int)std::floor(2.0 * u0[1]);                                         // np.random.randint(0, 2)  (CTG:266)
  const double mu = cf.friction_lo + u0[2] * (cf.friction_hi - cf.friction_lo);           // CTG:277
  const double px[2] = {-2.0 + 4.0 * u0[3], -2.0 + 4.0 * u1[1]}, py[2] = {-2.0 + 4.0 * u1[0], -2.0 + 4.0 * u1[2]};   // CTG:205-206
  const double yaws[2] = {360.0 * u1[3], 360.0 * u2[0]};
  double yaw_acc = a.yaw_accum_deg;      // get_init_states_info() hands both robots the same dict => one running yaw (CTG:209-215)
  for (int i = 0; i < 2; i++) {
    Env& e = *ev[i];
    e.fix_spd = fix_spd; e.with_flag = i == 0 ? wflag : 1 - wflag; e.switch_flag = 0; e.foot_mu = mu; e.flag_draws = 0;
    e.counter = 0; e.total_spd = 0; e.max_spd = 0; e.time = 0; e.reward_sum = 0; e.episode_steps = 0;
    e.push_count = cf.push_start_count; e.push_draws = 0;
    double st[LLQ_STATE_DIM];
    std::memcpy(st, E.init_state, sizeof(st));
    yaw_acc = std::fmod(yaw_acc + yaws[i], 360.0);
    double ang = yaw_acc * M_PI / 180.0;
    Q4 qn = qmul(qnormalize({st[3], st[4], st[5], st[6]}), Q4{0, 0, std::sin(ang / 2), std::cos(ang / 2)});
    st[3] = qn.x; st[4] = qn.y; st[5] = qn.z; st[6] = qn.w;
    st[0] = px[i]; st[1] = py[i]; st[2] = 0.5;
    unpack_state(e, st);
    e.yaw_accum_deg = yaw_acc;
    for (int s = 0; s < LLQ_MAX_SPHERES; s++) e.warm[s] = 0;
    e.flag_x = -2.0 + 4.0 * u2[1]; e.flag_y = -2.0 + 4.0 * u2[2];                          // CTG:218-221
    double prop[LLQ_PROP_DIM];
    make_prop(st, prop);
    for (int h = 0; h < 3; h++) { std::memcpy(e.prop_hist[h], prop, sizeof(prop)); for (int t = 0; t < 12; t++) e.act_hist[h][t] = 0; }
  }
  a.yaw_accum_deg = b.yaw_accum_deg;     // the accumulator is the pair's
  a.push_f[0] = a.push_f[1] = a.push_f[2] = 0; b.push_f[0] = b.push_f[1] = b.push_f[2] = 0;
  if (cf.push_enabled) { double f[3]; sepmc_randomize_push(E, a, b, gid, f); }             // PR:54: draw #0 = _randomized_force
  // reset() runs _prepare_drill too (CTG:302), whose flag-switch test reads getContactPoints(): still the manifolds of the last
  // stepSimulation of the previous episode (nothing has been stepped since)
  PairContacts stale = {false, {a.touch != 0, b.touch != 0}};
  sepmc_finish_obs(E, ev, gid, stale, false);
}

void sepmc_step(llq_engine& E, Env& a, Env& b, int64_t gid, const float* act_a, const float* act_b, double* rew2, bool* done,
                int64_t* ncr, int64_t* nlr) {   // CTG:378-424
  const llq_config& cf = E.cfg;
  Env* ev[2] = {&a, &b};
  const float* acts[2] = {act_a, act_b};
  double act[2][12], tgt[2][12];
  for (int i = 0; i < 2; i++) {
    ev[i]->episode_steps += 1; ev[i]->margin = 1e30;
    for (int j = 0; j < 12; j++) { act[i][j] = (double)acts[i][j]; tgt[i][j] = ev[i]->q[j] + act[i][j]; }   // CTG:379-380
  }
  bool ok = true;
  PairContacts pc = {false, {false, false}};
  for (int s = 0; s < cf.substeps; s++) {
    double tau[2][12];
    for (int i = 0; i < 2; i++)
      for (int j = 0; j < 12; j++) {
        double tg = clampd(tgt[i][j], -3.0, 3.0);
        tau[i][j] = clampd(cf.kp * (tg - ev[i]->q[j]) + cf.kd * (0.0 - ev[i]->qd[j]), -cf.max_tau, cf.max_tau);
      }
    // push randomiser with two robots (PR:56-87): inside the window every robot gets a freshly randomised force every sub-step
    const double* push[2] = {nullptr, nullptr};
    double pf[2][3];
    if (cf.push_enabled) {
      a.push_count += 1; b.push_count = a.push_count;
      if (a.push_count > 0) {
        double f[3];
        if (a.push_count % cf.push_interval_steps == 0) { sepmc_randomize_push(E, a, b, gid, f); a.push_count = b.push_count = 0; }
        if (a.push_count < cf.push_duration_steps) {
          // robot 0 gets the current _randomized_force = draw #(push_draws - 1); robot 1 the next draw; then one more draw
          double u[4];
          for (int i = 0; i < 2; i++) {
            stream_uniforms(cf.seed, gid, a.episode - 1, 2, (uint32_t)(a.push_draws - 1 + i), u);
            double theta = 2.0 * M_PI * u[0], h = cf.push_h_lo + u[1] * (cf.push_h_hi - cf.push_h_lo);
            pf[i][0] = h * std::cos(theta); pf[i][1] = h * std::sin(theta); pf[i][2] = cf.push_v_lo + u[2] * (cf.push_v_hi - cf.push_v_lo);
            push[i] = pf[i];
            for (int t = 0; t < 3; t++) ev[i]->push_f[t] = pf[i][t];
          }
          a.push_draws += 2; b.push_draws = a.push_draws;
        }
      }
    }
    if (s == cf.substeps - 1) {                                        // manifolds of the last stepSimulation: its pre-step poses
      pc = sepmc_contacts(E, a, b);
      a.touch = pc.flag_touch[0]; b.touch = pc.flag_touch[1];
    }
    for (int i = 0; i < 2; i++) {
      if (ok) ok = physics_substep(E, *ev[i], tau[i], ncr, nlr, push[i]);
      ev[i]->time += cf.sim_dt;
    }
  }
  for (int i = 0; i < 2; i++) {
    double st[LLQ_STATE_DIM], prop[LLQ_PROP_DIM];
    pack_state(*ev[i], st);
    make_prop(st, prop);
    std::memmove(ev[i]->prop_hist[0], ev[i]->prop_hist[1], 2 * sizeof(ev[i]->prop_hist[0]));
    std::memcpy(ev[i]->prop_hist[2], prop, sizeof(prop));
    std::memmove(ev[i]->act_hist[0], ev[i]->act_hist[1], 2 * sizeof(ev[i]->act_hist[0]));
    std::memcpy(ev[i]->act_hist[2], act[i], sizeof(act[i]));
  }
  sepmc_finish_obs(E, ev, gid, pc, false);
  for (int i = 0; i < 2; i++) {                                         // stat_spd (CTG:368-373)
    double spd = std::sqrt(ev[i]->linv[0] * ev[i]->linv[0] + ev[i]->linv[1] * ev[i]->linv[1]);
    ev[i]->total_spd += spd;
    if (spd > ev[i]->max_spd) ev[i]->max_spd = spd;
    ev[i]->counter += 1;
  }
  // termination (CTG:458-470): robot 0's fall only, time, robot-0-body contact with robot 1
  M3 R = qmat(qnormalize({a.quat[0], a.quat[1], a.quat[2], a.quat[3]}));
  double left_z = R.m[0][2] * R.m[1][0] - R.m[1][2] * R.m[0][0];
  bool fall0 = left_z > std::sin(45.0 * M_PI / 180.0) || left_z < std::sin(-45.0 * M_PI / 180.0) || R.m[2][2] < std::cos(60.0 * M_PI / 180.0);
  *done = fall0 || a.counter >= cf.max_steps || pc.tag || !ok;
  // rewards (CTG:640-652, 412-419)
  double sw = (double)a.switch_flag;
  if (a.with_flag) { rew2[0] = sw; rew2[1] = -sw; } else { rew2[0] = -sw; rew2[1] = sw; }
  if (*done && pc.tag) {
    if (a.with_flag) { rew2[0] += 1.0; rew2[1] -= 1.0; } else { rew2[0] -= 1.0; rew2[1] += 1.0; }
  }
  if (!ok) rew2[0] = rew2[1] = 0.0;                                   // a bad step pays nothing, as in PMC and EPMC
  a.reward_sum += rew2[0]; b.reward_sum += rew2[1];
}

void update_sampling(llq_engine& E) {  // PLE:239-240
  double tot = 0;
  for (int c = 0; c < E.n_clips; c++) {
    E.sample_prob[c] = std::pow(1.0 - E.avg_reward[c], E.cfg.prioritized_sample_factor);
    tot += E.sample_prob[c];
  }
  for (int c = 0; c < E.n_clips; c++) E.sample_prob[c] /= tot;
}

int check_ready(llq_handle h, bool need_reset) {
  if (!h) return fail(LLQ_EINVAL, "null handle");
  if (!h->has_model) return fail(LLQ_ESTATE, "llq_load_model has not been called");
  if (h->cfg.env_kind == LLQ_ENV_PMC && !h->has_mocap) return fail(LLQ_ESTATE, "llq_load_mocap has not been called");
  if (h->cfg.env_kind != LLQ_ENV_PMC && !h->has_init_state) return fail(LLQ_ESTATE, "llq_set_init_state has not been called");
  if (need_reset && !h->was_reset) return fail(LLQ_ESTATE, "llq_reset has not been called");
  return LLQ_OK;
}

}  // namespace

// ====================================================================== C ABI
extern "C" {

int llq_abi_version(int* is_cuda) {
  if (is_cuda) *is_cuda = 0;
  return LLQ_ABI_VERSION;
}

int llq_default_config(llq_config* c) {
  if (!c) return fail(LLQ_EINVAL, "null config");
  std::memset(c, 0, sizeof(*c));
  c->struct_size = (int32_t)sizeof(llq_config);
  c->n_envs = 1; c->device = 0; c->substeps = 10; c->solver_iters = 10; c->auto_reset = 0; c->num_threads = 0;
  c->global_env_offset = 0; c->seed = 0;
  c->sim_dt = 1.0 / 500.0; c->policy_dt = 1.0 / 50.0;
  c->kp = 50.0; c->kd = 0.5; c->max_tau = 18.0;
  c->gravity_z = -9.80665; c->ground_friction = 0.9; c->foot_friction = 0.5;
  c->contact_erp = 0.08; c->joint_erp = 0.2; c->linear_slop = 1e-5; c->warmstart = 0.1;
  c->contact_breaking = 0.02 * 0.025;
  c->lin_damping = 0.04; c->ang_damping = 0.04; c->max_coord_vel = 100.0; c->max_applied_impulse = 1000.0;
  c->w_joint_pos = 0.3; c->w_joint_vel = 0.05; c->w_end_effector = 0.1; c->w_root_pose = 0.5; c->w_root_vel = 0.05;
  c->prioritized_sample_factor = 3.0;
  // EPMC defaults = train_scripts/example_epmc_train.sh:100-117 (only used when env_kind = LLQ_ENV_EPMC)
  c->env_kind = LLQ_ENV_PMC; c->max_steps = 1000; c->cmd_freq_lo = 9999; c->cmd_freq_hi = 10000;
  c->push_start_count = -250; c->push_interval_steps = 499; c->push_duration_steps = 100; c->push_enabled = 1;
  c->friction_lo = 0.4; c->friction_hi = 3.0; c->push_h_lo = 0.0; c->push_h_hi = 50.0; c->push_v_lo = 0.0; c->push_v_hi = 10.0;
  c->target_spd_lo = 0.5; c->target_spd_hi = 3.0;
  c->element_id = 0; c->wall_width_lo = 0.02; c->wall_width_hi = 0.5; c->wall_gap_lo = 1.0; c->wall_gap_hi = 20.0;
  c->hole_gap_lo = 0.25; c->hole_gap_hi = 0.3;
  c->knee_contacts = 2; c->reserved1 = 0; c->link_friction = 0.5; c->auxiliary_radius = 0.0;
  return LLQ_OK;
}

int llq_create(const llq_config* cfg, llq_handle* out) {
  if (!cfg || !out) return fail(LLQ_EINVAL, "null argument");
  if (cfg->struct_size != (int32_t)sizeof(llq_config)) return fail(LLQ_EINVAL, "llq_config size mismatch (ABI)");
  if (cfg->n_envs <= 0) return fail(LLQ_EINVAL, "n_envs must be positive");
  if (cfg->substeps <= 0 || cfg->solver_iters < 0 || !(cfg->sim_dt > 0)) return fail(LLQ_EINVAL, "bad step configuration");
  if (cfg->env_kind != LLQ_ENV_PMC && cfg->env_kind != LLQ_ENV_EPMC && cfg->env_kind != LLQ_ENV_SEPMC) return fail(LLQ_EINVAL, "unknown env_kind");
  if (cfg->env_kind == LLQ_ENV_SEPMC && (cfg->n_envs % 2 != 0 || cfg->max_steps <= 0 || cfg->push_interval_steps <= 0))
    return fail(LLQ_EINVAL, "SEPMC: n_envs counts robots and must be even");
  if (cfg->env_kind == LLQ_ENV_EPMC && (cfg->max_steps <= 0 || cfg->cmd_freq_hi <= cfg->cmd_freq_lo || cfg->cmd_freq_lo <= 0 ||
                                        cfg->push_interval_steps <= 0))
    return fail(LLQ_EINVAL, "bad EPMC configuration");
  if (cfg->env_kind == LLQ_ENV_EPMC && (cfg->element_id < 0 || cfg->element_id > 3)) return fail(LLQ_EINVAL, "EPMC element_id must be 0..3");
  llq_engine* e = new (std::nothrow) llq_engine();
  if (!e) return fail(LLQ_ENOMEM, "out of memory");
  e->cfg = *cfg;
  e->envs.resize(cfg->n_envs);
  for (auto& en : e->envs) std::memset(&en, 0, sizeof(Env));
  *out = e;
  return LLQ_OK;
}

int llq_destroy(llq_handle h) {
  delete h;
  return LLQ_OK;
}

int llq_load_model(llq_handle h, const double* b, int64_t n) {
  if (!h || !b) return fail(LLQ_EINVAL, "null argument");
  if (n < LLQ_HDR || (int64_t)b[LLQ_H_MAGIC] != LLQ_MODEL_MAGIC || (int64_t)b[LLQ_H_TOTAL] != n)
    return fail(LLQ_EINVAL, "bad model blob (magic/size)");
  Model md;
  int nl = (int)b[LLQ_H_NLINKS];
  if (nl < 1 || nl > MAXL) return fail(LLQ_EINVAL, "unsupported link count");
  md.ndof = (int)b[LLQ_H_NDOF];
  if (md.ndof != 12) return fail(LLQ_EUNSUPPORTED, "oracle env logic expects 12 actuated joints");
  md.dof_link.assign(md.ndof, -1);
  const double* g = b + (int64_t)b[LLQ_H_OFF_GENERIC];
  for (int i = 0; i < nl; i++, g += LLQ_GL) {
    LinkM l;
    l.parent = (int)g[LLQ_G_PARENT]; l.jtype = (int)g[LLQ_G_JTYPE]; l.dof = (int)g[LLQ_G_DOF];
    l.jxyz = {g[LLQ_G_JXYZ], g[LLQ_G_JXYZ + 1], g[LLQ_G_JXYZ + 2]};
    l.jrot = from9(g + LLQ_G_JROT);
    l.axis = {g[LLQ_G_AXIS], g[LLQ_G_AXIS + 1], g[LLQ_G_AXIS + 2]};
    l.mass = g[LLQ_G_MASS];
    l.com = {g[LLQ_G_COM], g[LLQ_G_COM + 1], g[LLQ_G_COM + 2]};
    l.Rin = from9(g + LLQ_G_RIN);
    l.idiag = {g[LLQ_G_IDIAG], g[LLQ_G_IDIAG + 1], g[LLQ_G_IDIAG + 2]};
    l.lower = g[LLQ_G_LOWER]; l.upper = g[LLQ_G_UPPER]; l.jdamp = g[LLQ_G_JDAMP]; l.haslim = g[LLQ_G_HASLIM] != 0;
    if (i > 0 && (l.parent < 0 || l.parent >= i)) return fail(LLQ_EINVAL, "links must be parent-first");
    if (l.jtype == 1) {
      if (l.dof < 0 || l.dof >= md.ndof) return fail(LLQ_EINVAL, "bad dof index");
      md.dof_link[l.dof] = i;
    }
    md.links.push_back(l);
  }
  const double* s = b + (int64_t)b[LLQ_H_OFF_SPHERES];
  int ns = (int)b[LLQ_H_NSPHERES];
  if (ns > LLQ_MAX_SPHERES) return fail(LLQ_EINVAL, "too many contact spheres");
  // llq_config.knee_contacts: 0 = the foot spheres, 1 = + the knee wheels (one contact per leg), 2 = every collision sphere of the blob
  for (int i = 0; i < ns; i++, s += LLQ_SPH) {
    const int kind = (int)s[6];
    if (kind == 0) md.spheres.push_back({(int)s[0], V3{s[1], s[2], s[3]}, s[4], h->cfg.foot_friction});
    else if (h->cfg.knee_contacts == 2 || (h->cfg.knee_contacts == 1 && kind == 1))
      md.spheres.push_back({(int)s[0], V3{s[1], s[2], s[3]}, s[4], h->cfg.link_friction});
  }
  if ((int64_t)b[LLQ_H_NPROXIES] > 0) {
    const double* pr = b + (int64_t)b[LLQ_H_OFF_PROXIES];
    for (int i = 0; i < (int)b[LLQ_H_NPROXIES]; i++, pr += LLQ_PROXY)
      md.proxies.push_back({(int)pr[0], V3{pr[1], pr[2], pr[3]}, pr[4], (int)pr[5]});
  }
  h->model = md;
  h->has_model = true;
  return LLQ_OK;
}

int llq_load_mocap(llq_handle h, const double* frames, const int32_t* off, int32_t n_clips, double frame_dt) {
  if (!h || !frames || !off || n_clips <= 0 || !(frame_dt > 0)) return fail(LLQ_EINVAL, "bad mocap arguments");
  h->frame_dt = frame_dt;
  h->frame_rate = (int)(1.0 / frame_dt);                                                           // ML:34
  h->margin = (int)std::ceil(h->cfg.policy_dt / frame_dt) + h->frame_rate + 2;                     // ML:35
  h->n_clips = n_clips;
  h->clip_off.assign(off, off + n_clips + 1);
  for (int c = 0; c < n_clips; c++)
    if (off[c + 1] - off[c] < h->margin + 3) return fail(LLQ_EINVAL, "mocap clip shorter than margin + 3 frames");
  h->frames.assign(frames, frames + (size_t)off[n_clips] * LLQ_MOCAP_FRAME);
  for (int p = 0; p < 128; p++)   // replicated tail frames: a stale cursor never reads past the table
    for (int t = 0; t < LLQ_MOCAP_FRAME; t++) h->frames.push_back(frames[((size_t)off[n_clips] - 1) * LLQ_MOCAP_FRAME + t]);
  h->max_steps.resize(n_clips);
  for (int c = 0; c < n_clips; c++) h->max_steps[c] = (off[c + 1] - off[c] - h->margin) * frame_dt / h->cfg.policy_dt;  // ML:45
  h->sample_prob.assign(n_clips, 1.0 / n_clips);                                                   // ML:46
  h->avg_reward.assign(n_clips, 0.0);                                                              // PLE:133
  h->has_mocap = true;
  return LLQ_OK;
}

int llq_load_obstacles(llq_handle h, const double* table, const int32_t* offsets, int32_t n_clips, double hx, double hy, double hz) {
  if (!h || !offsets || n_clips <= 0) return fail(LLQ_EINVAL, "bad obstacle arguments");
  if (!h->has_mocap || n_clips != h->n_clips) return fail(LLQ_ESTATE, "llq_load_obstacles needs the mocap table first (same clip count)");
  if (offsets[0] != 0 || (offsets[n_clips] > 0 && !table)) return fail(LLQ_EINVAL, "bad obstacle table");
  for (int c = 0; c < n_clips; c++) if (offsets[c + 1] < offsets[c]) return fail(LLQ_EINVAL, "obstacle offsets must be non-decreasing");
  h->ob_off.assign(offsets, offsets + n_clips + 1);
  h->ob_table.assign(table, table + (size_t)offsets[n_clips] * 4);
  h->ob_half[0] = hx; h->ob_half[1] = hy; h->ob_half[2] = hz;
  h->has_obstacles = true;
  return LLQ_OK;
}

int llq_reset(llq_handle h, const uint8_t* mask, float* obs) {
  int rc = check_ready(h, false);
  if (rc) return rc;
  const int od = h->obs_dim();
  for (int i = 0; i < h->cfg.n_envs; i++) {
    if (h->cfg.env_kind == LLQ_ENV_SEPMC) {            // a pair is reset as a whole (mask of either robot)
      if (i % 2) continue;
      if (mask && !mask[i] && !mask[i + 1]) continue;
      sepmc_reset(*h, h->envs[i], h->envs[i + 1], h->cfg.global_env_offset + i);
      continue;
    }
    if (mask && !mask[i]) continue;
    if (h->cfg.env_kind == LLQ_ENV_EPMC) epmc_reset(*h, h->envs[i], h->cfg.global_env_offset + i);
    else sample_reset(*h, h->envs[i], h->cfg.global_env_offset + i);
  }
  h->was_reset = true;
  if (obs)
    for (int i = 0; i < h->cfg.n_envs; i++) std::memcpy(obs + (size_t)i * od, h->envs[i].obs, sizeof(float) * od);
  return LLQ_OK;
}

int llq_reset_to(llq_handle h, const uint8_t* mask, const int32_t* clip, const double* time, float* obs) {
  int rc = check_ready(h, false);
  if (rc) return rc;
  if (h->cfg.env_kind != LLQ_ENV_PMC) return fail(LLQ_EUNSUPPORTED, "llq_reset_to is a PMC (mocap) entry point");
  if (!clip || !time) return fail(LLQ_EINVAL, "null clip/time");
  for (int i = 0; i < h->cfg.n_envs; i++) {
    if (mask && !mask[i]) continue;
    if (clip[i] < 0 || clip[i] >= h->n_clips) return fail(LLQ_EINVAL, "clip id out of range");
    int nf = h->clip_off[clip[i] + 1] - h->clip_off[clip[i]];
    if (!(time[i] >= 0) || time[i] >= h->frame_dt * (nf - h->margin - 1)) return fail(LLQ_EINVAL, "reset time outside clip");
    reset_env(*h, h->envs[i], clip[i], time[i]);
  }
  h->was_reset = true;
  if (obs)
    for (int i = 0; i < h->cfg.n_envs; i++) std::memcpy(obs + (size_t)i * LLQ_OBS_DIM, h->envs[i].obs, sizeof(float) * LLQ_OBS_DIM);
  return LLQ_OK;
}

int llq_step_ex(llq_handle h, const float* actions, float* obs, int64_t obs_ld, float* reward, uint8_t* done, int io_mode,
                void* stream) {
  (void)stream;
  int rc = check_ready(h, true);
  if (rc) return rc;
  if (!actions) return fail(LLQ_EINVAL, "null actions");
  if (io_mode != LLQ_IO_HOST && io_mode != LLQ_IO_PINNED) return fail(LLQ_EUNSUPPORTED, "CPU oracle only takes host pointers");
  const int od = h->obs_dim();
  if (obs && obs_ld < od) return fail(LLQ_EINVAL, "obs_ld smaller than the observation width");
  const int n = h->cfg.n_envs;
  const bool epmc = h->cfg.env_kind != LLQ_ENV_PMC;   // no mocap table / sampling bookkeeping
  const bool sepmc = h->cfg.env_kind == LLQ_ENV_SEPMC;
  std::vector<double> rew(n); std::vector<uint8_t> dn(n);
  int64_t ncr = 0, nlr = 0;
#ifdef _OPENMP
  int nt = h->cfg.num_threads > 0 ? h->cfg.num_threads : omp_get_max_threads();
#pragma omp parallel for schedule(dynamic, 4) num_threads(nt) reduction(+ : ncr, nlr)
#endif
  for (int i = 0; i < n; i++) {
    bool d = false;
    if (sepmc) {
      if (i % 2) continue;
      double r2[2];
      sepmc_step(*h, h->envs[i], h->envs[i + 1], h->cfg.global_env_offset + i, actions + (size_t)i * LLQ_ACTION_DIM,
                 actions + (size_t)(i + 1) * LLQ_ACTION_DIM, r2, &d, &ncr, &nlr);
      rew[i] = r2[0]; rew[i + 1] = r2[1]; dn[i] = dn[i + 1] = d ? 1 : 0;
      continue;
    }
    if (epmc) rew[i] = epmc_step(*h, h->envs[i], h->cfg.global_env_offset + i, actions + (size_t)i * LLQ_ACTION_DIM, &d, &ncr, &nlr);
    else rew[i] = step_env(*h, h->envs[i], actions + (size_t)i * LLQ_ACTION_DIM, &d, &ncr, &nlr);
    dn[i] = d ? 1 : 0;
  }
  // prioritized-sampling bookkeeping (PLE:235-240).  Batched rule: envs are applied in index order, so the
  // highest finished env index owning a clip wins that clip's slot -- same rule as the CUDA engine.
  bool any = false;
  for (int i = 0; i < n; i++)
    if (dn[i]) {
      Env& e = h->envs[i];
      if (!epmc) h->avg_reward[e.clip] = e.reward_sum / h->max_steps[e.clip];
      any = true;
      h->counters[LLQ_CNT_EPISODES]++;
    }
  if (any && !epmc) update_sampling(*h);
  for (int i = 0; i < n; i++) {
    if (reward) reward[i] = (float)rew[i];
    if (done) done[i] = dn[i];
  }
  if (h->cfg.auto_reset)
    for (int i = 0; i < n; i++)
      if (dn[i]) {
        if (sepmc) { if (i % 2 == 0) sepmc_reset(*h, h->envs[i], h->envs[i + 1], h->cfg.global_env_offset + i); }
        else if (epmc) epmc_reset(*h, h->envs[i], h->cfg.global_env_offset + i);
        else sample_reset(*h, h->envs[i], h->cfg.global_env_offset + i);
      }
  if (obs)
    for (int i = 0; i < n; i++) std::memcpy(obs + (size_t)i * obs_ld, h->envs[i].obs, sizeof(float) * od);
  h->counters[LLQ_CNT_ENV_STEPS] += n; h->counters[LLQ_CNT_CONTACT_ROWS] += ncr; h->counters[LLQ_CNT_LIMIT_ROWS] += nlr;
  return LLQ_OK;
}

int llq_step(llq_handle h, const float* actions, float* obs, float* reward, uint8_t* done) {
  if (!h) return fail(LLQ_EINVAL, "null handle");
  return llq_step_ex(h, actions, obs, h->obs_dim(), reward, done, LLQ_IO_HOST, nullptr);
}

int llq_obs_dim(llq_handle h) { return h ? h->obs_dim() : fail(LLQ_EINVAL, "null handle"); }

int llq_set_init_state(llq_handle h, const double* st) {
  if (!h || !st) return fail(LLQ_EINVAL, "null argument");
  std::memcpy(h->init_state, st, sizeof(h->init_state));
  h->has_init_state = true;
  return LLQ_OK;
}

int llq_get_field(llq_handle h, int field, void* dst) {
  if (!h || !dst) return fail(LLQ_EINVAL, "null argument");
  const int n = h->cfg.n_envs;
  for (int i = 0; i < n; i++) {
    const Env& e = h->envs[i];
    switch (field) {
      case LLQ_F_STATE: { double st[LLQ_STATE_DIM]; pack_state(e, st); for (int t = 0; t < LLQ_STATE_DIM; t++) ((float*)dst)[(size_t)i * LLQ_STATE_DIM + t] = (float)st[t]; break; }
      case LLQ_F_KIN_STATE: for (int t = 0; t < LLQ_STATE_DIM; t++) ((float*)dst)[(size_t)i * LLQ_STATE_DIM + t] = (float)e.kin[t]; break;
      case LLQ_F_CLIP: ((int32_t*)dst)[i] = e.clip; break;
      case LLQ_F_TIME: ((double*)dst)[i] = e.time; break;
      case LLQ_F_REWARD_SUM: ((float*)dst)[i] = (float)e.reward_sum; break;
      case LLQ_F_EPISODE_STEPS: ((int32_t*)dst)[i] = e.episode_steps; break;
      case LLQ_F_WARMSTART:   // per collision sphere: the remembered normal impulse of its manifold point
        for (int t = 0; t < LLQ_MAX_SPHERES; t++) ((float*)dst)[(size_t)i * LLQ_MAX_SPHERES + t] = (float)e.warm[t];
        break;
      case LLQ_F_OBS: std::memcpy((float*)dst + (size_t)i * h->obs_dim(), e.obs, sizeof(float) * h->obs_dim()); break;
      case LLQ_F_AUX: {
        double* a = (double*)dst + (size_t)i * LLQ_AUX_DIM;
        a[LLQ_AUX_COUNTER] = e.counter; a[LLQ_AUX_TOTAL_SPD] = e.total_spd; a[LLQ_AUX_MAX_SPD] = e.max_spd;
        a[LLQ_AUX_PUSH_COUNT] = e.push_count;
        for (int t = 0; t < 3; t++) a[LLQ_AUX_PUSH_F + t] = e.push_f[t];
        a[LLQ_AUX_FOOT_FRICTION] = e.foot_mu; a[LLQ_AUX_PUSH_DRAWS] = e.push_draws; a[LLQ_AUX_YAW_ACCUM_DEG] = e.yaw_accum_deg;
        if (h->cfg.env_kind == LLQ_ENV_SEPMC) {
          a[LLQ_AUX_WITH_FLAG] = e.with_flag; a[LLQ_AUX_FLAG_X] = e.flag_x; a[LLQ_AUX_FLAG_Y] = e.flag_y; a[LLQ_AUX_CONTROL_SPD] = e.fix_spd;
          a[LLQ_AUX_OPPO_VISIBLE] = e.visible; a[LLQ_AUX_SWITCH_FLAG] = e.switch_flag; a[LLQ_AUX_FLAG_DRAWS] = e.flag_draws;
          a[LLQ_AUX_FLAG_TOUCH] = e.touch;
        } else {
          a[LLQ_AUX_CMD_FREQ] = e.cmd_freq; a[LLQ_AUX_TARGET_X] = e.tgt_x; a[LLQ_AUX_TARGET_Y] = e.tgt_y; a[LLQ_AUX_TARGET_SPD] = e.target_spd;
          a[LLQ_AUX_TARGET_ANGLE] = e.target_angle; a[LLQ_AUX_LAST_POS_DIFF_LEN] = e.last_pos_diff_len; a[LLQ_AUX_CMD_DRAWS] = e.cmd_draws;
          a[LLQ_AUX_INIT_POS_DIFF_LEN] = e.init_pos_diff_len;
        }
        break;
      }
      case LLQ_F_EPISODE_ID: ((int64_t*)dst)[i] = e.episode; break;
      case LLQ_F_FOOT_POS: for (int t = 0; t < 12; t++) ((float*)dst)[(size_t)i * 12 + t] = (float)e.foot_pos[t]; break;
      case LLQ_F_DECISION_MARGIN: ((float*)dst)[i] = (float)e.margin; break;
      case LLQ_F_OB_ID: ((int32_t*)dst)[i] = e.ob_id; break;
      case LLQ_F_NBOX: ((int32_t*)dst)[i] = e.n_boxes; break;
      case LLQ_F_BOXES:
        for (int b = 0; b < LLQ_MAX_BOXES; b++) for (int t = 0; t < 6; t++)
          ((float*)dst)[((size_t)i * LLQ_MAX_BOXES + b) * 6 + t] = b < e.n_boxes ? (float)e.boxes[b][t] : 0.0f;
        break;
      case LLQ_F_SAMPLE_PROB: case LLQ_F_AVG_REWARD: break;
      default: return fail(LLQ_EINVAL, "unknown field");
    }
  }
  if (field == LLQ_F_SAMPLE_PROB || field == LLQ_F_AVG_REWARD) {
    if (!h->has_mocap) return fail(LLQ_ESTATE, "no mocap loaded");
    const std::vector<double>& v = field == LLQ_F_SAMPLE_PROB ? h->sample_prob : h->avg_reward;
    std::memcpy(dst, v.data(), sizeof(double) * v.size());
  }
  return LLQ_OK;
}

int llq_set_field(llq_handle h, int field, const void* src) {
  if (!h || !src) return fail(LLQ_EINVAL, "null argument");
  const int n = h->cfg.n_envs;
  if (field == LLQ_F_SAMPLE_PROB || field == LLQ_F_AVG_REWARD) {
    if (!h->has_mocap) return fail(LLQ_ESTATE, "no mocap loaded");
    std::vector<double>& v = field == LLQ_F_SAMPLE_PROB ? h->sample_prob : h->avg_reward;
    std::memcpy(v.data(), src, sizeof(double) * v.size());
    return LLQ_OK;
  }
  for (int i = 0; i < n; i++) {
    Env& e = h->envs[i];
    switch (field) {
      case LLQ_F_STATE: { double st[LLQ_STATE_DIM]; for (int t = 0; t < LLQ_STATE_DIM; t++) st[t] = ((const float*)src)[(size_t)i * LLQ_STATE_DIM + t]; unpack_state(e, st); break; }
      case LLQ_F_CLIP: e.clip = ((const int32_t*)src)[i]; if (e.clip < 0 || e.clip >= h->n_clips) return fail(LLQ_EINVAL, "clip id out of range"); break;
      case LLQ_F_TIME: e.time = ((const double*)src)[i]; if (h->has_mocap) motion_set_time(*h, e, e.time); break;
      case LLQ_F_REWARD_SUM: e.reward_sum = ((const float*)src)[i]; break;
      case LLQ_F_EPISODE_STEPS: e.episode_steps = ((const int32_t*)src)[i]; break;
      case LLQ_F_WARMSTART:
        for (int t = 0; t < LLQ_MAX_SPHERES; t++) e.warm[t] = ((const float*)src)[(size_t)i * LLQ_MAX_SPHERES + t];
        break;
      case LLQ_F_EPISODE_ID: e.episode = ((const int64_t*)src)[i]; break;
      case LLQ_F_OB_ID: e.ob_id = ((const int32_t*)src)[i]; break;
      case LLQ_F_AUX: {
        const double* a = (const double*)src + (size_t)i * LLQ_AUX_DIM;
        e.counter = (int)a[LLQ_AUX_COUNTER]; e.total_spd = a[LLQ_AUX_TOTAL_SPD]; e.max_spd = a[LLQ_AUX_MAX_SPD];
        e.push_count = (int)a[LLQ_AUX_PUSH_COUNT];
        for (int t = 0; t < 3; t++) e.push_f[t] = a[LLQ_AUX_PUSH_F + t];
        e.foot_mu = a[LLQ_AUX_FOOT_FRICTION]; e.push_draws = (int)a[LLQ_AUX_PUSH_DRAWS]; e.yaw_accum_deg = a[LLQ_AUX_YAW_ACCUM_DEG];
        if (h->cfg.env_kind == LLQ_ENV_SEPMC) {
          e.with_flag = (int)a[LLQ_AUX_WITH_FLAG]; e.flag_x = a[LLQ_AUX_FLAG_X]; e.flag_y = a[LLQ_AUX_FLAG_Y]; e.fix_spd = a[LLQ_AUX_CONTROL_SPD];
          e.visible = (int)a[LLQ_AUX_OPPO_VISIBLE]; e.switch_flag = (int)a[LLQ_AUX_SWITCH_FLAG]; e.flag_draws = (int)a[LLQ_AUX_FLAG_DRAWS];
          e.touch = (int)a[LLQ_AUX_FLAG_TOUCH];
          break;
        }
        e.cmd_freq = (int)a[LLQ_AUX_CMD_FREQ]; e.tgt_x = a[LLQ_AUX_TARGET_X]; e.tgt_y = a[LLQ_AUX_TARGET_Y]; e.target_spd = a[LLQ_AUX_TARGET_SPD];
        e.target_angle = a[LLQ_AUX_TARGET_ANGLE]; e.last_pos_diff_len = a[LLQ_AUX_LAST_POS_DIFF_LEN]; e.cmd_draws = (int)a[LLQ_AUX_CMD_DRAWS];
        e.init_pos_diff_len = a[LLQ_AUX_INIT_POS_DIFF_LEN];
        if (e.cmd_freq <= 0) return fail(LLQ_EINVAL, "cmd_vary_freq must be positive");
        break;
      }
      case LLQ_F_OBS: {
        const float* o = (const float*)src + (size_t)i * h->obs_dim();
        std::memcpy(e.obs, o, sizeof(float) * h->obs_dim());
        for (int hh = 0; hh < 3; hh++) {
          for (int t = 0; t < LLQ_PROP_DIM; t++) e.prop_hist[hh][t] = o[hh * LLQ_PROP_DIM + t];
          for (int t = 0; t < LLQ_ACTION_DIM; t++) e.act_hist[hh][t] = o[3 * LLQ_PROP_DIM + hh * LLQ_ACTION_DIM + t];
        }
        break;
      }
      default: return fail(LLQ_EINVAL, "field is not settable");
    }
  }
  return LLQ_OK;
}

int llq_get_counters(llq_handle h, int64_t* out, int32_t n) {
  if (!h || !out || n < 0 || n > 8) return fail(LLQ_EINVAL, "bad arguments");
  for (int i = 0; i < n; i++) out[i] = h->counters[i];
  return LLQ_OK;
}

int llq_sync(llq_handle h) { return h ? LLQ_OK : fail(LLQ_EINVAL, "null handle"); }
int llq_host_alloc(void** out, int64_t bytes) {
  if (!out || bytes <= 0) return fail(LLQ_EINVAL, "bad arguments");
  *out = std::malloc((size_t)bytes);
  return *out ? LLQ_OK : fail(LLQ_ENOMEM, "out of memory");
}
int llq_host_free(void* p) { std::free(p); return LLQ_OK; }

int llq_set_option(llq_handle, const char*, double) { return fail(LLQ_EUNSUPPORTED, "the CPU oracle has no options"); }
int llq_get_timing(llq_handle, double*, int32_t) { return fail(LLQ_EUNSUPPORTED, "the CPU oracle has no device timing"); }

const char* llq_last_error(void) { return g_err.c_str(); }

// ---- oracle-only hooks (not part of include/llq.h): fp64 state access and a bare physics sub-step with caller-supplied
// joint torques.  tests/golden/pybullet_shim.py builds a stand-in `pybullet` module on these so that the *unmodified*
// reference PrimitiveLevelEnv / LeggedRobot / MotionLib can be executed here and their outputs frozen as golden vectors.
int llq_oracle_get_state64(llq_handle h, int32_t env, double* st37) {
  if (!h || !st37 || env < 0 || env >= h->cfg.n_envs) return fail(LLQ_EINVAL, "bad arguments");
  pack_state(h->envs[env], st37);
  return LLQ_OK;
}
int llq_oracle_set_state64(llq_handle h, int32_t env, const double* st37) {
  if (!h || !st37 || env < 0 || env >= h->cfg.n_envs) return fail(LLQ_EINVAL, "bad arguments");
  unpack_state(h->envs[env], st37);
  for (int s = 0; s < LLQ_MAX_SPHERES; s++) h->envs[env].warm[s] = 0;   // resetBasePositionAndOrientation drops the contact cache
  return LLQ_OK;
}
int llq_oracle_substep(llq_handle h, int32_t env, const double* tau12) {
  if (!h || !tau12 || env < 0 || env >= h->cfg.n_envs) return fail(LLQ_EINVAL, "bad arguments");
  if (!h->has_model) return fail(LLQ_ESTATE, "llq_load_model has not been called");
  int64_t a = 0, b = 0;
  h->envs[env].margin = 1e30;
  if (!(h->envs[env].foot_mu > 0)) h->envs[env].foot_mu = h->cfg.foot_friction;
  return physics_substep(*h, h->envs[env], tau12, &a, &b) ? LLQ_OK : fail(LLQ_ESTATE, "physics sub-step failed");
}
int llq_oracle_substep_push(llq_handle h, int32_t env, const double* tau12, const double* push_local3, double foot_mu) {
  if (!h || !tau12 || env < 0 || env >= h->cfg.n_envs) return fail(LLQ_EINVAL, "bad arguments");
  if (!h->has_model) return fail(LLQ_ESTATE, "llq_load_model has not been called");
  int64_t a = 0, b = 0;
  h->envs[env].margin = 1e30;
  h->envs[env].foot_mu = foot_mu;
  return physics_substep(*h, h->envs[env], tau12, &a, &b, push_local3) ? LLQ_OK : fail(LLQ_ESTATE, "physics sub-step failed");
}
int llq_oracle_obstacle_hit(llq_handle h, const double* st37, const double* pose_xy_yaw, const double* half3, int32_t* hit) {
  if (!h || !st37 || !pose_xy_yaw || !half3 || !hit) return fail(LLQ_EINVAL, "bad arguments");
  if (!h->has_model) return fail(LLQ_ESTATE, "llq_load_model has not been called");
  Kin k;
  kinematics(h->model, st37, st37 + 3, st37 + 13, k);
  double cy = std::cos(pose_xy_yaw[2]), sy = std::sin(pose_xy_yaw[2]);
  *hit = 0;
  for (const ProxyM& p : h->model.proxies) {
    if (p.kind > 3) continue;
    V3 w = k.pl[p.link] + mul(k.Rl[p.link], p.c);
    double dx = w.x - pose_xy_yaw[0], dy = w.y - pose_xy_yaw[1], dz = w.z;
    double bx = cy * dx + sy * dy, by = -sy * dx + cy * dy;
    double qx = bx - clampd(bx, -half3[0], half3[0]), qy = by - clampd(by, -half3[1], half3[1]), qz = dz - clampd(dz, -half3[2], half3[2]);
    if (std::sqrt(qx * qx + qy * qy + qz * qz) - p.r < h->cfg.contact_breaking) { *hit = 1; break; }
  }
  return LLQ_OK;
}
// oracle-only hook: world positions of the model's detection proxies ([n][3]) for a 37-double state; returns n through *count
int llq_oracle_proxy_positions(llq_handle h, const double* st37, double* out, int32_t max_n, int32_t* count) {
  if (!h || !st37 || !out || !count) return fail(LLQ_EINVAL, "bad arguments");
  if (!h->has_model) return fail(LLQ_ESTATE, "llq_load_model has not been called");
  const int n = (int)h->model.proxies.size();
  if (n > max_n || n > 32) return fail(LLQ_EINVAL, "proxy buffer too small");
  V3 p[32];
  proxy_positions(*h, st37, p);
  for (int i = 0; i < n; i++) { out[3 * i] = p[i].x; out[3 * i + 1] = p[i].y; out[3 * i + 2] = p[i].z; }
  *count = n;
  return LLQ_OK;
}

// oracle-only hook: replace the static boxes env `env` collides with / is seen through (the pybullet shim mirrors its body list here)
int llq_oracle_set_boxes(llq_handle h, int32_t env, const double* boxes6, int32_t n) {
  if (!h || env < 0 || env >= h->cfg.n_envs || n < 0 || n > LLQ_MAX_BOXES || (n > 0 && !boxes6)) return fail(LLQ_EINVAL, "bad arguments");
  Env& e = h->envs[env];
  e.n_boxes = n;
  for (int b = 0; b < n; b++) for (int t = 0; t < 6; t++) e.boxes[b][t] = boxes6[b * 6 + t];
  return LLQ_OK;
}

// oracle-only hook: replace the auxiliary cylinders of env `env` (the pybullet shim mirrors the ones the reference creates)
int llq_oracle_set_cylinders(llq_handle h, int32_t env, const double* cyl5, int32_t n) {
  if (!h || env < 0 || env >= h->cfg.n_envs || n < 0 || n > 2 * LLQ_MAX_BOXES || (n > 0 && !cyl5)) return fail(LLQ_EINVAL, "bad arguments");
  Env& e = h->envs[env];
  e.n_cyl = n;
  for (int c = 0; c < n; c++) for (int t = 0; t < 5; t++) e.cyl[c][t] = cyl5[c * 5 + t];
  return LLQ_OK;
}

int llq_oracle_foot_positions(llq_handle h, const double* st37, double* out12) {
  if (!h || !st37 || !out12) return fail(LLQ_EINVAL, "bad arguments");
  if (!h->has_model) return fail(LLQ_ESTATE, "llq_load_model has not been called");
  foot_positions(*h, st37, out12);
  return LLQ_OK;
}

}  // extern "C"

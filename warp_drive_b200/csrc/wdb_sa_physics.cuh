// wdb_sa_physics.cuh -- one-step physics of the single-agent classic-control envs, and the
// Ornstein-Uhlenbeck exploration step of their continuous actions, as out-of-line device
// functions shared by the stand-alone kernels (wdb_classic_control.cu, wdb_core.cu) and the
// whole-rollout kernel (wdb_sa_rollout.cu): ONE compiled body each, so the fused path
// produces the same bits as the stand-alone kernels that are pinned to the reference's numba
// binaries (tests/test_gpu_classic_control.py).  sa_env_step wraps them with each env's
// reward and done rules, and sa_check_env_arrays holds the refusals both paths make.
#pragma once
#include <math.h>

#include <type_traits>

#include "wdb_common.cuh"

namespace wdb {

// numba's `_clip(v, lo, hi)` (mountain_car_step_numba.py:5-11): two ordered tests.
static __device__ __forceinline__ double sa_clip_f64(double v, double lo, double hi) {
  if (v < lo) return lo;
  if (v > hi) return hi;
  return v;
}

// ========================================================================= CartPole
// NumbaClassicControlCartPoleEnvStep, cartpole_step_numba.py:42-75.  float32 everywhere
// except where the float64 literal 4.0/3.0 promotes (thetaacc, xacc and the two velocity
// updates).  Fused multiply-adds exactly where the reference binary has them (ptxas on
// numba's PTX, oracle/_ref/numba_cartpole.cubin): FFMA for the force sum, g*sin - cos*temp
// and the two position updates; DFMA for the two velocity updates; plain mul/div elsewhere.
static __device__ __noinline__ float4 cartpole_physics(float4 s, int action, float gravity,
                                                       float masspole, float total_mass,
                                                       float length, float polemass_length,
                                                       float force_mag, float tau) {
  const float x = s.x, x_dot = s.y, theta = s.z, theta_dot = s.w;
  const float force = (action > 0.5f) ? force_mag : -force_mag;
  const float costheta = cosf(theta), sintheta = sinf(theta);
  const float temp = __fdiv_rn(
      __fmaf_rn(__fmul_rn(polemass_length, __fmul_rn(theta_dot, theta_dot)), sintheta, force),
      total_mass);
  const float c2m = __fdiv_rn(__fmul_rn(masspole, __fmul_rn(costheta, costheta)), total_mass);
  const float torque = __fmaf_rn(gravity, sintheta, -__fmul_rn(costheta, temp));
  const double thetaacc =
      __ddiv_rn((double)torque, __dmul_rn((double)length, __dsub_rn(4.0 / 3.0, (double)c2m)));
  const double xacc = __dsub_rn(
      (double)temp,
      __ddiv_rn(__dmul_rn(__dmul_rn((double)polemass_length, thetaacc), (double)costheta),
                (double)total_mass));
  float4 n;
  n.x = __fmaf_rn(tau, x_dot, x);
  n.y = (float)__fma_rn((double)tau, xacc, (double)x_dot);
  n.z = __fmaf_rn(tau, theta_dot, theta);
  n.w = (float)__fma_rn((double)tau, thetaacc, (double)theta_dot);
  return n;
}
static __device__ __forceinline__ bool cartpole_terminated(float4 n, float theta_thr, float x_thr) {
  return (n.x < -x_thr) || (n.x > x_thr) || (n.z < -theta_thr) || (n.z > theta_thr);
}

// ===================================================================== MountainCar
// NumbaClassicControlMountainCarEnvStep, mountain_car_step_numba.py:14-70.
//   velocity += (action - 1) * force + cos(3 * position) * (-gravity)   -- all float64
//   (reference SASS: DMUL g*cos; DFMA force*(action-1) - that; DADD velocity)
//   terminated is decided on the float64 values BEFORE they are rounded into state.
static __device__ __noinline__ float2 mountain_car_physics(float2 s, int action,
                                                           float min_position,
                                                           float max_position, float max_speed,
                                                           float goal_position,
                                                           float goal_velocity, float force,
                                                           float gravity, int *terminated) {
  const double pos0 = (double)s.x;
  const double c = cos(__dmul_rn(pos0, 3.0));
  const double push = __fma_rn((double)force, (double)(long long)(action - 1),
                               -__dmul_rn((double)gravity, c));
  double vel = __dadd_rn(push, (double)s.y);
  vel = sa_clip_f64(vel, (double)(-max_speed), (double)max_speed);
  double pos = __dadd_rn(pos0, vel);
  pos = sa_clip_f64(pos, (double)min_position, (double)max_position);
  if (pos == (double)min_position && vel < 0.0) vel = 0.0;
  *terminated = (pos >= (double)goal_position && vel >= (double)goal_velocity) ? 1 : 0;
  return make_float2((float)pos, (float)vel);
}

// new state, reward and terminal flag of one continuous-action step
struct ContinuousStep {
  float2 s;
  float reward;
  int terminated;
};

// ============================================================ ContinuousMountainCar
// NumbaClassicControlContinuousMountainCarEnvStep, continuous_mountain_car_step_numba.py:
// 14-71.  force = clip(action) and force * power stay float32; the rest is float64
// (reference SASS: FMUL force*power; DFMA cos * -0.0025 + that; DADD velocity).
// reward = (terminated ? 100 : 0) - pow(action, 2) * 0.1 in float64 (:64-69).
static __device__ __noinline__ ContinuousStep continuous_mountain_car_physics(
    float2 s, float a, float min_action, float max_action, float min_position,
    float max_position, float max_speed, float goal_position, float goal_velocity,
    float power) {
  float f = a;
  if (a < min_action) f = min_action;
  else if (a > max_action) f = max_action;
  const float fp = __fmul_rn(f, power);
  const double pos0 = (double)s.x;
  const double c = cos(__dmul_rn(pos0, 3.0));
  double vel = __dadd_rn(__fma_rn(c, -0.0025, (double)fp), (double)s.y);
  vel = sa_clip_f64(vel, (double)(-max_speed), (double)max_speed);
  double pos = __dadd_rn(pos0, vel);
  pos = sa_clip_f64(pos, (double)min_position, (double)max_position);
  if (pos == (double)min_position && vel < 0.0) vel = 0.0;
  ContinuousStep r;
  r.s = make_float2((float)pos, (float)vel);
  const bool terminated = pos >= (double)goal_position && vel >= (double)goal_velocity;
  const double rew = terminated ? 100.0 : 0.0;
  r.reward = (float)__dsub_rn(rew, __dmul_rn(pow((double)a, 2.0), 0.1));
  r.terminated = terminated ? 1 : 0;
  return r;
}

// ========================================================================= Pendulum
// NumbaClassicControlPendulumEnvStep, pendulum_step_numba.py:30-72 (g = 9.81, m = l = 1,
// dt = 0.05, max_speed = 8, max_torque = 2 are module constants there, :9-14).
//   u = clip(action, -2, 2) in float64; angle_normalize(th) = ((th + pi) % 2pi) - pi in
//   float64, where NVVM lowers `%` to  a - floor(|a| / b) * b  with the sign of a restored
//   and Python's "result takes the divisor's sign" fix-up; sin(th) is the FLOAT32 routine
//   (th is float32), cos/sin(newth) the float64 ones.  FMA placement from the reference SASS:
//   costs = fma(u*u, 0.001, fma(an, an, 0.1 * (double)(thdot*thdot)))
//   newthdot = fma(fma(u, 3, 14.715 * sin(th)), dt, thdot);  newth = fma(newthdot, dt, th).
static __device__ __forceinline__ double python_mod_2pi(double a) {
  const double b = 2.0 * 3.141592653589793;
  const double q = floor(__ddiv_rn(fabs(a), b));
  double r = __fma_rn(-q, b, fabs(a));
  if (!(a >= 0.0)) r = -r;
  if (r < 0.0) r = __dadd_rn(r, b);
  return r;
}

// writes the 3-wide observation row `o` (global memory); never terminates
static __device__ __noinline__ ContinuousStep pendulum_physics(float2 s, float action,
                                                               float *o) {
  constexpr double kPi = 3.141592653589793;
  constexpr double kDt = 0.05;
  constexpr double kGain = 3 * 9.81 / (2 * 1.0);  // 3 * g / (2 * l)
  const double u = sa_clip_f64((double)action, -2.0, 2.0);
  const double th = (double)s.x, thdot = (double)s.y;
  const double an = __dsub_rn(python_mod_2pi(__dadd_rn(th, kPi)), kPi);
  const double td2 = (double)__fmul_rn(s.y, s.y);
  const double costs = __fma_rn(__dmul_rn(u, u), 0.001, __fma_rn(an, an, __dmul_rn(td2, 0.1)));
  double newthdot = __fma_rn(__fma_rn(u, 3.0, __dmul_rn((double)sinf(s.x), kGain)), kDt, thdot);
  newthdot = sa_clip_f64(newthdot, -8.0, 8.0);
  const double newth = __fma_rn(newthdot, kDt, th);
  ContinuousStep r;
  r.s = make_float2((float)newth, (float)newthdot);
  o[0] = (float)cos(newth);
  o[1] = (float)sin(newth);
  o[2] = (float)newthdot;
  r.reward = (float)(-costs);
  r.terminated = 0;
  return r;
}

// ================================================================ OU exploration
// sample_ou_process (numba_includes/core/random.py:74-105) for one action:
//   n ~ N(0, 1): `*normal` if given (test hook), else ONE Philox draw at (stream, off);
//   ou' = (1 - damping) * ou + stddev * n;  action = mean + scale * ou'.
// scale < 1e-8 is the deterministic bypass: action = mean, nothing drawn, ou' = ou.
struct OuStep {
  float action, ou;
  int draws;          // Philox draws consumed (0 or 1)
};

static __device__ __noinline__ OuStep ou_step(float mean, float ou, const float *normal,
                                              RngHeader h, unsigned long long stream,
                                              unsigned long long off, float damping,
                                              float stddev, float scale) {
  OuStep r;
  r.draws = 0;
  if (scale < 1.0e-8f) {
    r.action = mean;
    r.ou = ou;
    return r;
  }
  float nv;
  if (normal) {
    nv = *normal;
  } else {
    const uint4 d = rng_draw4(h, stream, off);
    nv = u32x2_to_normal(d.x, d.y);
    r.draws = 1;
  }
  nv = stddev * nv;
  const float s = (1.0f - damping) * ou + nv;
  r.ou = s;
  r.action = mean + scale * s;
  return r;
}

// ========================================================================== Acrobot
// NumbaClassicControlAcrobotEnvStep, acrobot_step_numba.py:24-168: RK4 (dt = 0.2) of the
// two-link dynamics `_dsdt` (:70-109), book (not "nips") version.  All link constants are
// 1.0 / 0.5 (:8-14), so the constant sub-expressions below are the values Python's left-to-
// right float64 evaluation gives.  Types per numba: the state and every k / k_update array
// are float32 (each stage is ROUNDED to float32 on store, :116-131); cos/sin of float32
// angles are the float32 routines; everything that touches a constant is float64.
struct Vec4 { float v[4]; };

static __device__ __forceinline__ Vec4 acrobot_dsdt(const Vec4 &s, double torque) {
  constexpr double kPi = 3.141592653589793;
  const float theta1 = s.v[0], theta2 = s.v[1], dtheta1 = s.v[2], dtheta2 = s.v[3];
  const double c2 = (double)cosf(theta2);
  const double s2 = (double)sinf(theta2);
  // d1 = m1*lc1^2 + m2*(l1^2 + lc2^2 + 2*l1*lc2*cos(theta2)) + I1 + I2
  const double d1 = ((0.25 + (1.25 + c2)) + 1.0) + 1.0;
  // d2 = m2*(lc2^2 + l1*lc2*cos(theta2)) + I2
  const double d2 = (0.25 + 0.5 * c2) + 1.0;
  // phi2 = m2*lc2*g*cos(theta1 + theta2 - pi/2); theta1 + theta2 is a float32 add
  const double phi2 = (1.0 * 0.5 * 9.8) * cos((double)__fadd_rn(theta1, theta2) - kPi / 2);
  const double phi1 = ((-0.5 * (double)__fmul_rn(dtheta2, dtheta2)) * s2
                       - ((double)dtheta2 * (double)dtheta1) * s2
                       + ((1.0 * 0.5 + 1.0 * 1.0) * 9.8) * cos((double)theta1 - kPi / 2))
                      + phi2;
  const double ddtheta2 =
      (torque + d2 / d1 * phi1 - (0.5 * (double)__fmul_rn(dtheta1, dtheta1)) * s2 - phi2) /
      ((0.25 + 1.0) - d2 * d2 / d1);
  const double ddtheta1 = -(d2 * ddtheta2 + phi1) / d1;
  Vec4 d;
  d.v[0] = dtheta1;
  d.v[1] = dtheta2;
  d.v[2] = (float)ddtheta1;
  d.v[3] = (float)ddtheta2;
  return d;
}

static __device__ __forceinline__ double acrobot_wrap(double x, double m, double M) {
  const double diff = M - m;
  while (x > M) x = x - diff;
  while (x < m) x = x + diff;
  return x;
}

// one RK4 step + wrap / clip; returns the new state, writes obs[6], reward and the terminal flag
static __device__ __noinline__ float4 acrobot_physics(float4 s4, int action, float *o,
                                                      float *reward, int *terminated_out) {
  constexpr double kPi = 3.141592653589793;
  constexpr double kMaxVel1 = 12.566370614359172, kMaxVel2 = 28.274333882308138;
  constexpr double kDt = 0.2, kDt2 = 0.1;
  const double torque = (double)(action - 1);  // AVAIL_TORQUE = [-1, 0, 1] (:6)
  Vec4 s; s.v[0] = s4.x; s.v[1] = s4.y; s.v[2] = s4.z; s.v[3] = s4.w;
  // rk4 (:112-134)
  const Vec4 k1 = acrobot_dsdt(s, torque);
  Vec4 u;
#pragma unroll
  for (int i = 0; i < 4; i++) u.v[i] = (float)((double)s.v[i] + (double)k1.v[i] * kDt2);
  const Vec4 k2 = acrobot_dsdt(u, torque);
#pragma unroll
  for (int i = 0; i < 4; i++) u.v[i] = (float)((double)s.v[i] + (double)k2.v[i] * kDt2);
  const Vec4 k3 = acrobot_dsdt(u, torque);
#pragma unroll
  for (int i = 0; i < 4; i++) u.v[i] = (float)((double)s.v[i] + (double)k3.v[i] * kDt);
  const Vec4 k4 = acrobot_dsdt(u, torque);
  float ns[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const double sum = (((double)k1.v[i] + 2.0 * (double)k2.v[i]) + 2.0 * (double)k3.v[i]) +
                       (double)k4.v[i];
    ns[i] = (float)((double)s.v[i] + (kDt / 6.0) * sum);
  }
  ns[0] = (float)acrobot_wrap((double)ns[0], -kPi, kPi);
  ns[1] = (float)acrobot_wrap((double)ns[1], -kPi, kPi);
  ns[2] = (float)fmin(fmax((double)ns[2], -kMaxVel1), kMaxVel1);
  ns[3] = (float)fmin(fmax((double)ns[3], -kMaxVel2), kMaxVel2);
  // _terminal (:151-153): float32 throughout
  const float c0 = cosf(ns[0]);
  const bool terminated = __fsub_rn(-c0, cosf(__fadd_rn(ns[1], ns[0]))) > 1.0f;
  *reward = terminated ? 0.0f : -1.0f;
  *terminated_out = terminated ? 1 : 0;
  // _get_ob (:156-168)
  o[0] = c0;
  o[1] = sinf(ns[0]);
  o[2] = cosf(ns[1]);
  o[3] = sinf(ns[1]);
  o[4] = ns[2];
  o[5] = ns[3];
  return make_float4(ns[0], ns[1], ns[2], ns[3]);
}

// ======================================================================== one env step
// state / observation widths per kind (WDB_SA_*); the step loads and stores a state row as
// one float2 / float4, and an observation row as one too where it is as wide as the state
constexpr int kSaStateDim[] = {4, 2, 4, 2, 2};
constexpr int kSaObsDim[] = {4, 2, 6, 2, 3};
// policy head width per kind: the discrete action count (CartPole push left / right,
// MountainCar and Acrobot -1 / 0 / +1), one tanh output for the continuous kinds
constexpr int kSaNActions[] = {2, 3, 3, 1, 1};

template <int Kind>
using SaAction = std::conditional_t<(Kind >= WDB_SA_CONTINUOUS_MOUNTAIN_CAR), float, int>;

struct SaStepOut {
  float reward;
  int done;  // 0; 1 at the episode end or a terminal state; MountainCar: 2 at the goal
};

// One step of replica `env` of env `Kind` at timestep t (already incremented): the physics
// above, then the reference kernels' reward and done rules.  `state` and `obs` are the whole
// [E, k] arrays; `p` holds the scalar arguments of the kind's wdb_*_step entry point, in its
// order.  The stand-alone step kernel and the rollout kernel both call this, so each rule is
// written once.  The observation row's address is formed after the physics call: computed
// before it, it would stay live across the call and raise the step kernels' register count.
template <int Kind>
static __device__ __forceinline__ SaStepOut sa_env_step(float *state, float *obs, int env,
                                                        SaAction<Kind> a, const float *p, int t,
                                                        int episode_length) {
  constexpr size_t kObs = kSaObsDim[Kind];
  SaStepOut r;
  if constexpr (Kind == WDB_SA_CARTPOLE) {
    // gravity, masspole, total_mass, length, polemass_length, force_mag, tau,
    // theta_threshold_radians, x_threshold
    float4 *s = reinterpret_cast<float4 *>(state);
    const float4 n = cartpole_physics(s[env], a, p[0], p[1], p[2], p[3], p[4], p[5], p[6]);
    s[env] = n;
    reinterpret_cast<float4 *>(obs)[env] = n;
    const bool terminated = cartpole_terminated(n, p[7], p[8]);
    r.reward = 1.0f;
    r.done = (t == episode_length || terminated) ? 1 : 0;
  } else if constexpr (Kind == WDB_SA_MOUNTAIN_CAR) {
    // min_position, max_position, max_speed, goal_position, goal_velocity, force, gravity
    float2 *s = reinterpret_cast<float2 *>(state);
    int terminated = 0;
    const float2 n = mountain_car_physics(s[env], a, p[0], p[1], p[2], p[3], p[4], p[5], p[6],
                                          &terminated);
    s[env] = n;
    reinterpret_cast<float2 *>(obs)[env] = n;
    r.reward = -1.0f;
    r.done = (t == episode_length) ? 1 : (terminated ? 2 : 0);  // mountain_car_step_numba.py:66-70
  } else if constexpr (Kind == WDB_SA_ACROBOT) {
    float4 *s = reinterpret_cast<float4 *>(state);
    float o6[6], reward;
    int terminated = 0;
    s[env] = acrobot_physics(s[env], a, o6, &reward, &terminated);
    float *o = obs + env * kObs;
#pragma unroll
    for (int i = 0; i < 6; i++) o[i] = o6[i];
    r.reward = reward;
    r.done = (t == episode_length || terminated) ? 1 : 0;
  } else {
    float2 *s = reinterpret_cast<float2 *>(state);
    ContinuousStep c;
    if constexpr (Kind == WDB_SA_CONTINUOUS_MOUNTAIN_CAR) {
      // min_action, max_action, min_position, max_position, max_speed, goal_position,
      // goal_velocity, power
      c = continuous_mountain_car_physics(s[env], a, p[0], p[1], p[2], p[3], p[4], p[5], p[6],
                                          p[7]);
      reinterpret_cast<float2 *>(obs)[env] = c.s;
    } else {
      static_assert(Kind == WDB_SA_PENDULUM, "unknown env kind");
      c = pendulum_physics(s[env], a, obs + env * kObs);
    }
    s[env] = c.s;
    r.reward = c.reward;
    r.done = (t == episode_length || c.terminated) ? 1 : 0;
  }
  return r;
}

// The refusals both the stand-alone step and the rollout make before a launch: an unknown
// kind, n_envs <= 0 or a NULL array is cudaErrorInvalidValue; a state row (or an observation
// row as wide as the state) that is not aligned for its vector load is
// cudaErrorMisalignedAddress.
inline int sa_check_env_arrays(int kind, int n_envs, const void *state, const void *action,
                               const void *done, const void *reward, const void *obs,
                               const void *env_timestep) {
  if (kind < WDB_SA_CARTPOLE || kind > WDB_SA_PENDULUM || n_envs <= 0 || !state || !action ||
      !done || !reward || !obs || !env_timestep)
    return (int)cudaErrorInvalidValue;
  const uintptr_t mask = kSaStateDim[kind] * sizeof(float) - 1;
  if ((uintptr_t)state & mask) return (int)cudaErrorMisalignedAddress;
  if (kSaObsDim[kind] == kSaStateDim[kind] && ((uintptr_t)obs & mask))
    return (int)cudaErrorMisalignedAddress;
  return (int)cudaSuccess;
}

}  // namespace wdb

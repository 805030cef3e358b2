// wdb_classic_control.cu -- MountainCar, ContinuousMountainCar, Acrobot and Pendulum steps
// (SURVEY section 8 row f2).  The reference has these only as numba kernels
// (example_envs/single_agent/classic_control/*/*_step_numba.py) launched as one 1-thread
// block per env; here one thread per env in 256-thread CTAs, vector state I/O.
//
// Arithmetic types are NOT the ones the Python source suggests at first sight: numba's type
// inference promotes `3 * position` (int64 * float32) and every expression touching a
// Python float literal to float64, keeps float32 where only float32 values meet, and picks
// the float32 or float64 libdevice routine by the argument type.  The types below were read
// off numba's own type annotations of the reference kernels and the fused-multiply-add
// placement off the SASS that ptxas makes of numba's PTX (the test tree compiles both from
// the reference sources; tests/test_gpu_classic_control.py runs those reference binaries
// next to these kernels).  Where a float64 result is rounded to float32 on store, a different FMA
// contraction can only matter in a 1e-8 fraction of the cases, so only the documented
// patterns are forced with intrinsics.
#include <math.h>

#include "wdb_common.cuh"
#include "wdb_sa_physics.cuh"

namespace wdb {
namespace {

constexpr int kCcThreads = 256;


// ===================================================================== MountainCar
// NumbaClassicControlMountainCarEnvStep, mountain_car_step_numba.py:14-70.
//   velocity += (action - 1) * force + cos(3 * position) * (-gravity)   -- all float64
//   (reference SASS: DMUL g*cos; DFMA force*(action-1) - that; DADD velocity)
//   terminated is decided on the float64 values BEFORE they are rounded into state.
//   done = 1 at the episode end, else 2 when the goal is reached (:66-70).
__global__ void __launch_bounds__(kCcThreads)
mountain_car_step_kernel(int n_envs, float2 *__restrict__ state, const int *__restrict__ action,
                         int *__restrict__ done, float *__restrict__ reward,
                         float2 *__restrict__ obs, float min_position, float max_position,
                         float max_speed, float goal_position, float goal_velocity,
                         float force, float gravity, int *__restrict__ env_timestep,
                         int episode_length) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  const int t = env_timestep[env] + 1;
  env_timestep[env] = t;
  int terminated = 0;
  const float2 n = mountain_car_physics(state[env], action[env], min_position, max_position,
                                        max_speed, goal_position, goal_velocity, force,
                                        gravity, &terminated);
  state[env] = n;
  obs[env] = n;
  reward[env] = -1.0f;
  if (t == episode_length) done[env] = 1;
  else if (terminated) done[env] = 2;
}

// ============================================================ ContinuousMountainCar
// continuous_mountain_car_physics (wdb_sa_physics.cuh); done = 1 at the episode end or the goal.
__global__ void __launch_bounds__(kCcThreads)
continuous_mountain_car_step_kernel(int n_envs, float2 *__restrict__ state,
                                    const float *__restrict__ action, int *__restrict__ done,
                                    float *__restrict__ reward, float2 *__restrict__ obs,
                                    float min_action, float max_action, float min_position,
                                    float max_position, float max_speed, float goal_position,
                                    float goal_velocity, float power,
                                    int *__restrict__ env_timestep, int episode_length) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  const int t = env_timestep[env] + 1;
  env_timestep[env] = t;
  const ContinuousStep r = continuous_mountain_car_physics(
      state[env], action[env], min_action, max_action, min_position, max_position, max_speed,
      goal_position, goal_velocity, power);
  state[env] = r.s;
  obs[env] = r.s;
  reward[env] = r.reward;
  if (t == episode_length || r.terminated) done[env] = 1;
}

// ========================================================================= Pendulum
// pendulum_physics (wdb_sa_physics.cuh); done = 1 at the episode end only.
__global__ void __launch_bounds__(kCcThreads)
pendulum_step_kernel(int n_envs, float2 *__restrict__ state, const float *__restrict__ action,
                     int *__restrict__ done, float *__restrict__ reward,
                     float *__restrict__ obs /*[E,1,3]*/, int *__restrict__ env_timestep,
                     int episode_length) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  const int t = env_timestep[env] + 1;
  env_timestep[env] = t;
  const ContinuousStep r = pendulum_physics(state[env], action[env], obs + (size_t)env * 3);
  state[env] = r.s;
  reward[env] = r.reward;
  if (t == episode_length) done[env] = 1;
}

// ========================================================================== Acrobot
// NumbaClassicControlAcrobotEnvStep, acrobot_step_numba.py:24-168: RK4 (dt = 0.2) of the
// two-link dynamics `_dsdt` (:70-109), book (not "nips") version.  All link constants are
// 1.0 / 0.5 (:8-14), so the constant sub-expressions below are the values Python's left-to-
// right float64 evaluation gives.  Types per numba: the state and every k / k_update array
// are float32 (each stage is ROUNDED to float32 on store, :116-131); cos/sin of float32
// angles are the float32 routines; everything that touches a constant is float64.
__global__ void __launch_bounds__(kCcThreads)
acrobot_step_kernel(int n_envs, float4 *__restrict__ state, const int *__restrict__ action,
                    int *__restrict__ done, float *__restrict__ reward,
                    float *__restrict__ obs /*[E,1,6]*/, int *__restrict__ env_timestep,
                    int episode_length) {
  const int env = blockIdx.x * blockDim.x + threadIdx.x;
  if (env >= n_envs) return;
  const int t = env_timestep[env] + 1;
  env_timestep[env] = t;
  float o6[6], rew;
  int terminated = 0;
  state[env] = acrobot_physics(state[env], action[env], o6, &rew, &terminated);
  reward[env] = rew;
  float *o = obs + (size_t)env * 6;
#pragma unroll
  for (int i = 0; i < 6; i++) o[i] = o6[i];
  if (t == episode_length || terminated) done[env] = 1;
}

inline bool misaligned(const void *p, uintptr_t mask) {
  return (reinterpret_cast<uintptr_t>(p) & mask) != 0;
}

}  // namespace
}  // namespace wdb

using namespace wdb;

WDB_API int wdb_mountain_car_step(void *stream, int n_envs, float *state, const int *action,
                                  int *done, float *reward, float *obs, float min_position,
                                  float max_position, float max_speed, float goal_position,
                                  float goal_velocity, float force, float gravity,
                                  int *env_timestep, int episode_length) {
  if (!state || !action || !done || !reward || !obs || !env_timestep || n_envs <= 0)
    return (int)cudaErrorInvalidValue;
  if (misaligned(state, 7) || misaligned(obs, 7)) return (int)cudaErrorMisalignedAddress;
  mountain_car_step_kernel<<<(n_envs + kCcThreads - 1) / kCcThreads, kCcThreads, 0,
                             as_stream(stream)>>>(
      n_envs, reinterpret_cast<float2 *>(state), action, done, reward,
      reinterpret_cast<float2 *>(obs), min_position, max_position, max_speed, goal_position,
      goal_velocity, force, gravity, env_timestep, episode_length);
  return finish_launch();
}

WDB_API int wdb_continuous_mountain_car_step(
    void *stream, int n_envs, float *state, const float *action, int *done, float *reward,
    float *obs, float min_action, float max_action, float min_position, float max_position,
    float max_speed, float goal_position, float goal_velocity, float power,
    int *env_timestep, int episode_length) {
  if (!state || !action || !done || !reward || !obs || !env_timestep || n_envs <= 0)
    return (int)cudaErrorInvalidValue;
  if (misaligned(state, 7) || misaligned(obs, 7)) return (int)cudaErrorMisalignedAddress;
  continuous_mountain_car_step_kernel<<<(n_envs + kCcThreads - 1) / kCcThreads, kCcThreads, 0,
                                        as_stream(stream)>>>(
      n_envs, reinterpret_cast<float2 *>(state), action, done, reward,
      reinterpret_cast<float2 *>(obs), min_action, max_action, min_position, max_position,
      max_speed, goal_position, goal_velocity, power, env_timestep, episode_length);
  return finish_launch();
}

WDB_API int wdb_pendulum_step(void *stream, int n_envs, float *state, const float *action,
                              int *done, float *reward, float *obs, int *env_timestep,
                              int episode_length) {
  if (!state || !action || !done || !reward || !obs || !env_timestep || n_envs <= 0)
    return (int)cudaErrorInvalidValue;
  if (misaligned(state, 7)) return (int)cudaErrorMisalignedAddress;
  pendulum_step_kernel<<<(n_envs + kCcThreads - 1) / kCcThreads, kCcThreads, 0,
                         as_stream(stream)>>>(
      n_envs, reinterpret_cast<float2 *>(state), action, done, reward, obs, env_timestep,
      episode_length);
  return finish_launch();
}

WDB_API int wdb_acrobot_step(void *stream, int n_envs, float *state, const int *action,
                             int *done, float *reward, float *obs, int *env_timestep,
                             int episode_length) {
  if (!state || !action || !done || !reward || !obs || !env_timestep || n_envs <= 0)
    return (int)cudaErrorInvalidValue;
  if (misaligned(state, 15)) return (int)cudaErrorMisalignedAddress;
  acrobot_step_kernel<<<(n_envs + kCcThreads - 1) / kCcThreads, kCcThreads, 0,
                        as_stream(stream)>>>(
      n_envs, reinterpret_cast<float4 *>(state), action, done, reward, obs, env_timestep,
      episode_length);
  return finish_launch();
}

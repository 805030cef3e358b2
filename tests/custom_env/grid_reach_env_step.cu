// A multi-agent env with MultiDiscrete((5, 3)) actions, written like reach_env_step.cu.
//
// Every agent is a point on an integer grid that moves toward the goal (0, 0):
//   pos    <- clip(pos + (a_0 - 2, a_1 - 1), -kBound, kBound)   (actions: int32 [E, N, 2])
//   reward  = -1 if pos was not the goal before the move, else 0 (and the agent stays put)
//   obs     = [(0 - x) / 6, (0 - y) / 3]
// An action outside its head's range counts as the no-op.  done when t == episode_length.

extern "C" {

#define kBound 8

__global__ void CudaGridReachEnvStep(int *pos, const int *actions, float *rewards, float *obs,
                                     int *done, int *env_timestep, int episode_length) {
  const int kEnvId = getEnvID(blockIdx.x);
  const int kThisAgentId = getAgentID(threadIdx.x, blockIdx.x, blockDim.x);
  const int t = env_timestep[kEnvId] + 1;
  if (kThisAgentId < wkNumberAgents) {
    const long long row = (long long)kEnvId * wkNumberAgents + kThisAgentId;
    int *p = pos + row * 2;
    int x = p[0], y = p[1];
    const bool at_goal = x == 0 && y == 0;
    if (!at_goal) {
      const int ax = actions[row * 2 + 0], ay = actions[row * 2 + 1];
      const int dx = (ax >= 0 && ax < 5) ? ax - 2 : 0, dy = (ay >= 0 && ay < 3) ? ay - 1 : 0;
      x = min(max(x + dx, -kBound), kBound);
      y = min(max(y + dy, -kBound), kBound);
      p[0] = x;
      p[1] = y;
    }
    rewards[row] = at_goal ? 0.0f : -1.0f;
    obs[row * 2 + 0] = (float)(-x) / 6.0f;
    obs[row * 2 + 1] = (float)(-y) / 3.0f;
  }
  __sync_env_threads();
  if (kThisAgentId == 0) {
    env_timestep[kEnvId] = t;
    if (t == episode_length) done[kEnvId] = 1;
  }
}

}  // extern "C"

// A memory test written like grid_reach_env_step.cu: Discrete(2) actions, observations
// [cue, flag].
//
// An episode is episode_length (>= 3) steps.  The observation after reset is [0, 0].  The first
// step draws a cue c in {0, 1} per agent (a hash of env, agent and the env's draw counter, which
// no reset restores) and shows it once: obs = [2c - 1, 1].  Every later observation is [0, 0].
// The last step pays 1 if its action equals c, 0 otherwise; every other step pays 0.  The last
// action is chosen after two or more blank observations, so a policy without memory cannot
// expect more than 1/2.
extern "C" {

__device__ __forceinline__ unsigned int recall_hash(unsigned int x) {   // lowbias32
  x ^= x >> 16;
  x *= 0x7feb352dU;
  x ^= x >> 15;
  x *= 0x846ca68bU;
  x ^= x >> 16;
  return x;
}

__global__ void CudaRecallEnvStep(int *cue, int *draws, const int *actions, float *rewards,
                                  float *obs, int *done, int *env_timestep, int episode_length) {
  const int kEnvId = getEnvID(blockIdx.x);
  const int kThisAgentId = getAgentID(threadIdx.x, blockIdx.x, blockDim.x);
  const int t = env_timestep[kEnvId] + 1;
  if (kThisAgentId < wkNumberAgents) {
    const long long row = (long long)kEnvId * wkNumberAgents + kThisAgentId;
    float o0 = 0.0f, o1 = 0.0f, r = 0.0f;
    if (t == 1) {
      const unsigned int key = (unsigned int)(kEnvId * 977 + kThisAgentId * 7919) ^
                               recall_hash((unsigned int)draws[kEnvId] + 0x9e3779b9U);
      const int c = (int)(recall_hash(key) >> 31);
      cue[row] = c;
      o0 = c ? 1.0f : -1.0f;
      o1 = 1.0f;
    }
    if (t == episode_length) r = actions[row] == cue[row] ? 1.0f : 0.0f;
    rewards[row] = r;
    obs[row * 2 + 0] = o0;
    obs[row * 2 + 1] = o1;
  }
  __sync_env_threads();
  if (kThisAgentId == 0) {
    env_timestep[kEnvId] = t;
    if (t == 1) draws[kEnvId] += 1;
    if (t == episode_length) done[kEnvId] = 1;
  }
}

}  // extern "C"

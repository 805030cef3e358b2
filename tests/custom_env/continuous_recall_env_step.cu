// A memory test with Box actions, written like recall_env_step.cu: Box(-1, 1, (2,)) actions,
// observations [c_x, c_y, flag].
//
// An episode is episode_length (>= 3) steps.  The observation after reset is [0, 0, 0].  The
// first step draws a cue c per agent, uniform on the circle of radius kRadius: the angle is
// 2 pi u with u = (h >> 8) * 2^-24 and h a hash of env, agent and the env's draw counter (which
// no reset restores), as RecallEnv draws its cue.  That step shows it once: obs = [c_x, c_y, 1].
// Every later observation is [0, 0, 0].  The last step pays -|clip(a, -1, 1) - c|; every other
// step pays 0.  The last action is chosen after two or more blank observations, so a policy
// without memory cannot expect more than -kRadius (the origin minimises the expected distance
// to a point drawn uniformly on a circle around it).
extern "C" {

#define kRadius 0.8f

__device__ __forceinline__ unsigned int continuous_recall_hash(unsigned int x) {   // lowbias32
  x ^= x >> 16;
  x *= 0x7feb352dU;
  x ^= x >> 15;
  x *= 0x846ca68bU;
  x ^= x >> 16;
  return x;
}

__global__ void CudaContinuousRecallEnvStep(float *cue, int *draws, const float *actions,
                                            float *rewards, float *obs, int *done,
                                            int *env_timestep, int episode_length) {
  const int kEnvId = getEnvID(blockIdx.x);
  const int kThisAgentId = getAgentID(threadIdx.x, blockIdx.x, blockDim.x);
  const int t = env_timestep[kEnvId] + 1;
  if (kThisAgentId < wkNumberAgents) {
    const long long row = (long long)kEnvId * wkNumberAgents + kThisAgentId;
    float o0 = 0.0f, o1 = 0.0f, o2 = 0.0f, r = 0.0f;
    if (t == 1) {
      const unsigned int key = (unsigned int)(kEnvId * 977 + kThisAgentId * 7919) ^
                               continuous_recall_hash((unsigned int)draws[kEnvId] + 0x9e3779b9U);
      const float u = (float)(continuous_recall_hash(key) >> 8) * 5.9604645e-8f;   // 2^-24
      float s, c;
      sincosf(6.2831853f * u, &s, &c);
      cue[row * 2 + 0] = kRadius * c;
      cue[row * 2 + 1] = kRadius * s;
      o0 = kRadius * c;
      o1 = kRadius * s;
      o2 = 1.0f;
    }
    if (t == episode_length) {
      const float dx = fminf(fmaxf(actions[row * 2 + 0], -1.0f), 1.0f) - cue[row * 2 + 0];
      const float dy = fminf(fmaxf(actions[row * 2 + 1], -1.0f), 1.0f) - cue[row * 2 + 1];
      r = -sqrtf(dx * dx + dy * dy);
    }
    rewards[row] = r;
    obs[row * 3 + 0] = o0;
    obs[row * 3 + 1] = o1;
    obs[row * 3 + 2] = o2;
  }
  __sync_env_threads();
  if (kThisAgentId == 0) {
    env_timestep[kEnvId] = t;
    if (t == 1) draws[kEnvId] += 1;
    if (t == episode_length) done[kEnvId] = 1;
  }
}

}  // extern "C"

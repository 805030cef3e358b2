// A custom env whose agents are not alike, written like masked_counter_env_step.cu.
//
// Agent 0 is a planner (with_planner = 1): MultiDiscrete([3, 5]) actions (move its level down /
// keep it / move it up; announce a value) and a Dict observation {"state", "action_mask"}.
// Its level stays in 0..4 and it may only announce a value <= its level, so which actions are
// valid depends on its state; an invalid action leaves the level as it was (or announces 0)
// and is counted in invalid_actions[0], an array no reset touches.
//   planner reward = the value announced
//   planner state  = [level, announced, episode_length - t]
//   planner mask   = [level > 0, 1, level < 4 | j <= level for j = 0..4] (int32, 1 = valid)
// Agents 1..N-1 (every agent when with_planner = 0) are workers: Discrete(4) actions and a Box
// observation of shape (2, 3).  Each worker owns a phase in 0..3 that its observation shows as
// two bits.
//   worker reward = 1 if the action equals the phase, else 0
//   phase        <- (phase + 1 + announced) % 4
//   worker obs    = [[phase & 1, phase >> 1, 1], [level, announced, worker % 3]]
// written agent-first ([E, Nw, 2, 3]) or agent-last ([E, 2, 3, Nw], agents_last = 1).
// The planner's step arrays hold one agent, so both layouts are the same memory for them.
// Every value is a small integer, so a NumPy twin (hetero_env.py) reproduces it exactly.
// done when t == episode_length.

extern "C" {

__global__ void CudaHeteroEnvStep(int *level, int *announced, int *phase,
                                  const int *planner_actions, const int *worker_actions,
                                  int *done, float *planner_rewards, float *worker_rewards,
                                  float *planner_state, int *planner_mask, float *worker_obs,
                                  int *invalid_actions, int *env_timestep, int episode_length,
                                  int with_planner, int agents_last) {
  const int kEnvId = getEnvID(blockIdx.x);
  const int kThisAgentId = getAgentID(threadIdx.x, blockIdx.x, blockDim.x);
  const int t = env_timestep[kEnvId] + 1;
  const int n_workers = wkNumberAgents - with_planner;
  if (with_planner && kThisAgentId == 0) {
    const int lv = level[kEnvId];
    const int move = planner_actions[kEnvId * 2 + 0], say = planner_actions[kEnvId * 2 + 1];
    int next = lv + move - 1, value = say, invalid = 0;
    if (next < 0 || next > 4) {
      next = lv;
      invalid++;
    }
    if (say > lv) {
      value = 0;
      invalid++;
    }
    if (invalid) atomicAdd(invalid_actions, invalid);
    level[kEnvId] = next;
    announced[kEnvId] = value;
    planner_rewards[kEnvId] = (float)value;
    planner_state[kEnvId * 3 + 0] = (float)next;
    planner_state[kEnvId * 3 + 1] = (float)value;
    planner_state[kEnvId * 3 + 2] = (float)(episode_length - t);
    int *mask = planner_mask + kEnvId * 8;
    mask[0] = next > 0;
    mask[1] = 1;
    mask[2] = next < 4;
    for (int j = 0; j < 5; j++) mask[3 + j] = j <= next;
  }
  __sync_env_threads();
  const int w = kThisAgentId - with_planner;
  if (w >= 0 && kThisAgentId < wkNumberAgents) {
    const int lv = with_planner ? level[kEnvId] : 0;
    const int value = with_planner ? announced[kEnvId] : 0;
    const int idx = kEnvId * n_workers + w;
    const int ph = phase[idx];
    worker_rewards[idx] = worker_actions[idx] == ph ? 1.0f : 0.0f;
    const int next = (ph + 1 + value) % 4;
    phase[idx] = next;
    const float obs[6] = {(float)(next & 1), (float)(next >> 1), 1.0f,
                          (float)lv, (float)value, (float)(w % 3)};
    for (int c = 0; c < 6; c++) {
      const long long at = agents_last ? ((long long)kEnvId * 6 + c) * n_workers + w
                                       : (long long)idx * 6 + c;
      worker_obs[at] = obs[c];
    }
  }
  if (kThisAgentId == 0) {
    env_timestep[kEnvId] = t;
    if (t == episode_length) done[kEnvId] = 1;
  }
}

}  // extern "C"

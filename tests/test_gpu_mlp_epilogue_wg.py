"""The sampling policy forward (wdb_mlp_policy_forward_sampled) runs its output epilogue in a
warpgroup of its own: two MMA warpgroups hand each tile's logits to it through a
single-buffered staging buffer per warpgroup.  The handoff is exercised at every
tile-ownership edge: rows < 64, an empty second half of the last tile, a CTA whose tiles end
on a half-tile, CTAs with a single tile next to CTAs with two.  Both entries (fp32
observations and bf16 obs tiles), bit for bit: the probabilities and values are the plain
FastShape forward's, the actions are what the reference's search picks on the float32 CDF of
those probabilities (uniforms on CDF entries and above the float32 total included), and with
an RNG state every drawing stream advances by exactly one.  Every launch must leave the guard
row past `rows` untouched."""
import ctypes

import numpy as np
import pytest

from test_gpu_forward_sampling import _cdf32, _search_index
from test_gpu_mlp_tile_edges import SENTINEL, SHAPE, _fastshape, _outputs, _setup

pytestmark = pytest.mark.gpu

N_AGENTS, SLOT_AGENT = 3, 2      # one policy agent (slot 0) of three per env: row r is agent 3 r + 2

# (rows, max_ctas): max_ctas 0 = one CTA per tile; 3 * 128 + 1 rows on 3 CTAs leaves CTA 0 two
# tiles (the second a single row) and CTAs 1 and 2 one tile each
CASES = ([(r, 0) for r in (1, 63, 64, 65, 127, 128, 129)]
         + [(129, 1), (3 * 128 + 1, 3), (3 * 128 + 64, 3), (7 * 128 + 65, 4), (2 * 132 * 128 + 1, 0)])


def _sampled(rows, max_ctas, entry, uniforms=None, rng_state=None):
    import torch

    from warp_drive_b200 import lib as wlib

    s = _setup()
    L = s["lib"]
    F, H, A0, A1 = SHAPE
    p0, p1, v = _outputs(rows)
    acts = torch.full((rows + 1, 2), -7, dtype=torch.int32, device="cuda")
    agent = torch.tensor([SLOT_AGENT], dtype=torch.int32, device="cuda")
    smp = wlib.MlpSampling()
    smp.actions, smp.agent_of_slot = wlib.ptr(acts), wlib.ptr(agent)
    smp.uniforms = wlib.ptr(uniforms) if uniforms is not None else None
    smp.rng_state = wlib.ptr(rng_state) if rng_state is not None else None
    smp.n_agents, smp.n_policy_agents = N_AGENTS, 1
    st = wlib.stream_ptr()
    x = s["x"]
    wlib.check(L.wdb_set_option(b"mlp_max_ctas", max_ctas), "set_option")
    try:
        if entry == "fp32":
            inp, is_tiles = x, 0
        else:
            inp = torch.zeros(int(L.wdb_mlp_obs_tiles_bytes(F, rows)), dtype=torch.uint8,
                              device="cuda")
            wlib.check(L.wdb_mlp_pack_obs(st, wlib.ptr(x), rows, F, wlib.ptr(inp)),
                       "mlp_pack_obs")
            is_tiles = 1
        wlib.check(L.wdb_mlp_policy_forward_sampled(
            st, wlib.ptr(s["blob"]), F, H, A0, A1, wlib.ptr(inp), is_tiles, rows, wlib.ptr(p0),
            wlib.ptr(p1), wlib.ptr(v), ctypes.byref(smp)), "mlp_policy_forward_sampled")
    finally:
        wlib.check(L.wdb_set_option(b"mlp_max_ctas", 0), "set_option")
    torch.cuda.synchronize()
    return p0, p1, v, acts


@pytest.mark.parametrize("entry", ("fp32", "tiles"))
@pytest.mark.parametrize("rows,max_ctas", CASES)
def test_epilogue_warpgroup_matches_the_plain_forward_and_search(wdb_lib, rows, max_ctas, entry):
    import torch

    want = _fastshape(rows, max_ctas, entry)
    torch.cuda.synchronize()
    gen = torch.Generator(device="cuda").manual_seed(rows)
    u = torch.rand((rows, N_AGENTS, 2), generator=gen, device="cuda")
    cdfs = [_cdf32(want[h][:rows].cpu().numpy()) for h in range(2)]
    for h in range(2):
        # every third row's uniform sits exactly on a CDF entry; the last row's is 1.0
        k = torch.randint(0, 21, (rows,), generator=gen, device="cuda")
        exact = torch.from_numpy(cdfs[h]).cuda().gather(1, k[:, None])[:, 0]
        uh = torch.where(torch.arange(rows, device="cuda") % 3 == 0, exact, u[:, SLOT_AGENT, h])
        uh[-1] = 1.0
        u[:, SLOT_AGENT, h] = uh
    got = _sampled(rows, max_ctas, entry, uniforms=u)
    for name, a, b in zip(("probs0", "probs1", "values"), got[:3], want):
        assert torch.equal(a, b), (name, rows, max_ctas)
    acts = got[3].cpu().numpy()
    for h in range(2):
        pick = _search_index(cdfs[h], u[:, SLOT_AGENT, h].cpu().numpy())
        assert np.array_equal(acts[:rows, h], pick), (h, int((acts[:rows, h] != pick).sum()))
    assert (acts[rows] == -7).all()
    for t in got[:3]:
        assert (t[rows] == SENTINEL).all()


@pytest.mark.parametrize("entry", ("fp32", "tiles"))
@pytest.mark.parametrize("rows,max_ctas", [(65, 0), (3 * 128 + 1, 3), (7 * 128 + 65, 4)])
def test_epilogue_warpgroup_advances_each_stream_once(wdb_lib, rows, max_ctas, entry):
    """With an RNG state, the stream of every row's agent advances by one and no other moves;
    the probabilities stay the plain forward's and the actions are valid."""
    import torch

    from warp_drive_b200 import lib as wlib

    want = _fastshape(rows, max_ctas, entry)
    L = _setup()["lib"]
    n = rows * N_AGENTS
    state = torch.zeros(int(L.wdb_rng_state_bytes(n)), dtype=torch.uint8, device="cuda")
    wlib.check(L.wdb_rng_init(wlib.stream_ptr(), wlib.ptr(state), n, 77), "rng_init")
    torch.cuda.synchronize()
    before = state[16:].view(torch.int64).clone()
    got = _sampled(rows, max_ctas, entry, rng_state=state)
    for name, a, b in zip(("probs0", "probs1", "values"), got[:3], want):
        assert torch.equal(a, b), (name, rows, max_ctas)
    moved = (state[16:].view(torch.int64) - before).view(rows, N_AGENTS).cpu().numpy()
    expect = np.zeros_like(moved)
    expect[:, SLOT_AGENT] = 1
    assert np.array_equal(moved, expect)
    acts = got[3][:rows].cpu().numpy()
    assert ((acts >= 0) & (acts < 21)).all()

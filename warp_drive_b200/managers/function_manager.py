"""CUDAFunctionManager / CUDAFunctionFeed / CUDASampler / CUDAEnvironmentReset /
CUDALogController on top of libwdb200.so.

Public contract of the reference's managers (warp_drive/managers/function_manager.py:
21-422 and pycuda_managers/pycuda_function_manager.py:43-753): kernels are looked up BY
NAME and called with the reference's positional argument lists, either pycuda-style
`f(*args, block=..., grid=...)` or numba-style `f[grid, block](*args)`.  Instead of
nvcc-JIT-compiling a module per (n_envs, n_agents) and cuModuleLoad-ing it, names resolve
to adapters that forward to the prebuilt C ABI (include/wdb200.h); sizes are run-time
arguments so nothing is recompiled per shape.
"""
import ctypes
import logging
import os
import time
from typing import Optional

import numpy as np
import torch

from warp_drive_b200 import lib as _libmod
from warp_drive_b200.managers.data_manager import CUDADataManager
from warp_drive_b200.utils.data_feed import DataFeed

_P = _libmod.ptr


def _scalar(v):
    if isinstance(v, (np.generic,)):
        return v.item()
    if torch.is_tensor(v):
        return v.item()
    return v


def _stream():
    return _libmod.stream_ptr()


# ------------------------------------------------------------------------------ adapters
# Each adapter receives the reference kernel's positional arguments.

def _k_tag_continuous_step(fm, a, block, grid, n_envs=None):
    # CudaTagContinuousStep(...) -- tag_continuous_step_pycuda.cu:351-385
    # n_envs: step only that many replicas (the per-env arrays passed are slices: env replicas
    # are independent, EnvWrapper.step_with_host_buffers pipelines groups of them)
    assert len(a) == 33, f"CudaTagContinuousStep takes 33 arguments, got {len(a)}"
    L = _libmod.load()
    _libmod.check(L.wdb_tag_continuous_step(
        _stream(), fm._num_envs if n_envs is None else int(n_envs), int(_scalar(a[31])),
        fm._blocks_per_env,
        _P(a[0]), _P(a[1]), _P(a[2]), _P(a[3]), _P(a[4]), _P(a[5]), _P(a[6]),
        float(_scalar(a[7])), float(_scalar(a[8])), _P(a[9]), _P(a[10]),
        float(_scalar(a[11])), int(_scalar(a[12])), _P(a[13]), int(_scalar(a[14])),
        _P(a[15]), int(_scalar(a[16])), _P(a[17]), _P(a[18]), _P(a[19]), _P(a[20]),
        _P(a[21]), _P(a[22]), _P(a[23]), _P(a[24]), float(_scalar(a[25])),
        float(_scalar(a[26])), float(_scalar(a[27])), float(_scalar(a[28])), _P(a[29]),
        _P(a[30]), int(_scalar(a[32])), _P(fm.stats_tensor),
    ), "CudaTagContinuousStep")


def _k_tag_gridworld_step(fm, a, block, grid):
    # CudaTagGridWorldStep(...) -- tag_gridworld_step_pycuda.cu:112-129
    assert len(a) == 14, f"CudaTagGridWorldStep takes 14 arguments, got {len(a)}"
    table = fm.shared_constant_tensor("kIndexToActionArr")
    L = _libmod.load()
    _libmod.check(L.wdb_tag_gridworld_step(
        _stream(), fm._num_envs, fm._num_agents, _P(a[0]), _P(a[1]), _P(a[2]), _P(a[3]),
        _P(a[4]), _P(a[5]), float(_scalar(a[6])), float(_scalar(a[7])),
        float(_scalar(a[8])), float(_scalar(a[9])), int(_scalar(a[10])),
        int(_scalar(a[11])), _P(a[12]), int(_scalar(a[13])), _P(table),
    ), "CudaTagGridWorldStep")


def _k_single_agent_step(lib_fn, n_scalars, float_actions=False):
    """Adapter of a Numba...EnvStep kernel of a single-agent env (cartpole_step_numba.py:7-23
    and the other *_step_numba.py): state, actions, done, rewards, observations, the env's
    `n_scalars` float constants, timestep, episode_length."""
    n_args = 7 + n_scalars

    def adapter(fm, a, block, grid):
        assert len(a) == n_args, f"{lib_fn} takes {n_args} arguments, got {len(a)}"
        if float_actions:
            t = a[1].tensor if hasattr(a[1], "tensor") else a[1]
            if torch.is_tensor(t) and t.dtype != torch.float32:
                raise TypeError(f"{lib_fn} takes continuous float32 actions, got {t.dtype}")
        _libmod.check(getattr(_libmod.load(), lib_fn)(
            _stream(), fm._num_envs, *[_P(v) for v in a[:5]],
            *[float(_scalar(v)) for v in a[5:5 + n_scalars]], _P(a[5 + n_scalars]),
            int(_scalar(a[6 + n_scalars])),
        ), lib_fn)

    return adapter


def _k_testkernel(fm, a, block, grid):
    # testkernel(x, y, done, actions, multiplier, target, step, episode_length)
    assert len(a) == 8
    L = _libmod.load()
    _libmod.check(L.wdb_testkernel(
        _stream(), fm._num_envs, fm._num_agents, _P(a[0]), _P(a[1]), _P(a[2]), _P(a[3]),
        float(_scalar(a[4])), int(_scalar(a[5])), int(_scalar(a[6])), int(_scalar(a[7])),
    ), "testkernel")


def _one_array_reset(fm, data, ref, done, elems_per_env, force_reset):
    desc = (_libmod.ResetDesc * 1)()
    desc[0].dst = _P(data)
    desc[0].ref = _P(ref)
    desc[0].bytes_per_env = 4 * int(elems_per_env)
    desc[0].pool_rows = 0
    raw = np.frombuffer(desc, dtype=np.uint8).copy()
    table = torch.from_numpy(raw).to(fm.device)
    fm._keepalive.append(table)
    if len(fm._keepalive) > 64:
        torch.cuda.current_stream().synchronize()
        del fm._keepalive[:-1]
    L = _libmod.load()
    dummy_t = fm.scratch_int(fm._num_envs)
    _libmod.check(L.wdb_reset_when_done(
        _stream(), _P(table), 1, _P(done), _P(dummy_t), fm._num_envs,
        int(_scalar(force_reset)), 0, None), "reset_when_done")


def _k_reset_2d(fm, a, block, grid):
    # reset_in_{float,int}_when_done_2d(data, ref, done, feature_dim, force_reset)
    _one_array_reset(fm, a[0], a[1], a[2], int(_scalar(a[3])), a[4])


def _k_reset_3d(fm, a, block, grid):
    # reset_in_{float,int}_when_done_3d(data, ref, done, agent_dim, feature_dim, force)
    _one_array_reset(fm, a[0], a[1], a[2], int(_scalar(a[3])) * int(_scalar(a[4])), a[5])


def _k_undo(fm, a, block, grid):
    # undo_done_flag_and_reset_timestep(done, timestep, force_reset)
    L = _libmod.load()
    _libmod.check(L.wdb_reset_when_done(
        _stream(), None, 0, _P(a[0]), _P(a[1]), fm._num_envs, int(_scalar(a[2])), 1,
        None), "undo_done_flag_and_reset_timestep")


def _k_reset_log_mask(fm, a, block, grid):
    _libmod.check(_libmod.load().wdb_reset_log_mask(_stream(), _P(a[0]), int(_scalar(a[1]))))


def _k_update_log_mask(fm, a, block, grid):
    _libmod.check(_libmod.load().wdb_update_log_mask(
        _stream(), _P(a[0]), int(_scalar(a[1])), int(_scalar(a[2]))))


def _k_log_one_step(fm, a, block, grid):
    # log_one_step_in_{float,int}(log, data, feature_dim, timestep, episode_length, env)
    _libmod.check(_libmod.load().wdb_log_one_step(
        _stream(), _P(a[0]), _P(a[1]), fm._num_agents, int(_scalar(a[2])),
        int(_scalar(a[3])), int(_scalar(a[4])), int(_scalar(a[5]))))


def _k_noop(fm, a, block, grid):
    return None


_KERNELS = {
    "CudaTagContinuousStep": _k_tag_continuous_step,
    "NumbaTagContinuousStep": _k_tag_continuous_step,
    "CudaTagGridWorldStep": _k_tag_gridworld_step,
    "NumbaTagGridWorldStep": _k_tag_gridworld_step,
    **{f"{prefix}ClassicControl{env}EnvStep": _k_single_agent_step(*adapter)
       for env, adapter in {
           "CartPole": ("wdb_cartpole_step", 9),
           "MountainCar": ("wdb_mountain_car_step", 7),
           "ContinuousMountainCar": ("wdb_continuous_mountain_car_step", 8, True),
           "Pendulum": ("wdb_pendulum_step", 0, True),
           "Acrobot": ("wdb_acrobot_step", 0),
       }.items() for prefix in ("Numba", "Cuda")},
    "testkernel": _k_testkernel,
    "reset_in_float_when_done_2d": _k_reset_2d,
    "reset_in_int_when_done_2d": _k_reset_2d,
    "reset_in_float_when_done_3d": _k_reset_3d,
    "reset_in_int_when_done_3d": _k_reset_3d,
    "undo_done_flag_and_reset_timestep": _k_undo,
    "reset_log_mask": _k_reset_log_mask,
    "update_log_mask": _k_update_log_mask,
    "log_one_step_in_float": _k_log_one_step,
    "log_one_step_in_int": _k_log_one_step,
    # RNG state is owned by CUDASampler here (no device heap to free)
    "init_random": _k_noop,
    "free_random": _k_noop,
}

_DEFAULT_FUNCTIONS = [
    "reset_log_mask", "update_log_mask", "log_one_step_in_float", "log_one_step_in_int",
    "reset_in_float_when_done_2d", "reset_in_int_when_done_2d",
    "reset_in_float_when_done_3d", "reset_in_int_when_done_3d",
    "undo_done_flag_and_reset_timestep", "init_random", "free_random", "sample_actions",
]


class KernelFunction:
    """Callable returned by get_function(): `f(*args, block=, grid=)` (pycuda style) or
    `f[grid, block](*args)` (numba style).  block/grid are accepted for call
    compatibility; the library picks its own launch geometry."""

    def __init__(self, manager, name, adapter):
        self._fm = manager
        self.name = name
        self._adapter = adapter

    def __call__(self, *args, block=None, grid=None, n_envs=None, **_ignored):
        if n_envs is not None:
            return self._adapter(self._fm, args, block, grid, n_envs=n_envs)
        return self._adapter(self._fm, args, block, grid)

    def __getitem__(self, launch_config):
        grid, block = launch_config[0], launch_config[1]
        return lambda *args: self._adapter(self._fm, args, block, grid)

    def __repr__(self):
        return f"<libwdb200 kernel {self.name}>"


class CUDAFunctionManager:
    def __init__(self, num_agents: int = 1, num_envs: int = 1, blocks_per_env: int = 1,
                 process_id: int = 0, device=None):
        self._num_agents = int(num_agents)
        self._num_envs = int(num_envs)
        self._blocks_per_env = int(blocks_per_env)
        self._process_id = process_id
        # kept for callers that pass them back as block= / grid= (function_manager.py:65-67)
        self._block = (int((self._num_agents - 1) // self._blocks_per_env + 1), 1, 1)
        self._grid = (int(self._num_envs * self._blocks_per_env), 1)
        self._default_functions_initialized = False
        self._cuda_functions = {}
        self._cuda_function_names = []
        self._custom = {}
        self._custom_modules = []      # user cubins (utils/custom_kernels.py)
        self._shared_tensors = {}
        self._keepalive = []
        self._scratch_int = None
        self.stats_tensor = None
        self.device = torch.device(device) if device is not None else (
            torch.device("cuda", torch.cuda.current_device())
            if torch.cuda.is_available() else torch.device("cpu"))
        _libmod.load()  # fail loudly if libwdb200.so is not built

    # --- module loading: the library is prebuilt, these only keep the reference's call
    # --- sites working (env_wrapper.py:177-219, tests load a .fatbin / numba module)
    def load_cuda_from_binary_file(self, cubin, default_functions_included=True):
        """Reference tests pass the path of their own prebuilt fatbin here
        (tests/.../test_action_sampler.py:33-40): ignored, the default kernels are in
        libwdb200.so.  A cubin built by utils.custom_kernels.compile_module IS loaded."""
        if isinstance(cubin, str) and cubin.endswith(".cubin") and os.path.exists(cubin):
            self._load_custom_module(cubin)
        if default_functions_included:
            self.initialize_default_functions()

    def load_cuda_from_source_code(self, code, default_functions_included=True):
        """Compile CUDA-C source (a path to a .cu file or the source text) for sm_90a with the
        reference's three compile-time constants and load it next to the prebuilt kernels
        (reference: pycuda_function_manager.py:197-232 does this with pycuda's
        SourceModule).  Its extern "C" kernels become get_function() names."""
        from warp_drive_b200.utils import custom_kernels

        cubin = custom_kernels.compile_module(code, self._num_envs, self._num_agents,
                                              self._blocks_per_env)
        self._load_custom_module(cubin)
        if default_functions_included:
            self.initialize_default_functions()

    def _load_custom_module(self, cubin):
        from warp_drive_b200.utils import custom_kernels

        module = custom_kernels.CustomCudaModule(cubin)
        self._custom_modules.append(module)
        return module

    def compile_and_load_cuda(self, env_name=None, template_header_file=None,
                              template_runner_file=None, template_path=None,
                              default_functions_included=True,
                              customized_env_registrar=None, event_messenger=None):
        """The built-in envs need no compilation.  If `customized_env_registrar` holds a `.cu`
        path for `env_name` (env_registrar.add_cuda_env_src_path, reference
        pycuda_function_manager.py:268-282), that file is compiled for sm_90a and its kernels
        take precedence over built-ins of the same name."""
        if customized_env_registrar is not None and env_name is not None:
            src = customized_env_registrar.get_cuda_env_src_path(env_name)
            if src is not None:
                self.load_cuda_from_source_code(src, default_functions_included=False)
        if default_functions_included:
            self.initialize_default_functions()

    def dynamic_import_numba(self, env_name=None, template_header_file=None,
                             template_runner_file=None, template_path=None,
                             default_functions_included=True,
                             customized_env_registrar=None, event_messenger=None):
        if default_functions_included:
            self.initialize_default_functions()

    def import_numba_from_source_code(self, numba_path=None,
                                      default_functions_included=True):
        if default_functions_included:
            self.initialize_default_functions()

    def register_function(self, name, fn):
        """Plug in a user kernel launcher: fn(manager, args, block, grid)."""
        self._custom[name] = fn

    def initialize_default_functions(self):
        if self._default_functions_initialized:
            return
        self.initialize_functions(_DEFAULT_FUNCTIONS)
        self._default_functions_initialized = True

    def initialize_functions(self, func_names: Optional[list] = None):
        for fname in func_names or []:
            if fname in self._cuda_functions:
                continue
            module = next((m for m in self._custom_modules if m.has(fname)), None)
            if fname in self._custom:
                adapter = self._custom[fname]
            elif module is not None:
                adapter = module.launcher(fname)
            elif fname == "sample_actions":
                adapter = _k_noop  # launched through CUDASampler.sample
            elif fname in _KERNELS:
                adapter = _KERNELS[fname]
            else:
                raise KeyError(f"libwdb200 has no kernel named '{fname}'")
            self._cuda_functions[fname] = KernelFunction(self, fname, adapter)
            self._cuda_function_names.append(fname)

    def initialize_shared_constants(self, data_manager: CUDADataManager,
                                    constant_names: list):
        """The reference memcpy's into __constant__ symbols of its module
        (pycuda_function_manager.py:363-379); here constants become small device tensors
        handed to the kernels that use them."""
        for cname in constant_names:
            value = np.ascontiguousarray(data_manager.shared_constant(cname))
            self._shared_tensors[cname] = torch.from_numpy(value.reshape(-1)).to(self.device)
            for module in self._custom_modules:   # user code keeps its __constant__ symbols
                module.set_constant(cname, value)

    def shared_constant_tensor(self, name):
        if name not in self._shared_tensors:
            raise RuntimeError(
                f"shared constant '{name}' has not been initialised: call "
                "data_manager.add_shared_constants({...}) and "
                "function_manager.initialize_shared_constants(data_manager, [...]) first")
        return self._shared_tensors[name]

    def scratch_int(self, n):
        if self._scratch_int is None or self._scratch_int.numel() < n:
            self._scratch_int = torch.zeros(n, dtype=torch.int32, device=self.device)
        return self._scratch_int

    def enable_stats(self):
        """Allocate the optional device counters of wdb_tag_continuous_step."""
        self.stats_tensor = torch.zeros(4, dtype=torch.int32, device=self.device)
        return self.stats_tensor

    def _get_function(self, fname):
        assert fname in self._cuda_functions, f"{fname} is not defined"
        return self._cuda_functions[fname]

    @property
    def get_function(self):
        return self._get_function

    @property
    def cuda_function_names(self):
        return self._cuda_function_names

    @property
    def block(self):
        return self._block

    @property
    def grid(self):
        return self._grid

    @property
    def blocks_per_env(self):
        return self._blocks_per_env


class CUDAFunctionFeed:
    """names -> kernel arguments, resolved once and cached
    (warp_drive/managers/function_manager.py:96-134)."""

    def __init__(self, data_manager: CUDADataManager):
        self.data_manager = data_manager
        self._function_feeds = None

    def __call__(self, arguments: list) -> list:
        if self._function_feeds is None:
            feeds = []
            for arg in arguments:
                if isinstance(arg, str):
                    feeds.append(self.data_manager.device_data(arg))
                elif isinstance(arg, tuple):
                    key, source = arg[0], arg[1].lower()
                    if source in ("d", "device"):
                        feeds.append(self.data_manager.device_data(key))
                    elif source in ("m", "meta"):
                        feeds.append(self.data_manager.meta_info(key))
                    elif source in ("s", "shared"):
                        feeds.append(self.data_manager.shared_constant(key))
                    else:
                        raise Exception(f"Unknown definition of CUDA function feed: {arg}")
                else:
                    raise Exception(f"Unknown definition of CUDA function feed: {arg}")
            self._function_feeds = feeds
        return self._function_feeds


class CUDASampler:
    """Categorical / argmax / OU-Gaussian / diagonal-Gaussian action sampling on the device
    (reference: CUDASampler function_manager.py:137-208, PyCUDASampler
    pycuda_function_manager.py:486-590, NumbaOUProcess numba_function_manager.py:731-817).
    RNG = counter-based Philox4x32-10; the state (one u64 offset per (env, agent) stream)
    is a torch tensor owned by this object."""

    def __init__(self, function_manager: CUDAFunctionManager):
        self._function_manager = function_manager
        assert function_manager._default_functions_initialized, (
            "Default CUDA functions are required to initialized before the sampler can "
            "work, call function_manager.initialize_default_functions() to proceed")
        self._block = function_manager.block
        self._grid = function_manager.grid
        self._blocks_per_env = function_manager.blocks_per_env
        self._num_envs = function_manager._num_envs
        self._num_agents = function_manager._num_agents
        self._random_initialized = False
        self.rng_state = None
        self.seed = None

    def init_random(self, seed: Optional[int] = None):
        if seed is None:
            seed = int(time.time())
            logging.info(f"random seed is not provided, using the timestamp {seed}")
        L = _libmod.load()
        n_streams = self._num_envs * self._num_agents
        nbytes = int(L.wdb_rng_state_bytes(n_streams))
        self.rng_state = torch.zeros(nbytes, dtype=torch.uint8,
                                     device=self._function_manager.device)
        _libmod.check(L.wdb_rng_init(_stream(), _P(self.rng_state), n_streams,
                                     int(seed) & 0xFFFFFFFFFFFFFFFF), "rng_init")
        self.seed = int(seed)
        self._random_initialized = True

    def register_actions(self, data_manager: CUDADataManager, action_name: str,
                         num_actions: int, is_deterministic=False):
        n_agents = data_manager.get_shape(action_name)[1]
        if is_deterministic:
            num_actions = 1
        host = np.zeros((self._grid[0], n_agents, num_actions), dtype=np.float32)
        feed = DataFeed()
        suffix = "_ou_state" if is_deterministic else "_cum_distr"
        feed.add_data(name=f"{action_name}{suffix}", data=host)
        data_manager.push_data_to_device(feed)

    def sample(self, data_manager: CUDADataManager, distribution: torch.Tensor,
               action_name: str, use_argmax: bool = False, uniforms=None,
               combined=None, write_cum_distr: bool = True, damping=None, stddev=None,
               scale=None, normals=None, nonzero=False):
        """distribution [n_envs, n_agents, n_actions] float32 -> `action_name` on device.
        nonzero=True: never select an index of probability 0 (wdb_sample_actions_nonzero; for
        policies with masked actions) instead of the reference's index search.
        `combined=(tensor, stride, offset)` additionally scatters the index into a
        multi-head action array (fuses trainer_base.py:507-512).
        `uniforms` / `normals` are test hooks replacing the RNG draw."""
        assert self._random_initialized, (
            "sample() requires the random seed initialized first, call init_random()")
        assert torch.is_tensor(distribution)
        assert distribution.shape[0] == self._num_envs
        n_agents = int(distribution.shape[1])
        assert data_manager.get_shape(action_name)[1] == n_agents
        n_actions = int(distribution.shape[2])
        L = _libmod.load()
        if distribution.dtype != torch.float32 or not distribution.is_contiguous():
            distribution = distribution.float().contiguous()
        if data_manager.is_data_on_device(f"{action_name}_ou_state") and not \
                data_manager.is_data_on_device(f"{action_name}_cum_distr"):
            assert n_actions == 1
            _libmod.check(L.wdb_sample_ou_process(
                _stream(), _P(self.rng_state), _P(distribution),
                _P(data_manager.device_data(action_name)),
                _P(data_manager.device_data(f"{action_name}_ou_state")),
                self._num_envs, n_agents,
                float(0.15 if damping is None else damping),
                float(0.2 if stddev is None else stddev),
                float(1.0 if scale is None else scale), _P(normals)), "sample_ou_process")
            return
        cum = None
        if write_cum_distr and data_manager.is_data_on_device(f"{action_name}_cum_distr"):
            assert data_manager.get_shape(f"{action_name}_cum_distr")[2] == n_actions
            cum = data_manager.device_data(f"{action_name}_cum_distr")
        ctensor, cstride, coffset = combined if combined is not None else (None, 0, 0)
        launch = L.wdb_sample_actions_nonzero if nonzero else L.wdb_sample_actions
        _libmod.check(launch(
            _stream(), _P(self.rng_state), _P(distribution),
            _P(data_manager.device_data(action_name)), _P(cum), self._num_envs, n_agents,
            n_actions, int(bool(use_argmax)), _P(ctensor), int(cstride), int(coffset),
            _P(uniforms)), "sample_actions")

    def sample_gaussian(self, mean: torch.Tensor, log_std: torch.Tensor, actions: torch.Tensor,
                        use_argmax: bool = False, normals=None):
        """Diagonal Gaussian policy: actions = mean + exp(log_std) * N(0, 1), drawn raw (the
        env bounds them); mean / actions [n_envs, n_agents, A] float32 (actions: the
        `sampled_actions` array or any float32 tensor of that shape), log_std [A].  Row r of
        the [n_envs * n_agents] rows draws from RNG stream r (wdb_sample_gaussian).
        use_argmax=True: actions = mean, no draw.  `normals` [n_envs, n_agents, A] is a test
        hook replacing the draws."""
        assert self._random_initialized, (
            "sample_gaussian() requires the random seed initialized first, call init_random()")
        assert mean.shape[0] == self._num_envs and mean.dim() == 3
        assert tuple(actions.shape) == tuple(mean.shape) and actions.dtype == torch.float32
        assert log_std.shape == (mean.shape[-1],)
        assert mean.shape[0] * mean.shape[1] <= self._num_envs * self._num_agents
        mean = mean.detach().float().contiguous()
        log_std = log_std.detach().float().contiguous()
        _libmod.check(_libmod.load().wdb_sample_gaussian(
            _stream(), _P(self.rng_state), _P(mean), _P(log_std), _P(actions),
            int(mean.shape[0] * mean.shape[1]), int(mean.shape[-1]), int(bool(use_argmax)),
            _P(normals)), "sample_gaussian")

    def sample_squashed_gaussian(self, head: torch.Tensor, actions: torch.Tensor,
                                 action_scale: float, action_bias: float, log_std_min: float,
                                 log_std_max: float, use_argmax: bool = False, normals=None):
        """Tanh-squashed Gaussian policy (SAC's actor): head [n_envs, n_agents, 2A] = mean mu ++
        raw log-std (clamped to [log_std_min, log_std_max]); actions [n_envs, n_agents, A] =
        action_scale * tanh(mu + exp(log_std) * N(0, 1)) + action_bias, row r of the
        [n_envs * n_agents] rows drawing from RNG stream r with wdb_sample_gaussian's pairing
        (wdb_sample_squashed_gaussian).  use_argmax=True: tanh(mu), no draw.  `normals`
        [n_envs, n_agents, A] is a test hook replacing the draws."""
        assert self._random_initialized, (
            "sample_squashed_gaussian() requires the random seed initialized first, call "
            "init_random()")
        assert head.shape[0] == self._num_envs and head.dim() == 3 and head.shape[-1] % 2 == 0
        A = head.shape[-1] // 2
        assert tuple(actions.shape) == tuple(head.shape[:-1]) + (A,)
        assert actions.dtype == torch.float32 and actions.is_contiguous()
        assert head.shape[0] * head.shape[1] <= self._num_envs * self._num_agents
        head = head.detach().float().contiguous()
        _libmod.check(_libmod.load().wdb_sample_squashed_gaussian(
            _stream(), _P(self.rng_state), _P(head), _P(actions),
            int(head.shape[0] * head.shape[1]), int(A), float(action_scale), float(action_bias),
            float(log_std_min), float(log_std_max), int(bool(use_argmax)), _P(normals)),
            "sample_squashed_gaussian")

    def sample_epsilon_greedy(self, q_values: torch.Tensor, actions: torch.Tensor,
                              epsilon: float = 0.0, words=None, action_mask=None,
                              branch_sizes=None):
        """Epsilon-greedy over Q values (DQN): q_values [n_envs, n_agents, A] float32 ->
        actions [n_envs, n_agents, 1] int32.  Row r of the [n_envs * n_agents] rows draws one
        Philox block on RNG stream r (its offset advances by 1) and explores iff the uniform of
        its first word is <= epsilon, with the action high(second word * A); otherwise it takes
        the first maximum of its Q values (wdb_sample_epsilon_greedy).  `words` (int32
        [n_envs, n_agents, 2], the two words of each row) is a test hook replacing the draw.
        `action_mask` (float32 [n_envs, n_agents, A], non-zero = valid): the same draw over the
        row's valid actions only, the k-th valid one when exploring and the first maximum among
        them otherwise; a row with none valid takes the unmasked action
        (wdb_sample_epsilon_greedy_masked).  `branch_sizes` [A_0, ..., A_{D-1}] (action
        branching, sum A_d = A): head d of each row is epsilon-greedy over its Q columns
        o_d .. o_d + A_d - 1 on its own, with the Philox block at the row's offset + d; the
        offset then advances by D, and actions are [n_envs, n_agents, D]
        (wdb_sample_epsilon_greedy_branching; `words` [n_envs, n_agents, D, 2])."""
        assert self._random_initialized, (
            "sample_epsilon_greedy() requires the random seed initialized first, call "
            "init_random()")
        assert q_values.shape[0] == self._num_envs and q_values.dim() == 3
        if branch_sizes is not None:
            assert action_mask is None, "branching Q values take no action mask"
            self._sample_epsilon_greedy_branching(q_values, actions, epsilon, words,
                                                  branch_sizes)
            return
        assert tuple(actions.shape) == tuple(q_values.shape[:-1]) + (1,)
        assert actions.dtype == torch.int32 and actions.is_contiguous()
        assert q_values.shape[0] * q_values.shape[1] <= self._num_envs * self._num_agents
        if not 0.0 <= float(epsilon) <= 1.0:
            raise ValueError(f"epsilon must be in [0, 1], got {epsilon}")
        if words is not None:
            assert tuple(words.shape) == tuple(q_values.shape[:-1]) + (2,)
            assert words.dtype == torch.int32 and words.is_contiguous()
        q_values = q_values.detach().float().contiguous()
        if action_mask is not None:
            assert tuple(action_mask.shape) == tuple(q_values.shape)
            assert action_mask.dtype == torch.float32 and action_mask.is_contiguous()
            _libmod.check(_libmod.load().wdb_sample_epsilon_greedy_masked(
                _stream(), _P(self.rng_state), _P(q_values), _P(action_mask), _P(actions),
                int(q_values.shape[0] * q_values.shape[1]), int(q_values.shape[-1]),
                float(epsilon), _P(words)), "sample_epsilon_greedy_masked")
            return
        _libmod.check(_libmod.load().wdb_sample_epsilon_greedy(
            _stream(), _P(self.rng_state), _P(q_values), _P(actions),
            int(q_values.shape[0] * q_values.shape[1]), int(q_values.shape[-1]),
            float(epsilon), _P(words)), "sample_epsilon_greedy")

    def _sample_epsilon_greedy_branching(self, q_values, actions, epsilon, words, branch_sizes):
        sizes = [int(a) for a in branch_sizes]
        D = len(sizes)
        if not 1 <= D <= _libmod.Q_MAX_BRANCHES or min(sizes) < 1:
            raise ValueError(f"branch_sizes holds 1 to {_libmod.Q_MAX_BRANCHES} head sizes >= 1, "
                             f"got {sizes}")
        assert q_values.shape[-1] == sum(sizes)
        assert tuple(actions.shape) == tuple(q_values.shape[:-1]) + (D,)
        assert actions.dtype == torch.int32 and actions.is_contiguous()
        assert q_values.shape[0] * q_values.shape[1] <= self._num_envs * self._num_agents
        if not 0.0 <= float(epsilon) <= 1.0:
            raise ValueError(f"epsilon must be in [0, 1], got {epsilon}")
        if words is not None:
            assert tuple(words.shape) == tuple(q_values.shape[:-1]) + (D, 2)
            assert words.dtype == torch.int32 and words.is_contiguous()
        q_values = q_values.detach().float().contiguous()
        b = _libmod.QBranches()
        b.n_heads = D
        for d, a in enumerate(sizes):
            b.sizes[d] = a
        _libmod.check(_libmod.load().wdb_sample_epsilon_greedy_branching(
            _stream(), _P(self.rng_state), _P(q_values), ctypes.byref(b), _P(actions),
            int(q_values.shape[0] * q_values.shape[1]), float(epsilon), _P(words)),
            "sample_epsilon_greedy_branching")

    @staticmethod
    def assign(data_manager: CUDADataManager, actions: np.ndarray, action_name: str):
        """Write actions directly (testing / debugging),
        pycuda_function_manager.py:574-590."""
        assert data_manager.is_data_on_device_via_torch(action_name)
        assert actions.shape == data_manager.get_shape(action_name)
        assert actions.dtype.name == data_manager.get_dtype(action_name)
        t = data_manager.data_on_device_via_torch(action_name)
        t[:] = torch.from_numpy(actions).to(t.device)


class CUDAEnvironmentReset:
    """Done-masked restore of every `save_copy_and_apply_at_reset` array (and reset
    pools) + undo of `_done_` / `_timestep_`, in ONE kernel launch over a cached
    device-side descriptor table.  Reference: function_manager.py:211-292 and
    pycuda_function_manager.py:593-753 (one launch per array + one for the undo)."""

    def __init__(self, function_manager: CUDAFunctionManager):
        self._function_manager = function_manager
        assert function_manager._default_functions_initialized, (
            "Default CUDA functions are required to initialized before EnvironmentReset "
            "can work, call function_manager.initialize_default_functions() to proceed")
        self._block = function_manager.block
        self._grid = function_manager.grid
        self._blocks_per_env = function_manager.blocks_per_env
        self._cuda_custom_reset = None
        self._cuda_reset_feed = None
        self._random_initialized = False
        self._table = None
        self._table_key = None
        self._pool_rng = None

    def register_custom_reset_function(self, data_manager: CUDADataManager,
                                       reset_function_name=None):
        fm = self._function_manager
        if reset_function_name is None or (
                reset_function_name not in fm._cuda_functions
                and reset_function_name not in fm._custom
                and not any(m.has(reset_function_name) for m in fm._custom_modules)):
            return
        fm.initialize_functions([reset_function_name])
        self._cuda_custom_reset = fm.get_function(reset_function_name)
        self._cuda_reset_feed = CUDAFunctionFeed(data_manager)

    def custom_reset(self, args: Optional[list] = None, block=None, grid=None):
        assert self._cuda_custom_reset is not None and self._cuda_reset_feed is not None, (
            "Custom Reset function is not defined, call "
            "register_custom_reset_function() first")
        assert args is None or isinstance(args, list)
        block = block or self._block
        grid = grid or self._grid
        if not args:
            self._cuda_custom_reset(block=block, grid=grid)
        else:
            self._cuda_custom_reset(*self._cuda_reset_feed(args), block=block, grid=grid)

    def init_reset_pool(self, data_manager: CUDADataManager, seed: Optional[int] = None):
        if len(data_manager.reset_target_to_pool) == 0:
            return
        if seed is None:
            seed = int(time.time())
        L = _libmod.load()
        n_envs = int(data_manager.meta_info("n_envs"))
        self._pool_rng = torch.zeros(int(L.wdb_rng_state_bytes(n_envs)), dtype=torch.uint8,
                                     device=self._function_manager.device)
        _libmod.check(L.wdb_rng_init(_stream(), _P(self._pool_rng), n_envs,
                                     int(seed) & 0xFFFFFFFFFFFFFFFF), "rng_init(pool)")
        self._random_initialized = True

    def build_table(self, data_manager: CUDADataManager):
        """(device tensor of wdb_reset_desc[], n_arrays) for the registered arrays, in
        registration order (deterministic arrays first, then pools)."""
        n_envs = int(data_manager.meta_info("n_envs"))
        entries = []
        for name in data_manager.reset_data_list:
            shape = data_manager.get_shape(name)
            assert shape[0] == n_envs, "reset function assumes the 0th dimension is n_envs"
            per_env = int(np.prod(shape[1:])) if len(shape) > 1 else 1
            entries.append((data_manager.device_data(name),
                            data_manager.device_data(f"{name}_at_reset"), per_env, 0))
        for target, pool in data_manager.reset_target_to_pool.items():
            shape = data_manager.get_shape(target)
            pshape = data_manager.get_shape(pool)
            assert shape[0] == n_envs
            per_env = int(np.prod(shape[1:])) if len(shape) > 1 else 1
            assert int(np.prod(pshape[1:])) == per_env, "pool rows must match the target"
            entries.append((data_manager.device_data(target),
                            data_manager.device_data(pool), per_env, int(pshape[0])))
        key = tuple((e[0].name, e[1].name) for e in entries)
        if self._table is not None and key == self._table_key:
            return self._table, len(entries)
        desc = (_libmod.ResetDesc * max(1, len(entries)))()
        for i, (dst, ref, per_env, pool_rows) in enumerate(entries):
            desc[i].dst = _P(dst)
            desc[i].ref = _P(ref)
            desc[i].bytes_per_env = 4 * per_env
            desc[i].pool_rows = pool_rows
        raw = np.frombuffer(desc, dtype=np.uint8).copy()
        self._table = torch.from_numpy(raw).to(self._function_manager.device)
        self._table_key = key
        return self._table, len(entries)

    def reset_when_done(self, data_manager: CUDADataManager, mode: str = "if_done",
                        undo_done_after_reset: bool = True):
        if mode == "if_done":
            force_reset = 0
        elif mode == "force_reset":
            force_reset = 1
        else:
            raise Exception(
                f"unknown reset mode: {mode}, only accept 'if_done' and 'force_reset' ")
        table, n = self.build_table(data_manager)
        if any(e > 0 for e in [len(data_manager.reset_target_to_pool)]):
            assert self._random_initialized, (
                "reset pools need init_reset_pool(data_manager, seed) first")
        _libmod.check(_libmod.load().wdb_reset_when_done(
            _stream(), _P(table) if n > 0 else None, n,
            _P(data_manager.device_data("_done_")),
            _P(data_manager.device_data("_timestep_")),
            int(data_manager.meta_info("n_envs")), force_reset,
            int(bool(undo_done_after_reset)), _P(self._pool_rng)), "reset_when_done")

    # the reference splits the work in three calls; keep them for API compatibility
    def reset_when_done_deterministic(self, data_manager, force_reset):
        self.reset_when_done(data_manager,
                             "force_reset" if int(force_reset) else "if_done",
                             undo_done_after_reset=False)

    def reset_when_done_from_pool(self, data_manager, force_reset):
        return

    def _undo_done_flag_and_reset_timestep(self, data_manager, force_reset):
        _libmod.check(_libmod.load().wdb_reset_when_done(
            _stream(), None, 0, _P(data_manager.device_data("_done_")),
            _P(data_manager.device_data("_timestep_")),
            int(data_manager.meta_info("n_envs")), int(force_reset), 1, None))


class CUDALogController:
    """Episode logging of ONE env for arrays pushed with log_data_across_episode=True
    (reference: function_manager.py:295-422, pycuda_function_manager.py:399-483)."""

    def __init__(self, function_manager: CUDAFunctionManager):
        self._function_manager = function_manager
        assert function_manager._default_functions_initialized
        self._block = function_manager.block
        self._grid = function_manager.grid
        self._blocks_per_env = function_manager.blocks_per_env
        self.last_valid_step = -1
        self._env_id = None

    def update_log(self, data_manager: CUDADataManager, step: int):
        assert step > self.last_valid_step, (
            "update_log is trying to update the existing timestep")
        self._log_one_step(data_manager, step, self._env_id)
        self._update_log_mask(data_manager, step)

    def reset_log(self, data_manager: CUDADataManager, env_id: int = 0):
        self._env_id = env_id
        self.last_valid_step = -1
        self._reset_log_mask(data_manager)
        self.update_log(data_manager, step=0)

    def fetch_log(self, data_manager: CUDADataManager, names=None, last_step=None,
                  check_last_valid_step: bool = True):
        if check_last_valid_step:
            self._cuda_check_last_valid_step(data_manager)
        last = self.last_valid_step
        if last_step is not None and last_step <= self.last_valid_step:
            last = last_step
        if names is None:
            names = data_manager.log_data_list
        out = {}
        for name in names:
            key = f"{name}_for_log"
            d = data_manager.pull_data_from_device(key)
            assert len(d) == int(data_manager.meta_info("episode_length")) + 1
            out[key] = d[: last + 1]
        return out

    def _log_one_step(self, data_manager, step, env_id=0):
        assert env_id < data_manager.meta_info("n_envs")
        L = _libmod.load()
        for name in data_manager.log_data_list:
            shape = data_manager.get_shape(name)
            assert shape[0] == data_manager.meta_info("n_envs")
            assert shape[1] == data_manager.meta_info("n_agents")
            feature_dim = int(np.prod(shape[2:])) if len(shape) >= 3 else 1
            _libmod.check(L.wdb_log_one_step(
                _stream(), _P(data_manager.device_data(f"{name}_for_log")),
                _P(data_manager.device_data(name)), int(shape[1]), feature_dim, int(step),
                int(data_manager.meta_info("episode_length")), int(env_id)), "log_one_step")

    def log_tensor_one_step(self, log, data, step, env_id=0):
        """Copy env `env_id`'s slice of `data` ([n_envs, ...], any 32-bit dtype) into row `step`
        of the device-side log `log` ([n_steps, ...]) with the log kernel -- the device ring
        Trainer.fetch_episode_states records an episode in (no `_for_log` registration needed)."""
        assert data.is_cuda and log.is_cuda and data.element_size() == 4 and log.dtype == data.dtype
        assert data.is_contiguous() and log.is_contiguous()
        assert 0 <= step < log.shape[0] and 0 <= env_id < data.shape[0]
        per_env = int(np.prod(data.shape[1:])) if data.dim() > 1 else 1
        assert int(np.prod(log.shape[1:])) == per_env if log.dim() > 1 else per_env == 1
        _libmod.check(_libmod.load().wdb_log_one_step(
            _stream(), _P(log), _P(data), per_env, 1, int(step), int(log.shape[0]) - 1,
            int(env_id)), "log_one_step")

    def _update_log_mask(self, data_manager, step):
        _libmod.check(_libmod.load().wdb_update_log_mask(
            _stream(), _P(data_manager.device_data("_log_mask_")), int(step),
            int(data_manager.meta_info("episode_length"))))
        self.last_valid_step = int(step)

    def _reset_log_mask(self, data_manager):
        _libmod.check(_libmod.load().wdb_reset_log_mask(
            _stream(), _P(data_manager.device_data("_log_mask_")),
            int(data_manager.meta_info("episode_length"))))

    def _cuda_check_last_valid_step(self, data_manager):
        log_mask = data_manager.pull_data_from_device("_log_mask_")
        ones = np.argwhere(log_mask == 1).reshape(-1)
        zeros = np.argwhere(log_mask == 0).reshape(-1)
        if len(ones) > 0 and len(zeros) > 0 and zeros[0] < ones[-1]:
            raise Exception("there is invalid log data in the middle")
        last = ones[-1] if len(ones) > 0 else -1
        assert last == self.last_valid_step, (
            f"inconsistency of last_valid_step derived from dense_log_mask = {last} "
            f"and the step() function = {self.last_valid_step}")


# names a reference user imports
PyCUDAFunctionManager = NumbaFunctionManager = B200FunctionManager = CUDAFunctionManager
PyCUDASampler = NumbaSampler = B200Sampler = CUDASampler
PyCUDAEnvironmentReset = NumbaEnvironmentReset = B200EnvironmentReset = CUDAEnvironmentReset
PyCUDALogController = NumbaLogController = B200LogController = CUDALogController

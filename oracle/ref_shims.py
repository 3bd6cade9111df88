"""TEST INFRASTRUCTURE ONLY -- never imported by the product (sample_factory_b200/).

In-memory stand-ins for the third-party packages the reference imports at module
load but which an offline install does not have (signal_slot, faster_fifo,
colorlog, tensorboardX, gymnasium).  They let `tests/golden/make_golden.py`
import and EXECUTE the unmodified reference classes from a reference checkout (oracle/install_ref.py: reference_dir())
(Learner, ActorCritic, BatchedVectorEnvRunner, gae_advantages, ...) so that the
golden vectors under tests/golden/ are produced by the reference's own code.

Only used to generate the goldens; no test needs the reference checkout itself, only the
stored vectors.  None of this is reference code: it is the minimum
surface (names + trivial behaviour) those imports need.
"""
from __future__ import annotations

import logging
import os
import queue
import sys
import types

import numpy as np


def _mod(name: str) -> types.ModuleType:
    m = types.ModuleType(name)
    sys.modules[name] = m
    return m


def install(reference_root: str | None = None) -> None:
    if "signal_slot" in sys.modules and getattr(sys.modules["signal_slot"], "_sfb200_shim", False):
        return

    # ---- signal_slot -------------------------------------------------------
    ss = _mod("signal_slot")
    ss._sfb200_shim = True
    sss = _mod("signal_slot.signal_slot")
    ss.signal_slot = sss

    class signal:  # noqa: N801  (descriptor-like placeholder)
        def __init__(self, *a, **k):
            self._slots = []

        def __set_name__(self, owner, name):
            self._name = name

        def connect(self, *a, **k):
            pass

        def emit(self, *a, **k):
            pass

        def disconnect(self, *a, **k):
            pass

    class EventLoopObject:
        def __init__(self, event_loop=None, object_id=None):
            self.event_loop = event_loop
            self.object_id = object_id

        def emit(self, *a, **k):
            pass

        def emit_many(self, *a, **k):
            pass

        def detach(self):
            pass

    class EventLoop(EventLoopObject):
        def __init__(self, unique_loop_name="loop", serial_mode=True):
            super().__init__(self, unique_loop_name)
            self.owner = None

        def exec(self):
            return 0

    class EventLoopProcess(EventLoopObject):
        pass

    class EventLoopStatus:
        NORMAL_TERMINATION, INTERRUPTED, ERROR = 0, 1, 2

    class Timer(EventLoopObject):
        def __init__(self, event_loop=None, interval_sec=1.0, single_shot=False):
            super().__init__(event_loop, "timer")
            self.timeout = signal()

        def stop(self):
            pass

    class TightLoop(EventLoopObject):
        def __init__(self, event_loop=None):
            super().__init__(event_loop, "tight")
            self.iteration = signal()

        def stop(self):
            pass

        def start(self):
            pass

    class StatusCode:
        SUCCESS, FAILURE, INTERRUPTED = 0, 1, 2

    sss.signal = signal
    sss.EventLoopObject = EventLoopObject
    sss.EventLoop = EventLoop
    sss.EventLoopProcess = EventLoopProcess
    sss.EventLoopStatus = EventLoopStatus
    sss.Timer = Timer
    sss.TightLoop = TightLoop
    sss.StatusCode = StatusCode
    sss.BoundMethod = tuple
    sss.process_name = lambda *a, **k: "main"
    sss.configure_logger = lambda *a, **k: None

    qu = _mod("signal_slot.queue_utils")
    ss.queue_utils = qu

    class _Q(queue.Queue):
        def get_many(self, block=True, timeout=None, max_messages_to_get=int(1e9)):
            out = [self.get(block=block, timeout=timeout)]
            while len(out) < max_messages_to_get:
                try:
                    out.append(self.get_nowait())
                except queue.Empty:
                    break
            return out

        def put_many(self, xs, block=True, timeout=None):
            for x in xs:
                self.put(x, block=block, timeout=timeout)

    qu.get_queue = lambda serial=True, buffer_size_bytes=0: _Q()

    # ---- colorlog / tensorboardX ------------------------------------------
    cl = _mod("colorlog")

    class ColoredFormatter(logging.Formatter):
        def __init__(self, fmt=None, datefmt=None, **kw):
            super().__init__("[%(asctime)s] %(message)s", datefmt)

    cl.ColoredFormatter = ColoredFormatter

    tbx = _mod("tensorboardX")

    class SummaryWriter:
        def __init__(self, *a, **k):
            pass

        def add_scalar(self, *a, **k):
            pass

        def flush(self):
            pass

        def close(self):
            pass

    tbx.SummaryWriter = SummaryWriter

    # ---- gymnasium (spaces + Env/Wrapper) ----------------------------------
    gym = _mod("gymnasium")
    spaces = _mod("gymnasium.spaces")
    core = _mod("gymnasium.core")
    wrappers = _mod("gymnasium.wrappers")
    gym.spaces, gym.core, gym.wrappers = spaces, core, wrappers

    class Space:
        def __init__(self, shape=None, dtype=None):
            self.shape = None if shape is None else tuple(shape)
            self.dtype = None if dtype is None else np.dtype(dtype)

        def __eq__(self, other):
            return type(self) is type(other) and self.__dict__.keys() == other.__dict__.keys() and all(
                np.array_equal(v, other.__dict__[k]) if isinstance(v, np.ndarray) else v == other.__dict__[k]
                for k, v in self.__dict__.items()
            )

        def __repr__(self):
            return f"{type(self).__name__}({self.__dict__})"

    class Discrete(Space):
        def __init__(self, n, start=0):
            super().__init__((), np.int64)
            self.n = int(n)
            self.start = start

    class Box(Space):
        def __init__(self, low, high, shape=None, dtype=np.float32):
            if shape is None:
                shape = np.asarray(low).shape
            super().__init__(shape, dtype)
            self.low = np.broadcast_to(np.asarray(low, dtype=dtype), self.shape).copy()
            self.high = np.broadcast_to(np.asarray(high, dtype=dtype), self.shape).copy()

    class Tuple(Space):
        def __init__(self, spaces_):
            super().__init__(None, None)
            self.spaces = tuple(spaces_)

        def __iter__(self):
            return iter(self.spaces)

        def __len__(self):
            return len(self.spaces)

        def __getitem__(self, i):
            return self.spaces[i]

    class Dict(Space):
        def __init__(self, spaces_=None, **kw):
            super().__init__(None, None)
            self.spaces = dict(spaces_ or {}, **kw)

        def keys(self):
            return self.spaces.keys()

        def items(self):
            return self.spaces.items()

        def __getitem__(self, k):
            return self.spaces[k]

        def __iter__(self):
            return iter(self.spaces)

        def __contains__(self, k):
            return k in self.spaces

    for c in (Space, Discrete, Box, Tuple, Dict):
        setattr(spaces, c.__name__, c)
    gym.Space = Space

    class Env:
        metadata = {}
        render_mode = None
        observation_space = None
        action_space = None

        @property
        def unwrapped(self):
            return self

        def close(self):
            pass

    class Wrapper(Env):
        def __init__(self, env):
            self.env = env

        def __getattr__(self, name):
            if name.startswith("_"):
                raise AttributeError(name)
            return getattr(self.env, name)

        @property
        def unwrapped(self):
            return self.env.unwrapped

        @property
        def observation_space(self):
            return self.__dict__.get("_obs_space", None) or self.env.observation_space

        @observation_space.setter
        def observation_space(self, v):
            self.__dict__["_obs_space"] = v

        @property
        def action_space(self):
            return self.__dict__.get("_act_space", None) or self.env.action_space

        @action_space.setter
        def action_space(self, v):
            self.__dict__["_act_space"] = v

        def reset(self, **kw):
            return self.env.reset(**kw)

        def step(self, a):
            return self.env.step(a)

        def close(self):
            return self.env.close()

    class ObservationWrapper(Wrapper):
        pass

    class RewardWrapper(Wrapper):
        pass

    class ActionWrapper(Wrapper):
        pass

    gym.Env, gym.Wrapper = Env, Wrapper
    gym.ObservationWrapper, gym.RewardWrapper, gym.ActionWrapper = ObservationWrapper, RewardWrapper, ActionWrapper
    gym.make = lambda *a, **k: (_ for _ in ()).throw(RuntimeError("gymnasium shim: no envs"))
    core.ActType = core.ObsType = object
    core.Env, core.Wrapper = Env, Wrapper
    core.ObservationWrapper, core.RewardWrapper, core.ActionWrapper = ObservationWrapper, RewardWrapper, ActionWrapper
    wrappers.RecordEpisodeStatistics = Wrapper

    if reference_root is None:
        from oracle.install_ref import reference_dir

        reference_root = reference_dir()
    if not reference_root or not os.path.isfile(os.path.join(reference_root, "sample_factory", "__init__.py")):
        raise RuntimeError("no reference checkout: set SF_REFERENCE_DIR to a sample-factory source tree "
                           "(never this repository's own sample_factory/ re-export package)")
    if reference_root not in sys.path:
        sys.path.insert(0, reference_root)

"""The device loop's host side without a GPU: the C ABI exports it, and DeviceLangevin.run_segment checks its
arguments and mode before it touches the device."""
import os
import re

import pytest

from ai2bmd_b200 import engine as vengine
from ai2bmd_b200.md import DeviceLangevin

ROOT = os.path.abspath(os.path.join(os.path.dirname(__file__), ".."))
LOOP_SYMBOLS = ("vb_md_run_loop", "vb_md_request_stop", "vb_md_loop_iterations")


def test_loop_symbols_are_declared_and_exported():
    header = open(os.path.join(ROOT, "include", "visnet_b200.h")).read()
    declared = set(re.findall(r"\b(vb_[a-z_0-9]+)\s*\(", header))
    lib = vengine.load_library()
    for sym in LOOP_SYMBOLS:
        assert sym in declared and sym in vengine.EXPORTED_SYMBOLS and hasattr(lib, sym), sym


class _NoDevice:
    """An engine stand-in that fails on any call reaching the device; options read as a handle without comm."""

    def __init__(self):
        self.calls = []

    def get_option(self, key):
        self.calls.append(key)
        return 0

    def __getattr__(self, name):
        raise AssertionError(f"run_segment reached the engine ({name}) before checking its arguments")


def _stub(group=None):
    dev = DeviceLangevin.__new__(DeviceLangevin)
    dev.engine, dev.group, dev.torch, dev.stream = _NoDevice(), group, None, None
    return dev


@pytest.mark.parametrize("n", [-1, -10 ** 9])
def test_negative_step_count_raises_first(n):
    with pytest.raises(ValueError, match="n_steps must be >= 0"):
        _stub().run_segment(n)


def test_torch_distributed_allreduce_raises_first():
    dev = _stub(group=object())                # a process group, and the handle has no all-reduce of its own
    with pytest.raises(ValueError, match="torch.distributed"):
        dev.run_segment(10)
    assert dev.engine.calls == ["comm_ready"]


class _Interrupted:
    """Stand-ins for the torch event, stream and engine of a run_segment whose wait is interrupted by Ctrl-C."""

    class Event:
        def record(self, stream):
            pass

        def query(self):
            raise KeyboardInterrupt

    def __init__(self, sharded):
        import types
        self.log = []
        self.torch = types.SimpleNamespace(cuda=types.SimpleNamespace(Event=_Interrupted.Event))
        self.stream = types.SimpleNamespace(cuda_stream=0, synchronize=lambda: self.log.append("synchronize"))
        log = self.log

        class Eng:
            def get_option(self, key):
                return 1                                   # comm_ready, comm_auto: the engine's own all-reduce

            def md_run_loop(self, n, stream):
                log.append("md_run_loop")

            def md_request_stop(self):
                log.append("md_request_stop")
                if sharded:                                # vb_md_request_stop refuses one rank of several
                    raise RuntimeError("vb_md_request_stop failed (-3): one rank of 2")

        self.engine = Eng()


@pytest.mark.parametrize("sharded", [False, True])
def test_keyboard_interrupt_waits_and_reraises(sharded):
    fake = _Interrupted(sharded)
    dev = DeviceLangevin.__new__(DeviceLangevin)
    dev.engine, dev.torch, dev.stream = fake.engine, fake.torch, fake.stream
    dev.group = object() if sharded else None
    with pytest.raises(KeyboardInterrupt):
        dev.run_segment(10)
    # one GPU: stop at the next step boundary, then wait; sharded: no stop request (the ranks could not agree on a step),
    # only the wait
    want = ["md_run_loop", "synchronize"] if sharded else ["md_run_loop", "md_request_stop", "synchronize"]
    assert fake.log == want

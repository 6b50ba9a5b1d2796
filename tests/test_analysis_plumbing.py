"""The shared plumbing of the analysis calls (data, inverse, rollout, ik, transition_fd, static_opt), without a device: the input-tensor
check and the initial_state parser of vec_env, the buffer-struct filler of abi, and the oracle extensions the device tests compare
against."""
import ctypes

import numpy as np
import pytest


def test_tensor_check_messages():
    """Every rejection of the input-check tests gives the message that names the expectation and what came in."""
    import torch
    from myosuite_b200.vec_env import _check_f64
    cpu = torch.device("cpu")
    good = torch.zeros(8, 4, 3, dtype=torch.float64)
    _check_f64("ctrl", good, (8, 4, 3), cpu)
    head = "ctrl must be a contiguous float64 tensor of shape (8, 4, 3) on cpu, got "
    cases = {
        "shape": (torch.zeros(8, 4, 2, dtype=torch.float64), "('Tensor', torch.float64, device(type='cpu'), (8, 4, 2), True)"),
        "dtype": (good.float(), "('Tensor', torch.float32, device(type='cpu'), (8, 4, 3), True)"),
        "device": (torch.zeros(8, 4, 3, dtype=torch.float64, device="meta"), "('Tensor', torch.float64, device(type='meta'), (8, 4, 3), True)"),
        "contiguity": (torch.zeros(8, 3, 4, dtype=torch.float64).transpose(1, 2), "('Tensor', torch.float64, device(type='cpu'), (8, 4, 3), False)"),
        "numpy": (good.numpy(), "('ndarray', dtype('float64'), 'cpu', (8, 4, 3), None)"),
    }
    for what, (bad, got) in cases.items():
        with pytest.raises(ValueError) as e:
            _check_f64("ctrl", bad, (8, 4, 3), cpu)
        assert str(e.value) == head + got, what


def test_fields_check():
    from myosuite_b200.vec_env import _check_fields
    assert _check_fields("ik", ["qpos", "err"], ("qpos", "niter", "err")) == ("qpos", "err")
    with pytest.raises(KeyError, match=r"unknown ik fields \['jac'\] \(available: \['qpos', 'niter', 'err'\]\)"):
        _check_fields("ik", ("qpos", "jac"), ("qpos", "niter", "err"))


def test_output_allocation():
    import torch
    from myosuite_b200.vec_env import _output
    cpu = torch.device("cpu")
    x = _output(cpu, (4, 2), ("nv", 3), dict(nv=5))
    assert x.shape == (4, 2, 5, 3) and x.dtype == torch.float64 and bool(torch.isnan(x).all())
    i = _output(cpu, (4,), (), {}, int32=True)
    assert i.shape == (4,) and i.dtype == torch.int32 and bool((i == -1).all())


ROLLOUT_WIDTH = dict(qpos=(7,), qvel=(6,), act=(0,), qacc_warmstart=(6,), time=())
FD_WIDTH = dict(qpos=(7,), qvel=(6,), act=(0,), qacc_warmstart=(6,))


@pytest.mark.parametrize("width", [ROLLOUT_WIDTH, FD_WIDTH], ids=["rollout", "transition_fd"])
def test_initial_state_parser(width):
    """The keys each caller accepts map to the start-state fields; time only for the rollout; a None value is left out."""
    import torch
    from myosuite_b200.vec_env import _initial_state
    cpu = torch.device("cpu")
    state = {k: torch.zeros((3,) + w, dtype=torch.float64) for k, w in width.items()}
    bufs = _initial_state(dict(state, act=None), width, 3, cpu)
    assert set(bufs) == {k + "0" for k in width if k != "act"}
    assert all(bufs[k + "0"] is state[k] for k in width if k != "act")
    assert _initial_state(None, width, 3, cpu) == {}
    for key in ("target", "ctrl") + (() if "time" in width else ("time",)):
        with pytest.raises(KeyError) as e:
            _initial_state({key: torch.zeros(3, dtype=torch.float64)}, width, 3, cpu)
        assert e.value.args[0] == "unknown initial_state key %r (available: %s)" % (key, list(width))
    with pytest.raises(ValueError, match=r"initial_state\['qpos'\] must be a contiguous float64 tensor of shape \(3, 7\)"):
        _initial_state({"qpos": torch.zeros(3, 8, dtype=torch.float64)}, width, 3, cpu)
    if "time" in width:
        with pytest.raises(ValueError, match=r"initial_state\['time'\] must be a contiguous float64 tensor of shape \(3,\)"):
            _initial_state({"time": torch.zeros(3, 1, dtype=torch.float64)}, width, 3, cpu)


def test_buffer_struct_filler():
    import torch
    from myosuite_b200 import abi
    a, b = torch.zeros(4, dtype=torch.float64), torch.zeros(2, 3, dtype=torch.int32)
    s = abi._buffers(abi.MyoInverseBuffers, dict(contact_force=b, qacc=a, actuator_moment=None))
    assert [getattr(s, k) for k in abi.INVERSE_FIELDS] == [a.data_ptr(), None, None, b.data_ptr(), None]
    assert ctypes.sizeof(s) == len(abi.INVERSE_FIELDS) * ctypes.sizeof(ctypes.c_void_p)
    with pytest.raises(KeyError, match="target_pos"):
        abi._buffers(abi.MyoInverseBuffers, dict(qacc=a, target_pos=a))
    with pytest.raises(ValueError, match="^qacc must be contiguous$"):
        abi._buffers(abi.MyoInverseBuffers, dict(qacc=torch.zeros(3, 2, dtype=torch.float64).t()))


def test_oracle_extensions_build():
    """Each oracle extension builds and runs the shipped elbow like the base oracle."""
    from fd_oracle import FdOracle
    from ik_oracle import IkOracle
    from inverse_oracle import InvOracle
    from rollout_oracle import AppliedOracle

    from myosuite_b200 import assets, blob
    from oracle.oracle_py import Oracle
    m = assets.load("myoelbow_1dof6muscles")
    I, D = blob.pack(m)
    nv = len(Oracle(I, D).f("qvel"))
    oracles = [InvOracle(I, D), AppliedOracle(I, D), IkOracle(I, D, m.site_quat), FdOracle(I, D)]
    assert [len(o.f("qvel")) for o in oracles] == [nv] * 4
    assert [len(o.f("qfrc_applied")) for o in oracles[1::2]] == [nv] * 2
    assert np.all(oracles[3].f("qfrc_applied") == 0)

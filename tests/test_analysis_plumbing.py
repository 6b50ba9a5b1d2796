"""The shared plumbing of the analysis calls (data, inverse, rollout, ik, transition_fd, static_opt, cmc), without a device: the input and
parameter checks, the output allocation, the initial_state parser and the row-0 host copy of vec_env, the buffer-struct filler of abi, and
the oracle extensions the device tests compare against."""
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


def test_outputs_allocation():
    """overflow is the [n] int32 zero tensor whatever the lead shape; niter and converged are int32 -1, the rest float64 NaN."""
    import torch
    from myosuite_b200 import abi
    from myosuite_b200.vec_env import _outputs
    cpu = torch.device("cpu")
    out = _outputs(cpu, ("qpos", "niter", "converged", "overflow"), (4, 3), abi.CMC_SHAPES, dict(nq=7))
    assert list(out) == ["qpos", "niter", "converged", "overflow"]
    assert out["qpos"].shape == (4, 3, 7) and out["qpos"].dtype == torch.float64 and bool(torch.isnan(out["qpos"]).all())
    for f in ("niter", "converged"):
        assert out[f].shape == (4, 3) and out[f].dtype == torch.int32 and bool((out[f] == -1).all())
    assert out["overflow"].shape == (4,) and out["overflow"].dtype == torch.int32 and bool((out["overflow"] == 0).all())


def test_flags():
    from myosuite_b200 import abi
    from myosuite_b200.vec_env import _flags
    assert (abi.INV_NOCONSTRAINT, abi.INV_DISCRETE) == (1, 2)
    assert [_flags(c, d) for c in (True, False) for d in (False, True)] == [0, 2, 1, 3]


def test_substeps_and_solver_checks():
    from myosuite_b200 import abi
    from myosuite_b200.vec_env import _check_solver, _check_substeps
    assert _check_substeps(3) == 3 and _check_substeps(2.0) == 2 and isinstance(_check_substeps(2.0), int)
    for bad in (0, -1):
        with pytest.raises(ValueError) as e:
            _check_substeps(bad)
        assert str(e.value) == "substeps must be >= 1, got %d" % bad
    good = abi.MyoStaticOptParams(max_iter=0, tol=0.0)
    assert _check_solver("static_opt", good, 0, 0.0) is good
    cases = (("static_opt", abi.MyoStaticOptParams, -1, 1e-12), ("static_opt", abi.MyoStaticOptParams, 5, -1.0),
             ("cmc", abi.MyoCmcParams, 5, float("nan")), ("cmc", abi.MyoCmcParams, 5, float("inf")))
    for call, P, max_iter, tol in cases:
        with pytest.raises(ValueError) as e:
            _check_solver(call, P(max_iter=max_iter, tol=tol), max_iter, tol)
        assert str(e.value) == "%s needs max_iter >= 0 and a finite tol >= 0, got max_iter %r, tol %r" % (call, max_iter, tol)


def test_vector_parameter():
    """reserve / weight / kp / kv: any numeric scalar, array or tensor of shape () or (width,), finite and > 0 (>= 0 for the gains), as a
    fresh contiguous float64 [width] tensor on the device."""
    import torch
    from myosuite_b200.vec_env import _vector
    cpu = torch.device("cpu")
    want = torch.tensor([1.0, 2.0, 3.0], dtype=torch.float64)
    t64 = want.clone()
    for x in ([1, 2, 3], np.array([1, 2, 3], np.int32), np.array([1, 2, 3], np.float32), want.float(),
              torch.tensor([1.0, 0.0, 2.0, 0.0, 3.0], dtype=torch.float64)[::2], t64):
        v = _vector("reserve", x, 3, cpu)
        assert v.dtype == torch.float64 and v.device == cpu and v.is_contiguous() and torch.equal(v, want), x
    assert _vector("reserve", t64, 3, cpu) is not t64
    for x in (2.5, np.float32(2.5), torch.tensor(2.5, dtype=torch.float32)):
        assert torch.equal(_vector("weight", x, 4, cpu), torch.full((4,), 2.5, dtype=torch.float64))
    assert torch.equal(_vector("kp", 0, 2, cpu, positive=False), torch.zeros(2, dtype=torch.float64))
    rejects = (("reserve", 0.0, True, "reserve must be finite and > 0"), ("reserve", [1.0, float("nan"), 1.0], True, "reserve must be finite and > 0"),
               ("weight", torch.tensor([1.0, -1.0, 1.0]), True, "weight must be finite and > 0"), ("kv", -1e-3, False, "kv must be finite and >= 0"),
               ("kp", float("inf"), False, "kp must be finite and >= 0"),
               ("reserve", np.ones(4), True, "reserve must be a scalar or of shape (3,), got float64 (4,)"),
               ("reserve", torch.ones(1, 3), True, "reserve must be a scalar or of shape (3,), got float32 (1, 3)"),
               ("reserve", "1", True, "reserve must be a scalar or of shape (3,), got <U1 ()"))
    for name, x, positive, msg in rejects:
        with pytest.raises(ValueError) as e:
            _vector(name, x, 3, cpu, positive=positive)
        assert str(e.value) == msg, msg


def test_state_width():
    from types import SimpleNamespace
    from myosuite_b200.vec_env import _state_width
    m = SimpleNamespace(nq=7, nv=6, na=0)
    assert _state_width(m) == ROLLOUT_WIDTH and list(_state_width(m)) == list(ROLLOUT_WIDTH)
    assert _state_width(m, time=False) == FD_WIDTH


def test_row0_unpack():
    """Row 0 of every field in one host copy: trailing shapes and dtypes kept, one-value-per-env fields as Python scalars."""
    import torch
    from myosuite_b200.vec_env import _row0
    g = torch.Generator().manual_seed(0)
    out = {"A": torch.randn(3, 2, 4, dtype=torch.float64, generator=g), "niter": torch.tensor([7, 8, 9], dtype=torch.int32),
           "converged": torch.tensor([[1, 0, 1], [0, 0, 0], [1, 1, 1]], dtype=torch.int32),
           "residual": torch.tensor([2.5e-13, 1.0, 2.0], dtype=torch.float64), "time": torch.randn(3, 5, dtype=torch.float64, generator=g),
           "overflow": torch.tensor([1, 0, 0], dtype=torch.int32), "empty": torch.zeros(3, 0, dtype=torch.float64)}
    r = _row0(out)
    assert list(r) == list(out)
    assert r["A"].shape == (2, 4) and r["A"].dtype == np.float64 and np.array_equal(r["A"], out["A"][0].numpy())
    assert r["time"].shape == (5,) and np.array_equal(r["time"], out["time"][0].numpy())
    assert r["converged"].dtype == np.int32 and r["converged"].shape == (3,) and r["converged"].tolist() == [1, 0, 1]
    assert type(r["niter"]) is int and r["niter"] == 7 and type(r["overflow"]) is int and r["overflow"] == 1
    assert type(r["residual"]) is float and r["residual"] == 2.5e-13
    assert r["empty"].shape == (0,)
    assert _row0({}) == {}


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

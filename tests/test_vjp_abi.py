"""CPU: mvs_forward_vjp is declared, exported and bound with its argument types; the Python surface exists."""
import ctypes
import inspect


def test_forward_vjp_symbol_and_argtypes():
    from mvsmplfitting_b200 import _lib, build
    build.build()
    lib = _lib.load()
    assert "mvs_forward_vjp" in _lib.EXPORTS
    assert hasattr(ctypes.CDLL(build.OUT), "mvs_forward_vjp")
    assert lib.mvs_forward_vjp.argtypes == [ctypes.c_void_p] * 6      # ctx, params, djoints, dverts, dparams, stream


def test_forward_vjp_python_surface():
    from mvsmplfitting_b200 import smplx
    from mvsmplfitting_b200.autograd import SMPLFunction
    from mvsmplfitting_b200.context import FittingContext
    assert list(inspect.signature(FittingContext.forward_vjp).parameters) == ["self", "params", "djoints", "dverts"]
    assert inspect.signature(smplx.SMPL.__init__).parameters["differentiable"].default is False
    assert hasattr(SMPLFunction, "backward")

"""Host-only rules of the shaped fused step (gantts_gan_step_shaped) and of the device MLPG table builder: every call
shape outside the configured capacity, and a null table, is refused with a message naming the rule before any device
work, so these run without a GPU."""
import ctypes

import pytest

from conftest import WINDOWS
from fused_step_helpers import FAKE, TTS_STREAMS, config_checker, fill_tables, step_config


@pytest.fixture(scope="module")
def lib():
    config_checker()            # builds the library
    from gantts_b200 import _lib
    return _lib.load()


def mlp_config():
    c = step_config([20, 32, 187], [58, 16, 1], TTS_STREAMS, list(range(60)) + [180, 183, 184], list(range(2, 60)))
    return fill_tables(c, 4)


def shaped(lib, c, B, T, table=FAKE):
    return lib.gantts_gan_step_shaped(ctypes.byref(c), B, T, table, 7, FAKE, FAKE, FAKE, 0.0, 1, FAKE, FAKE, FAKE, FAKE,
                                      1 << 40, None)


@pytest.mark.parametrize("B,T,table,needle", [
    (0, 16, FAKE, "batch size B = 0 must be in [1, configured B = 2]"),
    (3, 16, FAKE, "batch size B = 3 must be in [1, configured B = 2]"),
    (2, 0, FAKE, "padded length T = 0 must be in [1, configured T = 16]"),
    (1, 17, FAKE, "padded length T = 17 must be in [1, configured T = 16]"),
    (2, 16, None, "null MLPG table"),
])
def test_shaped_step_refuses_shapes_outside_the_capacity(lib, B, T, table, needle):
    c = mlp_config()
    assert lib.gantts_gan_step_workspace_bytes(ctypes.byref(c)) > 0          # the configuration itself is accepted
    rc = shaped(lib, c, B, T, table)
    msg = lib.gantts_last_error_string().decode()
    assert rc != 0 and needle in msg, (rc, msg)


def test_shaped_step_checks_the_configuration_first(lib):
    c = mlp_config()
    c.n_static_cols = 1
    assert shaped(lib, c, 1, 1) != 0
    assert "static column list" in lib.gantts_last_error_string().decode()


def test_device_table_builder_refuses_bad_arguments(lib):
    from gantts_b200 import _lib
    w = _lib.make_windows(WINDOWS)
    assert lib.gantts_mlpg_table_device(ctypes.byref(w), 0, FAKE, None) != 0
    assert "mlpg_table_device: bad arguments" in lib.gantts_last_error_string().decode()
    assert lib.gantts_mlpg_table_device(ctypes.byref(w), 8, None, None) != 0
    w.l[1] = 3
    assert lib.gantts_mlpg_table_device(ctypes.byref(w), 8, FAKE, None) != 0
    assert "window 1 taps out of range" in lib.gantts_last_error_string().decode()


def test_new_symbols_have_their_ctypes_signatures(lib):
    from gantts_b200 import _lib
    res, args = _lib.SIGNATURES["gantts_gan_step_shaped"]
    base_res, base_args = _lib.SIGNATURES["gantts_gan_step"]
    # (cfg, B, T, table) then the remaining arguments of gantts_gan_step
    assert res is base_res and args[0] is base_args[0] and args[4:] == base_args[1:]
    assert args[1:4] == [ctypes.c_int, ctypes.c_int, ctypes.c_void_p]
    assert _lib.SIGNATURES["gantts_mlpg_table_device"] == (ctypes.c_int, [ctypes.POINTER(_lib.WindowsT), ctypes.c_int,
                                                                          ctypes.c_void_p, ctypes.c_void_p])
    for name in ("gantts_gan_step_shaped", "gantts_mlpg_table_device"):
        assert getattr(lib, name).argtypes == _lib.SIGNATURES[name][1]

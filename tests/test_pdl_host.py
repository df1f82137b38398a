"""ops.pdl, the Python state behind programmatic dependent launch (no GPU needed): blocks nest, the enclosing mode comes
back on exit, and a library build loaded inside a block starts in the block's mode.  Stand-in libraries record what
vl2_set_pdl receives; whether the real library then launches with the attribute is checked by the captured decode
graph's programmatic edges (test_pdl_gpu.py)."""
from unittest import mock

import pytest

from videollama2_b200 import _lib, ops


class _Recorder:
    def __init__(self):
        self.modes = []

    def vl2_set_pdl(self, mode):
        self.modes.append(mode)
        return 0

    @property
    def mode(self):
        return self.modes[-1] if self.modes else -1


@pytest.fixture
def libs(monkeypatch):
    bf16 = _Recorder()
    monkeypatch.setattr(_lib, "_libs", {"bf16": bf16})
    monkeypatch.setattr(_lib, "pdl_mode", -1)
    return bf16


def test_blocks_nest_and_restore_the_outer_mode(libs):
    with ops.pdl(True):
        assert libs.mode == 1 and _lib.pdl_mode == 1
        with ops.pdl(False):
            assert libs.mode == 0
            with ops.pdl(True):
                assert libs.mode == 1
            assert libs.mode == 0
        assert libs.mode == 1 and _lib.pdl_mode == 1
    assert libs.mode == -1 and _lib.pdl_mode == -1       # outside every block: follow VL2_PDL again
    assert libs.modes == [1, 0, 1, 0, 1, -1]


def test_the_outer_mode_comes_back_after_an_exception(libs):
    with ops.pdl(False):
        with pytest.raises(RuntimeError):
            with ops.pdl(True):
                raise RuntimeError("inside")
        assert libs.mode == 0
    assert libs.mode == -1


def test_one_instance_reentered(libs):
    on = ops.pdl(True)
    with ops.pdl(False):
        with on:
            with ops.pdl(False):
                with on:
                    assert libs.mode == 1
                assert libs.mode == 0
            assert libs.mode == 1
        assert libs.mode == 0
    assert libs.mode == -1


def test_a_build_loaded_inside_a_block_follows_it(libs, monkeypatch, tmp_path):
    """_lib.load itself, with the fp16 build's shared object replaced by a recording stand-in."""
    f16 = mock.MagicMock()
    f16.vl2_storage_dtype.return_value = 1
    f16.vl2_set_pdl.return_value = 0
    path = tmp_path / "libvl2_f16.so"
    path.write_bytes(b"")
    monkeypatch.setattr(_lib, "LIB_PATH_F16", str(path))
    monkeypatch.setattr(_lib.C, "CDLL", lambda p: f16 if p == str(path) else pytest.fail(p))
    mode = lambda: f16.vl2_set_pdl.call_args.args[0]
    with ops.pdl(True):
        assert _lib.load("f16") is f16 and mode() == 1
        with ops.pdl(False):
            assert mode() == 0 and libs.mode == 0
        assert mode() == 1
    assert mode() == -1 and libs.mode == -1
    _lib.load("f16")                           # already loaded: not switched again
    assert [c.args[0] for c in f16.vl2_set_pdl.call_args_list] == [1, 0, 1, -1]


def test_bad_mode_is_refused(libs):
    with pytest.raises(ValueError):
        _lib.set_pdl(2)
    assert _lib.pdl_mode == -1 and libs.modes == []

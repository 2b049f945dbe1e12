"""Host-only checks of growing model banks: the options field that reserves a bank's capacity, the exported entry points
and the Python signatures.  No GPU needed."""
import ctypes
import inspect

import neuralampmodelercore_b200 as nb
from neuralampmodelercore_b200 import _capi

NEW_SYMBOLS = ("nam_b200_bank_capacity", "nam_b200_bank_add_models", "nam_b200_bank_replace_model")


def test_bank_capacity_takes_the_first_reserved_word():
    o = _capi.Options
    assert ctypes.sizeof(o) == 56
    assert o.bank_capacity.offset == o.jit.offset + 4 == 36
    assert o.reserved.offset == 40 and o.reserved.size == 16
    lib = _capi.load()
    opts = o()
    ctypes.memset(ctypes.byref(opts), 0x5A, ctypes.sizeof(opts))
    lib.nam_b200_default_options(ctypes.byref(opts))
    assert opts.struct_size == 56 and opts.bank_capacity == 0
    assert lib.nam_b200_abi_version() == 1


def test_new_entry_points_are_exported_and_declared():
    lib = _capi.load()
    header = (_capi.lib_path().parents[2] / "include" / "nam_b200.h").read_text()
    for name in NEW_SYMBOLS:
        assert name in _capi.EXPORTED_SYMBOLS
        assert hasattr(lib, name), name
        assert f"int {name}(" in header, name
    assert "int32_t bank_capacity;" in header and "int32_t reserved[4];" in header


def test_python_signatures_take_the_new_arguments():
    assert inspect.signature(nb.get_dsp_bank).parameters["capacity"].default == 0
    assert isinstance(inspect.getattr_static(nb.DSP, "bank_capacity"), property)
    assert list(inspect.signature(nb.DSP.add_models).parameters) == ["self", "configs"]
    assert list(inspect.signature(nb.DSP.replace_model).parameters) == ["self", "k", "config"]

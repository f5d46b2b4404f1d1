"""Swap preemption without a GPU: the ctypes aha_swap_stats against the header, and the argument checks of the Python wrappers."""
import ctypes as C
import os
import re

import pytest

from conftest import ROOT


def _header_struct(name):
    text = open(os.path.join(ROOT, "include", "aha_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    body = re.search(r"typedef struct " + name + r" \{(.*?)\} " + name + ";", text, flags=re.S).group(1)
    fields = []
    for decl in body.split(";"):
        decl = decl.strip()
        if decl:
            ctype, names = decl.split(None, 1)
            fields += [(n.strip(), ctype) for n in names.split(",")]
    return fields


def test_swap_stats_matches_the_header():
    from aha_b200 import _lib as L
    ctypes_of = {"uint64_t": C.c_uint64, "double": C.c_double}
    assert [(n, ctypes_of[t]) for n, t in _header_struct("aha_swap_stats")] == list(L.SwapStats._fields_)
    assert C.sizeof(L.SwapStats) == 72 and L.SwapStats.suspend_secs.offset == 56


class _NoLib:
    def __getattr__(self, name):
        raise AssertionError(f"{name} called although the arguments are invalid")


@pytest.mark.parametrize("call,args,err", [
    ("batch_swap_space", (-1,), ValueError), ("batch_swap_space", (1.5,), TypeError), ("batch_swap_space", (None,), TypeError),
    ("batch_cancel", (-1,), ValueError), ("batch_cancel", (64,), ValueError), ("batch_cancel", (True,), TypeError),
    ("batch_suspend", (-1,), ValueError), ("batch_suspend", ("0",), TypeError),
    ("batch_resume", (0,), ValueError), ("batch_resume", (2 ** 32,), ValueError), ("batch_resume", (1.0,), TypeError),
    ("batch_discard", (0,), ValueError), ("batch_discard", (False,), TypeError),
])
def test_wrappers_check_their_arguments(call, args, err):
    from aha_b200 import B200Model
    m = B200Model.__new__(B200Model)
    m._lib, m._h = _NoLib(), None
    with pytest.raises(err):
        getattr(m, call)(*args)


def test_swap_int():
    import numpy as np
    from aha_b200 import _lib as L
    assert L.swap_int("slot", np.int64(5), 0, 63) == 5 and L.swap_int("id", 2 ** 32 - 1, 1, 2 ** 32 - 1) == 2 ** 32 - 1

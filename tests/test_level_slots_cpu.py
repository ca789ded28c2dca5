"""Option "level_slots" without a GPU: the option refuses a null handle, and the header documents it with its two values.  The values, the
call order and everything the option changes need an engine and are checked in test_level_slots_gpu.py."""
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_level_slots_refuses_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    for d in (0, 2, 3, 4, 8):
        assert L.mv_set_option(None, b"level_slots", d) == capi.MV_ERR_ARG


def test_level_slots_is_documented(built):
    with open(os.path.join(ROOT, "include", "megaverse_b200.h")) as f:
        header = f.read()
    assert '"level_slots" (2 or 4, before the first reset' in header
    assert 'option "level_slots" 4' in header  # the asynchronous calls' contract texts name the way out

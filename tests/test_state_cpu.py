"""Env state store entry points without a GPU: every mv_states_* call refuses a null handle."""
import ctypes as C


def test_state_calls_refuse_a_null_handle(built):
    from megaverse_b200 import capi

    L = capi.lib()
    store, rows, nbytes = C.c_int(), (C.c_int32 * 1)(0), C.c_int64()
    assert L.mv_states_create(None, 1, C.byref(store)) == capi.MV_ERR_ARG
    assert L.mv_states_save(None, 0, rows, rows, 1) == capi.MV_ERR_ARG
    assert L.mv_states_load(None, 0, rows, rows, 1) == capi.MV_ERR_ARG
    assert L.mv_states_destroy(None, 0) == capi.MV_ERR_ARG
    assert L.mv_state_row_bytes(None, C.byref(nbytes)) == capi.MV_ERR_ARG

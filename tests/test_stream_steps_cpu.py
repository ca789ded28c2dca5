"""Stream steps (mv_step_stream) without a GPU: the export, its ctypes signature and the null-handle refusal."""
import ctypes as C


def test_export_and_signature(built):
    from megaverse_b200 import capi

    assert "mv_step_stream" in capi.EXPORTS
    fn = capi.lib().mv_step_stream
    assert fn.argtypes == [C.c_void_p] * 5
    assert callable(capi.Engine.step_stream)


def test_null_handle(built):
    from megaverse_b200 import capi

    assert capi.lib().mv_step_stream(None, None, None, None, None) == capi.MV_ERR_ARG

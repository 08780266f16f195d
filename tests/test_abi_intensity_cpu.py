"""CPU-side checks of the intensity additions to the C ABI: the new records' sizes and field
offsets match the C compiler's view of include/csm_abi.h, and bad arguments return
CSM_E_INVALID before any device is touched."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def csm():
    from cartographer_b200 import _lib
    if not os.path.exists(_lib.SO_PATH):
        _lib.build()
    return _lib


def _compile_and_run(src):
    with tempfile.TemporaryDirectory() as d:
        open(os.path.join(d, "t.c"), "w").write(src)
        subprocess.check_call(["gcc", "-I", ROOT, os.path.join(d, "t.c"), "-o", os.path.join(d, "t")])
        return [int(v) for v in subprocess.check_output([os.path.join(d, "t")]).split()]


def test_intensity_struct_layouts(csm):
    from cartographer_b200 import scan_matching as sm
    records = [("csm_ceres_intensity_job3d", sm.CsmCeresIntensityJob3D),
               ("csm_ceres_intensity_options3d", sm.CsmCeresIntensityOptions3D)]
    head = '#include <stdio.h>\n#include <stddef.h>\n#include "include/csm_abi.h"\nint main(){'
    sizes = _compile_and_run(head + "".join('printf("%%zu\\n", sizeof(%s));' % n
                                            for n, _ in records) + "}")
    assert sizes == [C.sizeof(t) for _, t in records]
    fields = [(n, t, f[0]) for n, t in records for f in t._fields_]
    offsets = _compile_and_run(head + "".join('printf("%%zu\\n", offsetof(%s, %s));' % (n, f)
                                              for n, _, f in fields) + "}")
    assert offsets == [getattr(t, f).offset for _, t, f in fields]


def test_invalid_arguments_return_status(csm):
    lib = csm.lib()
    out = C.c_void_p()
    idx = np.zeros((1, 3), np.int32)
    s, c = np.ones(1, np.float32), np.ones(1, np.int32)
    p = lambda a, t: a.ctypes.data_as(C.POINTER(t))  # noqa: E731
    assert lib.csm_intensity_grid3d_create(p(idx, C.c_int32), p(s, C.c_float), p(c, C.c_int32),
                                           C.c_int64(1), C.c_float(0.0), 0, C.byref(out)) == 1
    assert lib.csm_intensity_grid3d_create(None, None, None, C.c_int64(1), C.c_float(0.1), 0,
                                           C.byref(out)) == 1
    assert lib.csm_intensity_grid3d_create(p(idx, C.c_int32), p(s, C.c_float), p(c, C.c_int32),
                                           C.c_int64(-1), C.c_float(0.1), 0, C.byref(out)) == 1
    assert lib.csm_intensity_grid3d_destroy(None) == 0
    from cartographer_b200 import scan_matching as sm
    job, res = sm.CsmCeresJob3D(), sm.CsmCeresResult3D()
    opt, iopt = sm.CeresScanMatcherOptions3D()._c(), sm.CeresScanMatcherOptions3D()._c_intensity()
    # no intensity records / no job
    assert lib.csm_ceres_match3d_intensity_batch(C.byref(job), None, 1, C.byref(opt),
                                                 C.byref(iopt), C.byref(res), None) == 1
    assert lib.csm_ceres_evaluate3d_intensity(None, None, C.byref(opt), C.byref(iopt), None,
                                              None, None) == 1

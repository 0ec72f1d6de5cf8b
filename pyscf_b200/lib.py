"""ctypes binding of libb200jk.so (C ABI: include/b200jk.h).

This is the only place the product loads native code.  There is no CPU fallback: if the CUDA
library is missing or no GPU is present the calls raise RuntimeError (SURVEY.md §8b error
conventions; reference analogue: lib.load_library, pyscf/lib/misc.py:123).
"""
import ctypes
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(_HERE, 'libb200jk.so')

c_double_p = ctypes.POINTER(ctypes.c_double)
c_int_p = ctypes.POINTER(ctypes.c_int32)


class Stats(ctypes.Structure):
    _fields_ = [('ms_total', ctypes.c_double), ('ms_kernels', ctypes.c_double), ('ms_h2d', ctypes.c_double),
                ('ms_d2h', ctypes.c_double), ('quartets_computed', ctypes.c_uint64),
                ('quartets_screened', ctypes.c_uint64), ('kernel_launches', ctypes.c_uint64),
                ('n_dev_shells', ctypes.c_int32), ('n_cart', ctypes.c_int32), ('n_sph', ctypes.c_int32),
                ('n_pairs', ctypes.c_int32)]


class I8Test(ctypes.Structure):
    """b200jk_i8test: arguments and outputs of b200jk_i8engine_test (include/b200jk.h)."""
    _fields_ = [('stage', ctypes.c_int), ('packed', ctypes.c_int), ('ns', ctypes.c_int),
                ('a', c_double_p), ('ra', ctypes.c_int), ('k', ctypes.c_int), ('a_rowmax', c_double_p),
                ('b', c_double_p), ('rb', ctypes.c_int),
                ('a_row0', ctypes.c_int), ('m', ctypes.c_int), ('inner', ctypes.c_int), ('y_ncolp', ctypes.c_int),
                ('symmetric', ctypes.c_int), ('kb_per', ctypes.c_int),
                ('qa', ctypes.c_void_p), ('ea', c_int_p), ('qb', ctypes.c_void_p), ('eb', c_int_p), ('rowexp', c_int_p),
                ('rownorm2', ctypes.POINTER(ctypes.c_float)),
                ('c', c_double_p), ('rowmax', c_double_p), ('qy', ctypes.c_void_p), ('ey', c_int_p)]


_libs = {}

SYMBOLS = ['b200jk_create', 'b200jk_create2', 'b200jk_destroy', 'b200jk_set_screening', 'b200jk_direct_jk', 'b200jk_direct_jk_device',
           'b200jk_df_build', 'b200jk_df_jk', 'b200jk_df_naux', 'b200jk_get_q_cond', 'b200jk_get_stats',
           'b200jk_last_error', 'b200jk_version', 'b200jk_set_stream', 'b200jk_fp64_peak',
           'b200jk_set_profile', 'b200jk_get_class_times', 'b200jk_df_get_cderi', 'b200jk_i8gemm_test', 'b200jk_i8engine_test', 'b200jk_df_set_kmode', 'b200jk_df_set_kblock', 'b200jk_set_shard', 'b200jk_df_jk_device', 'b200jk_df_local_rows',
           'b200jk_df_prepare_j', 'b200jk_df_direct_j', 'b200jk_df_stage_times', 'b200jk_df_set_cderi', 'b200jk_df_get_cderi_cols',
           'b200jk_incore_set_eri', 'b200jk_incore_jk', 'b200jk_set_class_costs',
           'b200jk_df_set_device_rows', 'b200jk_df_row_split', 'b200jk_df_stream_stats',
           'b200jk_df_set_pair_tol', 'b200jk_df_pair_stats', 'b200jk_rys_test', 'b200jk_df_set_raw_test',
           'b200jk_df_get_metric_test', 'b200jk_get_dm_cond_test', 'b200jk_df_ao2mo', 'b200jk_df_get_ao_eri',
           'b200jk_df_set_ao2mo_tile', 'b200jk_df_ao2mo_times', 'b200jk_df_mp2', 'b200jk_df_mp2_times',
           'b200jk_df_rpa', 'b200jk_df_rpa_times']


def load(path=None):
    path = path or DEFAULT_LIB
    if path in _libs:
        return _libs[path]
    if not os.path.exists(path):
        raise RuntimeError('libb200jk.so not found at %s: build it with `python -c "import __graft_entry__ as g; '
                           'g.build()"`; pyscf_b200 has no CPU fallback' % path)
    lib = ctypes.CDLL(path)
    vp = ctypes.c_void_p
    lib.b200jk_create.argtypes = [ctypes.POINTER(vp), c_int_p, ctypes.c_int, c_int_p, ctypes.c_int, c_double_p,
                                  ctypes.c_int, ctypes.c_int]
    lib.b200jk_create2.argtypes = [ctypes.POINTER(vp), c_int_p, ctypes.c_int, c_int_p, ctypes.c_int, c_double_p,
                                   ctypes.c_int, ctypes.c_int, ctypes.c_int]
    lib.b200jk_destroy.argtypes = [vp]
    lib.b200jk_set_screening.argtypes = [vp, ctypes.c_double, ctypes.c_double]
    lib.b200jk_direct_jk.argtypes = [vp, c_double_p, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_double_p, c_double_p]
    lib.b200jk_direct_jk_device.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, vp, vp]
    lib.b200jk_df_build.argtypes = [vp, c_int_p, ctypes.c_int, c_int_p, ctypes.c_int, c_double_p, ctypes.c_int,
                                    ctypes.c_double, ctypes.c_double]
    lib.b200jk_df_prepare_j.argtypes = [vp, c_int_p, ctypes.c_int, c_int_p, ctypes.c_int, c_double_p, ctypes.c_int,
                                        ctypes.c_double, ctypes.c_double]
    lib.b200jk_df_direct_j.argtypes = [vp, c_double_p, ctypes.c_int, ctypes.c_int, c_double_p]
    lib.b200jk_df_jk.argtypes = [vp, c_double_p, ctypes.c_int, ctypes.c_int, c_double_p, ctypes.c_int, ctypes.c_int,
                                 c_double_p, c_double_p]
    lib.b200jk_df_naux.argtypes = [vp, ctypes.POINTER(ctypes.c_int)]
    lib.b200jk_df_stage_times.argtypes = [vp, c_double_p, c_int_p, ctypes.c_int]
    lib.b200jk_df_set_cderi.argtypes = [vp, c_double_p, ctypes.c_int, ctypes.c_int]
    lib.b200jk_df_get_cderi.argtypes = [vp, c_double_p, ctypes.c_int, ctypes.c_int]
    lib.b200jk_set_class_costs.argtypes = [vp, c_double_p, ctypes.c_int]
    lib.b200jk_incore_set_eri.argtypes = [vp, c_double_p, ctypes.c_int64, ctypes.c_int]
    lib.b200jk_incore_jk.argtypes = [vp, c_double_p, ctypes.c_int, ctypes.c_int, c_double_p, c_double_p]
    lib.b200jk_df_get_cderi_cols.argtypes = [vp, c_double_p, ctypes.POINTER(ctypes.c_int64), ctypes.c_int]
    lib.b200jk_i8gemm_test.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int, c_double_p, c_double_p, c_double_p,
                                       ctypes.c_int, ctypes.c_int]
    lib.b200jk_i8engine_test.argtypes = [vp, ctypes.POINTER(I8Test)]
    lib.b200jk_rys_test.argtypes = [vp, ctypes.c_int, ctypes.c_int, c_double_p, c_double_p, c_double_p]
    lib.b200jk_df_set_kblock.argtypes = [vp, ctypes.c_int, ctypes.c_int]
    lib.b200jk_df_set_kmode.argtypes = [vp, ctypes.c_int, ctypes.c_int]
    lib.b200jk_df_set_device_rows.argtypes = [vp, ctypes.c_int]
    lib.b200jk_df_row_split.argtypes = [vp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    lib.b200jk_df_stream_stats.argtypes = [vp, ctypes.POINTER(ctypes.c_int64), c_double_p, c_double_p]
    lib.b200jk_df_set_pair_tol.argtypes = [vp, ctypes.c_double]
    lib.b200jk_df_pair_stats.argtypes = [vp, ctypes.POINTER(ctypes.c_int64), ctypes.POINTER(ctypes.c_int64)]
    lib.b200jk_df_set_raw_test.argtypes = [vp, ctypes.c_int]
    lib.b200jk_df_get_metric_test.argtypes = [vp, c_double_p, ctypes.c_int]
    lib.b200jk_df_ao2mo.argtypes = [vp, c_double_p, ctypes.c_int, c_double_p, ctypes.c_int, ctypes.c_int, c_double_p, ctypes.c_int,
                                    c_double_p, ctypes.c_int, ctypes.c_int, c_double_p]
    lib.b200jk_df_get_ao_eri.argtypes = [vp, c_double_p]
    lib.b200jk_df_set_ao2mo_tile.argtypes = [vp, ctypes.c_int]
    lib.b200jk_df_ao2mo_times.argtypes = [vp, c_double_p, ctypes.c_int]
    c_double_pp = ctypes.POINTER(c_double_p)
    lib.b200jk_df_mp2.argtypes = [vp, ctypes.c_int, c_double_pp, c_int_p, c_double_pp, c_int_p, c_double_pp, c_double_pp, c_double_p,
                                  c_double_pp]
    lib.b200jk_df_mp2_times.argtypes = [vp, c_double_p, ctypes.c_int]
    lib.b200jk_df_rpa.argtypes = [vp, ctypes.c_int, c_double_pp, c_int_p, c_double_pp, c_int_p, c_double_pp, c_double_pp, ctypes.c_int,
                                  c_double_p, c_double_p, c_double_p, c_double_p]
    lib.b200jk_df_rpa_times.argtypes = [vp, c_double_p, ctypes.c_int]
    lib.b200jk_df_local_rows.argtypes = [vp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_int)]
    lib.b200jk_set_shard.argtypes = [vp, ctypes.c_int, ctypes.c_int]
    lib.b200jk_df_jk_device.argtypes = [vp, vp, ctypes.c_int, ctypes.c_int, vp, ctypes.c_int, ctypes.c_int, vp, vp]
    lib.b200jk_get_q_cond.argtypes = [vp, c_double_p, ctypes.c_int]
    lib.b200jk_get_dm_cond_test.argtypes = [vp, c_double_p, c_int_p, ctypes.c_int]
    lib.b200jk_get_stats.argtypes = [vp, ctypes.POINTER(Stats)]
    lib.b200jk_set_stream.argtypes = [vp, vp]
    lib.b200jk_fp64_peak.argtypes = [vp, c_double_p]
    lib.b200jk_set_profile.argtypes = [vp, ctypes.c_int]
    lib.b200jk_get_class_times.argtypes = [vp, c_double_p, ctypes.c_int]
    lib.b200jk_last_error.argtypes = [vp]
    lib.b200jk_last_error.restype = ctypes.c_char_p
    lib.b200jk_version.restype = ctypes.c_char_p
    _libs[path] = lib
    return lib


def dptr(a):
    return None if a is None else a.ctypes.data_as(c_double_p)


def iptr(a):
    return a.ctypes.data_as(c_int_p)


class Handle:
    """Owns one b200jk_handle (device memory for one molecule/basis)."""

    def __init__(self, atm, bas, env, device=0, libpath=None, cart=False):
        self.lib = load(libpath)
        self.cart = bool(cart)
        self._h = ctypes.c_void_p()
        self.atm = np.ascontiguousarray(atm, dtype=np.int32)
        self.bas = np.ascontiguousarray(bas, dtype=np.int32)
        self.env = np.ascontiguousarray(env, dtype=np.float64)
        rc = self.lib.b200jk_create2(ctypes.byref(self._h), iptr(self.atm), len(self.atm), iptr(self.bas),
                                     len(self.bas), dptr(self.env), len(self.env), device, int(self.cart))
        if rc != 0:
            msg = self.lib.b200jk_last_error(self._h).decode() if self._h else 'b200jk_create failed'
            if self._h:
                self.lib.b200jk_destroy(self._h)
                self._h = ctypes.c_void_p()
            raise RuntimeError('b200jk_create: ' + msg)

    def check(self, rc, what):
        if rc != 0:
            raise RuntimeError('%s: %s' % (what, self.lib.b200jk_last_error(self._h).decode()))

    def stats(self):
        s = Stats()
        self.lib.b200jk_get_stats(self._h, ctypes.byref(s))
        return {k: getattr(s, k) for k, _ in Stats._fields_}

    DF_STAGES = ('j_rho', 'j_acc', 'k_gemm1', 'k_slice', 'k_gemm2')   # B200JK_DF_STAGE_* of include/b200jk.h

    def df_stage_times(self):
        """{stage: (milliseconds, launches)} of the last DF J/K call (CUDA events around every launch)."""
        n = len(self.DF_STAGES)
        ms = np.zeros(n)
        cnt = np.zeros(n, dtype=np.int32)
        self.check(self.lib.b200jk_df_stage_times(self._h, dptr(ms), iptr(cnt), n), 'b200jk_df_stage_times')
        return {k: (float(ms[i]), int(cnt[i])) for i, k in enumerate(self.DF_STAGES)}

    def close(self):
        if getattr(self, '_h', None) and self._h:
            self.lib.b200jk_destroy(self._h)
            self._h = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

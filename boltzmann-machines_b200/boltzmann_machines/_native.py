"""ctypes binding of ``libbm.so`` (C-ABI in ``include/bm.h``) and the engine
objects the model classes talk to.

There is deliberately no fallback here: if the shared library is missing, was
not built for this GPU, or no GPU is visible, construction raises
``RuntimeError`` with the library's own message.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libbm.so')

UNIT_KINDS = {'bernoulli': 0, 'multinomial': 1, 'gaussian': 2}
DTYPES = {'float32': 0, 'float64': 1}
COMPUTE = {'fp32': 0, 'bf16': 1}
METRIC_BITS = {'l2_loss': 1, 'msre': 2, 'pll': 4, 'free_energy': 8}
METRIC_SLOTS = {'l2_loss': 0, 'msre': 1, 'pll': 2, 'free_energy': 3}

# every symbol include/bm.h declares (tests check the library exports all of them)
EXPORTS = (
    'bm_version', 'bm_last_error', 'bm_device_count', 'bm_ctx_create', 'bm_ctx_destroy', 'bm_ctx_sync',
    'bm_ctx_timer_start', 'bm_ctx_timer_stop', 'bm_ctx_flush_l2', 'bm_host_alloc', 'bm_host_free',
    'bm_host_pack_u8', 'bm_host_pack_bf16',
    'bm_ctx_launch_count', 'bm_ctx_profile_tc', 'bm_ctx_profile_read', 'bm_comm_unique_id', 'bm_ctx_comm_init',
    'bm_rbm_create', 'bm_rbm_destroy', 'bm_rbm_set_param', 'bm_rbm_get_param', 'bm_rbm_init_weights',
    'bm_rbm_train_step', 'bm_rbm_set_data', 'bm_rbm_train_step_at', 'bm_rbm_train_epoch', 'bm_rbm_train_epoch_u8', 'bm_rbm_train_epoch_bf16', 'bm_rbm_transform', 'bm_rbm_metrics',
    'bm_rbm_get_activation', 'bm_debug_tc_gemm', 'bm_debug_tc_op', 'bm_rbm_debug_tc_plan',
    'bm_dbm_create', 'bm_dbm_destroy', 'bm_dbm_set_param', 'bm_dbm_get_param', 'bm_dbm_init_particles',
    'bm_dbm_train_step', 'bm_dbm_val_metrics', 'bm_dbm_transform', 'bm_dbm_reconstruct', 'bm_dbm_log_proba',
    'bm_dbm_sample_v', 'bm_dbm_ais', 'bm_dbm_ais_rows', 'bm_dbm_ais_base', 'bm_dbm_ais_base_rows', 'bm_dbm_pt_counts', 'bm_debug_dbm_multinomial_rows',
    'bm_dbm_train_step_labeled', 'bm_dbm_predict_proba', 'bm_dbm_fill', 'bm_dbm_debug_last_fill', 'bm_dbm_debug_last_sample_v',
    'bm_dbm_exact', 'bm_dbm_debug_exact_chunk', 'bm_dbm_ais_clamped',
    'bm_crbm_create', 'bm_crbm_destroy', 'bm_crbm_set_param', 'bm_crbm_get_param', 'bm_crbm_init_weights',
    'bm_crbm_train_step', 'bm_crbm_predict_proba', 'bm_crbm_transform', 'bm_crbm_debug_last_step',
    'bm_rbm_group_create', 'bm_rbm_group_destroy', 'bm_rbm_group_train_epoch', 'bm_rbm_group_train_epoch_u8',
    'bm_rbm_group_train_epoch_bf16',
)


class RbmCfg(C.Structure):
    _fields_ = [
        ('n_visible', C.c_int32), ('n_hidden', C.c_int32),
        ('v_kind', C.c_int32), ('h_kind', C.c_int32),
        ('dtype', C.c_int32), ('compute', C.c_int32),
        ('sample_v', C.c_int32), ('sample_h', C.c_int32),
        ('max_batch', C.c_int32), ('reserved0', C.c_int32),
        ('l2', C.c_double), ('dropout_keep', C.c_double),
        ('sparsity_target', C.c_double), ('sparsity_cost', C.c_double), ('sparsity_damping', C.c_double),
        ('propup_mult', C.c_double), ('propdown_mult', C.c_double),
        ('v_n_samples', C.c_double), ('h_n_samples', C.c_double),
        ('sigma', C.POINTER(C.c_double)),
    ]


class DbmCfg(C.Structure):
    _fields_ = [
        ('n_layers', C.c_int32), ('n_visible', C.c_int32),
        ('n_hiddens', C.POINTER(C.c_int32)),
        ('v_kind', C.c_int32),
        ('h_kinds', C.POINTER(C.c_int32)),
        ('h_n_samples', C.POINTER(C.c_double)),
        ('dtype', C.c_int32), ('compute', C.c_int32),
        ('n_particles', C.c_int32), ('batch_size', C.c_int32), ('max_mf_updates', C.c_int32),
        ('sample_v', C.c_int32),
        ('sample_h', C.POINTER(C.c_int32)),
        ('mf_tol', C.c_double), ('l2', C.c_double), ('max_norm', C.c_double), ('sparsity_damping', C.c_double),
        ('sparsity_target', C.POINTER(C.c_double)),
        ('sparsity_cost', C.POINTER(C.c_double)),
        ('sigma', C.POINTER(C.c_double)),
        ('n_temps', C.c_int32),
        ('betas', C.POINTER(C.c_double)),
        ('n_classes', C.c_int32),
        ('centering', C.c_int32),
        ('offset_rate', C.c_double),
    ]


class CrbmCfg(C.Structure):
    _fields_ = [
        ('n_visible', C.c_int32), ('n_hidden', C.c_int32), ('n_classes', C.c_int32),
        ('dtype', C.c_int32), ('compute', C.c_int32),
        ('sample_v', C.c_int32), ('sample_h', C.c_int32),
        ('max_batch', C.c_int32),
        ('alpha', C.c_double), ('l2', C.c_double), ('dropout_keep', C.c_double), ('sparsity_cost', C.c_double),
        ('dbm_first', C.c_int32), ('dbm_last', C.c_int32),
        ('beta', C.c_double),
    ]


class TcOpArgs(C.Structure):
    _fields_ = [
        ('M', C.c_int32), ('N', C.c_int32), ('n_pairs', C.c_int32),
        ('K', C.c_int32 * 2), ('a_t', C.c_int32 * 2), ('b_t', C.c_int32 * 2), ('neg', C.c_int32 * 2),
        ('A', C.c_void_p * 2), ('B', C.c_void_p * 2),
        ('splits', C.c_int32), ('force_bn', C.c_int32), ('force_cluster', C.c_int32),
        ('acc_scale', C.c_float), ('bias_scale', C.c_float),
        ('bias', C.c_void_p), ('sigma', C.c_void_p), ('noise_sigma', C.c_void_p),
        ('act', C.c_int32), ('sample', C.c_int32),
        ('seed', C.c_uint64),
        ('site', C.c_uint32), ('t', C.c_uint32), ('tick', C.c_uint32), ('row0', C.c_uint32), ('tick_off', C.c_uint32),
        ('ais_kind', C.c_int32),
        ('ais_a', C.c_float), ('ais_b', C.c_float), ('ais_next', C.c_float), ('ais_lin', C.c_float),
        ('logw', C.c_void_p), ('logw_len', C.c_int32),
        ('mean_bf', C.c_void_p), ('mean_rows', C.c_int32), ('mean_ld', C.c_int32),
        ('state_bf', C.c_void_p), ('state_rows', C.c_int32), ('state_ld', C.c_int32),
        ('f32', C.c_void_p), ('f32_rows', C.c_int32), ('f32_ld', C.c_int32),
        ('mode', C.c_int32), ('bn', C.c_int32), ('cluster', C.c_int32), ('units', C.c_int32), ('ctas', C.c_int32),
    ]


class TcOpPlan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ('launch', 'mode', 'bn', 'm_groups', 'n_tiles', 'splits', 'pair_begin', 'pair_count',
                                         'follows_granules')]


_lib = None


def load_library(path=None):
    """dlopen libbm.so and declare the prototypes.  Raises if it is missing."""
    global _lib
    if _lib is not None and path is None:
        return _lib
    p = path or LIB_PATH
    if not os.path.isfile(p):
        raise RuntimeError("native library not found at '{0}': build it with "
                           "`python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)".format(p))
    lib = C.CDLL(p)
    vp, i32, u32, u64, i64, dbl, sz = C.c_void_p, C.c_int32, C.c_uint32, C.c_uint64, C.c_int64, C.c_double, C.c_size_t
    lib.bm_version.restype = C.c_char_p
    lib.bm_last_error.restype = C.c_char_p
    protos = {
        'bm_device_count': [C.POINTER(C.c_int)],
        'bm_ctx_create': [C.c_int, C.POINTER(vp)],
        'bm_ctx_sync': [vp], 'bm_ctx_timer_start': [vp], 'bm_ctx_timer_stop': [vp, C.POINTER(C.c_float)],
        'bm_ctx_flush_l2': [vp], 'bm_host_alloc': [C.POINTER(vp), sz], 'bm_host_free': [vp],
        'bm_host_pack_u8': [vp, i32, sz, vp, C.POINTER(i32)], 'bm_host_pack_bf16': [vp, sz, vp],
        'bm_ctx_launch_count': [vp, C.POINTER(u64)],
        'bm_ctx_profile_tc': [vp, C.c_int],
        'bm_ctx_profile_read': [vp, C.POINTER(dbl), C.POINTER(dbl), C.POINTER(u64)],
        'bm_comm_unique_id': [vp], 'bm_ctx_comm_init': [vp, vp, C.c_int, C.c_int],
        'bm_rbm_create': [vp, C.POINTER(RbmCfg), C.POINTER(vp)],
        'bm_rbm_set_param': [vp, C.c_char_p, vp, sz], 'bm_rbm_get_param': [vp, C.c_char_p, vp, sz],
        'bm_rbm_init_weights': [vp, dbl, u64],
        'bm_rbm_train_step': [vp, vp, i32, dbl, dbl, i32, u64, u32, u32, C.POINTER(dbl)],
        'bm_rbm_set_data': [vp, vp, i64],
        'bm_rbm_train_step_at': [vp, i64, i32, dbl, dbl, i32, u64, u32, u32, C.POINTER(dbl)],
        'bm_rbm_train_epoch': [vp, vp, i64, i32, dbl, dbl, i32, u64, u32, u32, i32, i64, vp],
        'bm_rbm_train_epoch_u8': [vp, vp, i64, i32, dbl, dbl, i32, u64, u32, u32, i32, i64, vp],
        'bm_rbm_train_epoch_bf16': [vp, vp, i64, i32, dbl, dbl, i32, u64, u32, u32, i32, i64, vp],
        'bm_rbm_transform': [vp, vp, i32, i32, u64, u32, vp],
        'bm_rbm_metrics': [vp, vp, i32, i32, u64, u32, u32, C.POINTER(dbl)],
        'bm_rbm_get_activation': [vp, C.c_char_p, vp, sz],
        'bm_debug_tc_gemm': [vp, i32, i32, i32, vp, i32, vp, i32, i32, vp, vp, i32, i32, i32, i32, vp],
        'bm_debug_tc_op': [vp, C.POINTER(TcOpArgs)],
        'bm_rbm_debug_tc_plan': [vp, C.POINTER(TcOpPlan), i32, C.POINTER(i32)],
        'bm_dbm_create': [vp, C.POINTER(DbmCfg), C.POINTER(vp)],
        'bm_dbm_set_param': [vp, C.c_char_p, vp, sz], 'bm_dbm_get_param': [vp, C.c_char_p, vp, sz],
        'bm_dbm_init_particles': [vp, u64],
        'bm_dbm_train_step': [vp, vp, i32, dbl, dbl, i32, u64, u32, i32, C.POINTER(dbl)],
        'bm_dbm_val_metrics': [vp, vp, i32, i32, u64, u32, C.POINTER(dbl)],
        'bm_dbm_transform': [vp, vp, i32, vp], 'bm_dbm_reconstruct': [vp, vp, i32, vp],
        'bm_dbm_log_proba': [vp, vp, i32, vp], 'bm_dbm_sample_v': [vp, i32, u64, u32, vp],
        'bm_dbm_ais': [vp, i32, i32, i32, u64, vp],
        'bm_dbm_ais_rows': [vp, i32, i32, i32, u64, u32, vp],
        'bm_dbm_ais_base': [vp, i32, i32, i32, u64, vp, vp],
        'bm_dbm_ais_base_rows': [vp, i32, i32, i32, u64, u32, vp, vp],
        'bm_dbm_pt_counts': [vp, vp, vp],
        'bm_dbm_train_step_labeled': [vp, vp, vp, i32, dbl, dbl, i32, u64, u32, i32, C.POINTER(dbl)],
        'bm_dbm_predict_proba': [vp, vp, i32, vp],
        'bm_dbm_fill': [vp, vp, vp, vp, i32, u32, i32, u64, u32, vp],
        'bm_dbm_debug_last_fill': [vp, C.c_char_p, vp, sz],
        'bm_dbm_debug_last_sample_v': [vp, C.c_char_p, vp, sz],
        'bm_dbm_exact': [vp, vp, i32, vp, vp], 'bm_dbm_debug_exact_chunk': [vp, i32],
        'bm_dbm_ais_clamped': [vp, vp, i32, u32, i32, i32, i32, u64, vp],
        'bm_debug_dbm_multinomial_rows': [vp, vp, i32, i32, dbl, i32, u64, u32, u32, u32, vp, vp, vp, vp],
        'bm_crbm_create': [vp, C.POINTER(CrbmCfg), C.POINTER(vp)],
        'bm_crbm_set_param': [vp, C.c_char_p, vp, sz], 'bm_crbm_get_param': [vp, C.c_char_p, vp, sz],
        'bm_crbm_init_weights': [vp, dbl, u64, u64],
        'bm_crbm_train_step': [vp, vp, vp, i32, dbl, dbl, i32, u64, u32, i32, C.POINTER(dbl)],
        'bm_crbm_predict_proba': [vp, vp, i32, vp], 'bm_crbm_transform': [vp, vp, i32, vp],
        'bm_crbm_debug_last_step': [vp, C.c_char_p, vp, sz],
        'bm_rbm_group_create': [vp, vp, i32, C.POINTER(vp)],
    }
    group_epoch = [vp, vp, i64, i32, vp, vp, i32, vp, vp, vp, vp, vp, vp]
    for name in ('bm_rbm_group_train_epoch', 'bm_rbm_group_train_epoch_u8', 'bm_rbm_group_train_epoch_bf16'):
        protos[name] = group_epoch
    for name, argtypes in protos.items():
        fn = getattr(lib, name)
        fn.argtypes = argtypes
        fn.restype = C.c_int
    lib.bm_ctx_destroy.argtypes = [vp]
    lib.bm_ctx_destroy.restype = None
    lib.bm_rbm_destroy.argtypes = [vp]
    lib.bm_rbm_destroy.restype = None
    lib.bm_dbm_destroy.argtypes = [vp]
    lib.bm_dbm_destroy.restype = None
    lib.bm_crbm_destroy.argtypes = [vp]
    lib.bm_crbm_destroy.restype = None
    lib.bm_rbm_group_destroy.argtypes = [vp]
    lib.bm_rbm_group_destroy.restype = None
    if path is None:
        _lib = lib
    return lib


def check(rc):
    if rc != 0:
        raise RuntimeError('libbm: ' + load_library().bm_last_error().decode('utf-8', 'replace'))


def device_count():
    n = C.c_int(0)
    check(load_library().bm_device_count(C.byref(n)))
    return n.value


class Context(object):
    """One GPU + compute stream (+ optional NCCL communicator)."""
    _default = {}

    def __init__(self, device=None):
        lib = load_library()
        if device is None:
            device = int(os.environ.get('LOCAL_RANK', os.environ.get('BM_DEVICE', '0')))
        self.device = device
        h = C.c_void_p()
        check(lib.bm_ctx_create(device, C.byref(h)))
        self.handle = h
        self.rank, self.nranks = 0, 1

    @classmethod
    def default(cls, device=None):
        key = device
        if key not in cls._default:
            cls._default[key] = cls(device)
        return cls._default[key]

    def sync(self):
        check(load_library().bm_ctx_sync(self.handle))

    def timer_start(self):
        check(load_library().bm_ctx_timer_start(self.handle))

    def timer_stop(self):
        ms = C.c_float(0)
        check(load_library().bm_ctx_timer_stop(self.handle, C.byref(ms)))
        return ms.value

    def flush_l2(self):
        check(load_library().bm_ctx_flush_l2(self.handle))

    def launch_count(self):
        n = C.c_uint64(0)
        check(load_library().bm_ctx_launch_count(self.handle, C.byref(n)))
        return n.value

    def profile_tc(self, enable):
        check(load_library().bm_ctx_profile_tc(self.handle, int(bool(enable))))

    def profile_read(self):
        """(algorithmic FLOPs, device ms, launches) of the tensor-core kernel since profiling was enabled."""
        f, ms, n = C.c_double(0), C.c_double(0), C.c_uint64(0)
        check(load_library().bm_ctx_profile_read(self.handle, C.byref(f), C.byref(ms), C.byref(n)))
        return f.value, ms.value, n.value

    def comm_init(self, unique_id, rank, nranks):
        buf = C.create_string_buffer(bytes(unique_id), 128)
        check(load_library().bm_ctx_comm_init(self.handle, buf, rank, nranks))
        self.rank, self.nranks = rank, nranks

    @staticmethod
    def comm_unique_id():
        buf = C.create_string_buffer(128)
        check(load_library().bm_comm_unique_id(buf))
        return buf.raw


# Page-locking is expensive (about 0.3 ms per MB): blocks released by `pinned_free` are kept in a small per-process pool and
# handed out again (what torch's caching host allocator does), so that the second `fit()` of a pipeline -- RBM #2 after RBM #1,
# the DBM after both -- or the next epoch's staging does not pay for it again.  `pinned_pool_clear()` returns them to the system.
_PINNED_POOL = {}            # bytes -> [addresses]
_PINNED_POOL_MAX = 2 << 30
_pinned_sizes = {}           # address -> bytes


def pinned_empty(shape, dtype=np.float32):
    """numpy array over page-locked host memory (for the per-batch feed path)."""
    n = max(1, int(np.prod(shape)) * np.dtype(dtype).itemsize)
    free = _PINNED_POOL.get(n)
    if free:
        addr = free.pop()
    else:
        p = C.c_void_p()
        check(load_library().bm_host_alloc(C.byref(p), n))
        addr = p.value
    _pinned_sizes[addr] = n
    buf = (C.c_char * n).from_address(addr)
    arr = np.frombuffer(buf, dtype=dtype, count=int(np.prod(shape))).reshape(shape)
    return arr


def pinned_free(arr):
    """Release an array made by `pinned_empty` / `pinned_copy` (the array must not be used afterwards)."""
    addr = np.asarray(arr).ctypes.data
    n = _pinned_sizes.pop(addr, None)
    if n is not None and sum(k * len(v) for k, v in _PINNED_POOL.items()) + n <= _PINNED_POOL_MAX:
        _PINNED_POOL.setdefault(n, []).append(addr)
        return
    check(load_library().bm_host_free(C.c_void_p(addr)))


def pinned_pool_clear():
    for n, addrs in list(_PINNED_POOL.items()):
        while addrs:
            check(load_library().bm_host_free(C.c_void_p(addrs.pop())))
    _PINNED_POOL.clear()


def pinned_copy(X):
    """Page-locked copy of a host array: lets `train_epoch` overlap the batch uploads with compute."""
    P = pinned_empty(X.shape, X.dtype)
    P[...] = X
    return P


def as_bytes(X, out=None):
    """X (float32 / float64) as uint8 if that is lossless (all values integers in 0..255), else None.  One multi-threaded
    native pass (bm_host_pack_u8); `out`: optional destination (e.g. page-locked memory) of X's shape."""
    if X.size == 0:
        return None
    if X.dtype not in (np.float32, np.float64) or not X.flags['C_CONTIGUOUS']:
        lo, hi = float(X.min()), float(X.max())
        if not (lo >= 0.0 and hi <= 255.0):          # also false for NaN
            return None
        Xb = X.astype(np.uint8)
        return Xb if np.array_equal(Xb, X) else None
    Xb = out if out is not None else np.empty(X.shape, dtype=np.uint8)
    exact = C.c_int32(0)
    check(load_library().bm_host_pack_u8(X.ctypes.data, DTYPES[X.dtype.name], X.size, Xb.ctypes.data, C.byref(exact)))
    return Xb if exact.value else None


class Bf16Array(np.ndarray):
    """uint16 array whose elements are bfloat16 bit patterns (a real-valued training set packed for
    bm_rbm_train_epoch_bf16).  `widen()` gives the float32 values back (exactly the rounded ones)."""
    def widen(self):
        return (np.asarray(self).astype(np.uint32) << 16).view(np.float32)


def as_bf16(X, out=None):
    """float32 X rounded to bfloat16 (round to nearest even, as the engine's own conversion), as a Bf16Array."""
    X = np.ascontiguousarray(X, dtype=np.float32)
    P = out if out is not None else np.empty(X.shape, dtype=np.uint16)
    check(load_library().bm_host_pack_bf16(X.ctypes.data, X.size, P.ctypes.data))
    return P.view(Bf16Array)


def debug_tc_gemm(A, B, a_t=False, b_t=False, A2=None, B2=None, neg2=False, splits=1, ctx=None,
                  force_bn=0, force_cluster=0):
    """Raw tensor-core GEMM (test hook): C = A' B'^T (+/- A2' B2'^T) with the operands stored as
    given: A is [M,K] (or [K,M] if a_t), B is [N,K] (or [K,N] if b_t)."""
    ctx = ctx or Context.default()
    A = np.ascontiguousarray(A, dtype=np.float32)
    B = np.ascontiguousarray(B, dtype=np.float32)
    M, K = (A.shape[1], A.shape[0]) if a_t else A.shape
    N = B.shape[1] if b_t else B.shape[0]
    K2 = 0
    p2a = p2b = None
    if A2 is not None:
        A2 = np.ascontiguousarray(A2, dtype=np.float32)
        B2 = np.ascontiguousarray(B2, dtype=np.float32)
        K2 = A2.shape[0] if a_t else A2.shape[1]
        p2a, p2b = A2.ctypes.data, B2.ctypes.data
    Cout = np.empty((M, N), dtype=np.float32)
    check(load_library().bm_debug_tc_gemm(ctx.handle, M, N, K, A.ctypes.data, int(a_t), B.ctypes.data, int(b_t),
                                          K2, p2a, p2b, int(neg2), int(splits), int(force_bn), int(force_cluster),
                                          Cout.ctypes.data))
    return Cout


# epilogue modes of the tensor-core kernel (csrc/bm_tc.cu), as debug_tc_op reports them
TC_MODES = ('GENERIC', 'SIG_BERN_MEAN_STATE', 'SIG_BERN_STATE', 'SIG_MEAN', 'RAW_F32', 'AIS_UNITS', 'AIS_STATE', 'AIS_UNITS_S',
            'AIS_UNITS_G')
TC_ACTS = {'linear': 0, 'sigmoid': 1, 'softplus': 2}
TC_SAMPLES = {None: 0, 'bernoulli': 1, 'gaussian': 2}
# what debug_tc_op fills its output buffers with before the launch: NaN bit patterns no epilogue produces
BF16_SENTINEL = 0xFFA5
F32_SENTINEL = 0xFFC0DEAD
LOGW_SENTINEL = -1234.5


def _round8(n):
    return (n + 7) // 8 * 8


def debug_tc_op(pairs, outputs=('f32',), splits=1, force_bn=0, force_cluster=0, acc_scale=1.0, bias_scale=1.0, bias=None,
                sigma=None, noise_sigma=None, act='linear', sample=None, seed=0, site=0, t=0, tick=0, row0=0, tick_off=0,
                ais_kind=0, ais_a=0.0, ais_b=0.0, ais_next=0.0, ais_lin=0.0, logw=None, mean_ld=None, state_ld=None,
                f32_ld=None, guard_rows=2, ctx=None, ais_base=None):
    """One fused tensor-core op (test hook, bm_debug_tc_op): C = sum over `pairs` of (+/-) A B^T, then the epilogue.

    pairs: 1 or 2 tuples (A, B, a_t, b_t, neg); A is [M,K] (a_t: [K,M]), B is [N,K] (b_t: [K,N]), rounded to bf16 here.
    outputs: any of 'mean', 'state' (bf16) and 'f32'.  Every output buffer has `guard_rows` rows past M and columns past
    round_up(N, 8), is filled with the sentinel bit pattern before the launch and is returned whole: 'mean' / 'state' as
    uint16 bf16 bit patterns [M + guard_rows, ld], 'f32' as float32 [splits, M + guard_rows, ld].  logw (float64 [M]) is
    added to by the AIS epilogues and returned with one guard entry (LOGW_SENTINEL) past M.  ais_base ([N] or None): the AIS
    ops' base bias a, added to every sigmoid argument after the beta scaling (it travels in the noise_sigma slot, which AIS ops
    never use).  'plan' describes the launch."""
    ctx = ctx or Context.default()
    if ais_base is not None:
        if not ais_kind or noise_sigma is not None:
            raise ValueError('ais_base belongs to an AIS op without noise_sigma')
        noise_sigma = ais_base
    if not 1 <= len(pairs) <= 2:
        raise ValueError('one or two operand pairs')
    a = TcOpArgs()
    keep = []
    for p, (A, B, a_t, b_t, neg) in enumerate(pairs):
        A, B = np.asarray(A, dtype=np.float32), np.asarray(B, dtype=np.float32)
        M, K = (A.shape[1], A.shape[0]) if a_t else A.shape
        N = B.shape[1] if b_t else B.shape[0]
        if p == 0:
            a.M, a.N = M, N
        elif (M, N) != (a.M, a.N):
            raise ValueError('the pairs disagree about the output shape')
        if (B.shape[0] if b_t else B.shape[1]) != K:
            raise ValueError('A and B of pair {0} disagree about K'.format(p))
        Ab, Bb = as_bf16(A), as_bf16(B)
        keep += [Ab, Bb]
        a.K[p], a.a_t[p], a.b_t[p], a.neg[p] = K, int(bool(a_t)), int(bool(b_t)), int(bool(neg))
        a.A[p], a.B[p] = Ab.ctypes.data, Bb.ctypes.data
    a.n_pairs = len(pairs)
    M, N = a.M, a.N
    a.splits, a.force_bn, a.force_cluster = int(splits), int(force_bn), int(force_cluster)
    a.acc_scale, a.bias_scale = float(acc_scale), float(bias_scale)
    for name, v in (('bias', bias), ('sigma', sigma), ('noise_sigma', noise_sigma)):
        if v is not None:
            v = np.ascontiguousarray(v, dtype=np.float32).reshape(N)
            keep.append(v)
            setattr(a, name, v.ctypes.data)
    a.act, a.sample = TC_ACTS[act], TC_SAMPLES[sample]
    a.seed, a.site, a.t, a.tick, a.row0, a.tick_off = int(seed) & (2 ** 64 - 1), int(site), int(t), int(tick), int(row0), int(tick_off)
    a.ais_kind, a.ais_a, a.ais_b, a.ais_next, a.ais_lin = int(ais_kind), float(ais_a), float(ais_b), float(ais_next), float(ais_lin)
    out = {}
    rows = M + int(guard_rows)
    if logw is not None:
        lw = np.empty(M + 1, dtype=np.float64)
        lw[:M], lw[M] = logw, LOGW_SENTINEL
        out['logw'] = lw
        a.logw, a.logw_len = lw.ctypes.data, M + 1
    for name in outputs:
        if name in ('mean', 'state'):
            ld = int((mean_ld if name == 'mean' else state_ld) or _round8(N) + 8)
            buf = np.full((rows, ld), BF16_SENTINEL, dtype=np.uint16)
            setattr(a, name + '_bf', buf.ctypes.data)
            setattr(a, name + '_rows', rows)
            setattr(a, name + '_ld', ld)
        elif name == 'f32':
            ld = int(f32_ld or _round8(N) + 2)
            buf = np.full((max(1, int(splits)), rows, ld), F32_SENTINEL, dtype=np.uint32).view(np.float32)
            a.f32, a.f32_rows, a.f32_ld = buf.ctypes.data, rows, ld
        else:
            raise ValueError('unknown output ' + repr(name))
        out[name] = buf
    check(load_library().bm_debug_tc_op(ctx.handle, C.byref(a)))
    out['plan'] = dict(mode=TC_MODES[a.mode], bn=a.bn, cluster=a.cluster, units=a.units, ctas=a.ctas)
    return out


def debug_dbm_multinomial_rows(pre, n_samples, n_draws, seed, site, t, tick, ctx=None):
    """The tensor-core DBM engine's multinomial row kernel on fp32 pre-activations (test hook,
    bm_debug_dbm_multinomial_rows).  Returns (bf16 bit patterns, fp32 output, reference means, reference counts or None):
    the last two from the CUDA-core engine's softmax_rows + multinomial_rows kernels on the same input."""
    ctx = ctx or Context.default()
    pre = np.ascontiguousarray(pre, dtype=np.float32)
    rows, cols = pre.shape
    out_bf = np.empty((rows, cols), np.uint16)
    out_f32, ref_means = np.empty((rows, cols), np.float32), np.empty((rows, cols), np.float32)
    ref_counts = np.empty((rows, cols), np.float32) if n_draws > 0 else None
    check(load_library().bm_debug_dbm_multinomial_rows(
        ctx.handle, pre.ctypes.data, rows, cols, float(n_samples), int(n_draws), int(seed), int(site), int(t), int(tick),
        out_bf.ctypes.data, out_f32.ctypes.data, ref_means.ctypes.data, None if ref_counts is None else ref_counts.ctypes.data))
    return out_bf, out_f32, ref_means, ref_counts


def _mask(names):
    m = 0
    for n in names:
        m |= METRIC_BITS[n]
    return m


class CudaRBM(object):
    """Engine object for ``BaseRBM``: a ``bm_rbm`` handle."""

    def __init__(self, cfg, ctx=None):
        self._lib = load_library()
        self.ctx = ctx or Context.default()
        self.cfg = dict(cfg)
        self.V, self.H = int(cfg['n_visible']), int(cfg['n_hidden'])
        self.dt = np.dtype(cfg.get('dtype', 'float32'))
        c = RbmCfg()
        c.n_visible, c.n_hidden = self.V, self.H
        c.v_kind = UNIT_KINDS[cfg.get('v_kind', 'bernoulli')]
        c.h_kind = UNIT_KINDS[cfg.get('h_kind', 'bernoulli')]
        c.dtype = DTYPES[self.dt.name]
        # float32 models run on the tensor cores (bf16 operands, fp32 accumulate) unless told
        # otherwise; float64 models always use the storage-precision CUDA-core path
        compute = 'fp32'
        if self.dt == np.float32:
            compute = cfg.get('compute') or os.environ.get('BM_COMPUTE') or 'bf16'
        self.compute = compute
        c.compute = COMPUTE[compute]
        c.sample_v, c.sample_h = int(cfg.get('sample_v', False)), int(cfg.get('sample_h', True))
        c.max_batch = int(cfg.get('max_batch', 0))
        c.l2 = float(cfg.get('l2', 0.))
        keep = cfg.get('dropout', None)
        c.dropout_keep = -1.0 if keep is None else float(keep)
        c.sparsity_target = float(cfg.get('sparsity_target', 0.1))
        c.sparsity_cost = float(cfg.get('sparsity_cost', 0.))
        c.sparsity_damping = float(cfg.get('sparsity_damping', 0.9))
        c.propup_mult = 2.0 if cfg.get('dbm_first', False) else 1.0
        c.propdown_mult = 2.0 if cfg.get('dbm_last', False) else 1.0
        c.v_n_samples = float(cfg.get('v_n_samples', 100))
        c.h_n_samples = float(cfg.get('h_n_samples', 100))
        self._sigma = None
        if cfg.get('sigma', None) is not None:
            self._sigma = np.ascontiguousarray(
                np.broadcast_to(np.asarray(cfg['sigma'], dtype=np.float64), (self.V,)))
            c.sigma = self._sigma.ctypes.data_as(C.POINTER(C.c_double))
        h = C.c_void_p()
        check(self._lib.bm_rbm_create(self.ctx.handle, C.byref(c), C.byref(h)))
        self.handle = h
        self._names = ['W', 'vb', 'hb', 'dW', 'dvb', 'dhb', 'q_means'] + (['sigma'] if self._sigma is not None else [])
        self._shapes = {'W': (self.V, self.H), 'dW': (self.V, self.H), 'vb': (self.V,), 'dvb': (self.V,),
                        'hb': (self.H,), 'dhb': (self.H,), 'q_means': (self.H,), 'sigma': (self.V,)}
        self._metrics_buf = (C.c_double * 4)()

    # ---- variables ---------------------------------------------------------------
    def set_params(self, d):
        for k, v in d.items():
            if k == 'sigma':
                continue                      # fixed at construction (rbm/rbm.py:101-107)
            a = np.ascontiguousarray(v, dtype=self.dt).reshape(self._shapes[k])
            check(self._lib.bm_rbm_set_param(self.handle, k.encode(), a.ctypes.data, a.nbytes))

    def get_params(self, names=None):
        out = {}
        for k in (names or self._names):
            a = np.empty(self._shapes[k], dtype=self.dt)
            check(self._lib.bm_rbm_get_param(self.handle, k.encode(), a.ctypes.data, a.nbytes))
            out[k] = a
        return out

    def init_normal_W(self, stddev, op_seed):
        check(self._lib.bm_rbm_init_weights(self.handle, float(stddev), int(op_seed) & (2 ** 64 - 1)))

    # ---- compute -------------------------------------------------------------------
    def _batch(self, X):
        if isinstance(X, Bf16Array):
            X = X.widen()
        X = np.ascontiguousarray(X, dtype=self.dt)
        if X.ndim != 2 or X.shape[1] != self.V:
            raise ValueError('batch has shape {0}, expected (rows, {1})'.format(X.shape, self.V))
        return X

    def _collect(self, names):
        return {n: float(self._metrics_buf[METRIC_SLOTS[n]]) for n in names}

    def train_step(self, X, lr, momentum, k, seed, tick, metrics=()):
        X = self._batch(X)
        check(self._lib.bm_rbm_train_step(self.handle, X.ctypes.data, X.shape[0], lr, momentum, int(k),
                                          int(seed), int(tick), _mask(metrics), self._metrics_buf))
        return self._collect(metrics) if metrics else None

    def train_epoch(self, X, batch, lr, momentum, k, seed, tick0, metrics=(), every=0, iter0=0):
        """One pass over the host dataset X in mini-batches (uploads overlap compute).  Returns
        {metric: [value of every reporting batch]}; batch i uses tick0 + i, exactly like
        train_step(X[i*batch:(i+1)*batch], ..., tick=tick0 + i)."""
        byte_valued = getattr(X, 'dtype', None) == np.uint8 and not isinstance(X, Bf16Array)   # see as_bytes(): exact, 4x less traffic
        packed_bf16 = isinstance(X, Bf16Array)                  # see pin(): real-valued data for the bf16 engine, 2x less traffic
        if byte_valued or packed_bf16:
            X = np.ascontiguousarray(X)
            if X.ndim != 2 or X.shape[1] != self.V:
                raise ValueError('batch has shape {0}, expected (rows, {1})'.format(X.shape, self.V))
        else:
            X = self._batch(X)
        nb = (X.shape[0] + batch - 1) // batch
        out = np.zeros((nb, 4), dtype=np.float64)
        fn = (self._lib.bm_rbm_train_epoch_u8 if byte_valued else
              self._lib.bm_rbm_train_epoch_bf16 if packed_bf16 else self._lib.bm_rbm_train_epoch)
        check(fn(self.handle, X.ctypes.data, X.shape[0], int(batch), lr, momentum, int(k),
                 int(seed), int(tick0), _mask(metrics), int(every), int(iter0), out.ctypes.data))
        rep = [i for i in range(nb) if every and (iter0 + i + 1) % every == 0]
        return {m: [float(out[i, METRIC_SLOTS[m]]) for i in rep] for m in metrics}

    def pin(self, X):
        """Page-locked copy of the training set for `train_epoch`.  Data whose every value is an integer in
        0..255 (binarised MNIST: {0, 1}) is kept as one byte per unit: the engine widens it exactly on the
        device, so results do not change and each epoch moves a quarter of the bytes over PCIe."""
        X = self._batch(X)
        if X.size == 0:
            return pinned_copy(X)
        P = pinned_empty(X.shape, np.uint8)
        if as_bytes(X, out=P) is not None:
            return P
        pinned_free(P)
        if self.feeds_bf16():
            return as_bf16(X, out=pinned_empty(X.shape, np.uint16))
        return pinned_copy(X)

    def feeds_bf16(self):
        """Whether real-valued training data goes to this engine as bfloat16: the bf16 engine rounds its input to bfloat16
        before the first GEMM, so feeding the rounded values is bit-identical and halves the copy (not with dropout / sigma
        scaling, which act on the fp32 input first)."""
        return (self.compute == 'bf16' and self.dt == np.float32 and self.cfg.get('v_kind', 'bernoulli') == 'bernoulli' and
                self.cfg.get('h_kind', 'bernoulli') == 'bernoulli' and self.cfg.get('dropout') is None)

    def unpin(self, P):
        pinned_free(np.asarray(P))

    def set_data(self, X):
        X = self._batch(X)
        check(self._lib.bm_rbm_set_data(self.handle, X.ctypes.data, X.shape[0]))

    def train_step_at(self, first_row, rows, lr, momentum, k, seed, tick, metrics=()):
        check(self._lib.bm_rbm_train_step_at(self.handle, int(first_row), int(rows), lr, momentum, int(k),
                                             int(seed), int(tick), _mask(metrics), self._metrics_buf))
        return self._collect(metrics) if metrics else None

    def transform(self, X, k, seed, tick):
        X = self._batch(X)
        Hout = np.empty((X.shape[0], self.H), dtype=self.dt)
        check(self._lib.bm_rbm_transform(self.handle, X.ctypes.data, X.shape[0], int(k), int(seed), int(tick),
                                         Hout.ctypes.data))
        return Hout

    def metrics(self, X, k, seed, tick, names):
        X = self._batch(X)
        check(self._lib.bm_rbm_metrics(self.handle, X.ctypes.data, X.shape[0], int(k), int(seed), int(tick),
                                       _mask(names), self._metrics_buf))
        return self._collect(names)

    def get_activation(self, name, rows):
        n = self.V if name in ('X', 'v_means', 'v_states') else self.H
        dt = np.float32 if self.compute == 'bf16' else self.dt
        a = np.empty((rows, n), dtype=dt)
        check(self._lib.bm_rbm_get_activation(self.handle, name.encode(), a.ctypes.data, a.nbytes))
        return a

    def debug_tc_plan(self):
        """(test hook, bm_rbm_debug_tc_plan) the ops of the last tensor-core program, in program order across its launches:
        one dict per op with launch, mode (a TC_MODES name), bn, m_groups, n_tiles, splits, units, pair_begin, pair_count and
        follows_granules (the op waits for its producer's 64-column granules one by one)."""
        n = C.c_int32(0)
        check(self._lib.bm_rbm_debug_tc_plan(self.handle, None, 0, C.byref(n)))
        recs = (TcOpPlan * max(1, n.value))()
        check(self._lib.bm_rbm_debug_tc_plan(self.handle, recs, n.value, C.byref(n)))
        out = []
        for r in recs[:n.value]:
            d = {f: int(getattr(r, f)) for f, _ in TcOpPlan._fields_}
            d['mode'] = TC_MODES[d['mode']]
            d['follows_granules'] = bool(d['follows_granules'])
            d['units'] = d['m_groups'] * d['n_tiles'] * d['splits']
            out.append(d)
        return out

    def close(self):
        if getattr(self, 'handle', None):
            self._lib.bm_rbm_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CudaRBMGroup(object):
    """Engine object for ``fit_many``: a ``bm_rbm_group`` handle over CudaRBM engines of one shape, which stay usable on
    their own.  Refused engine options raise NotImplementedError."""

    def __init__(self, engines):
        self._lib = load_library()
        self.engines = list(engines)
        n = len(self.engines)
        handles = (C.c_void_p * n)(*[e.handle.value for e in self.engines])
        h = C.c_void_p()
        self._check(self._lib.bm_rbm_group_create(self.engines[0].ctx.handle, handles, n, C.byref(h)))
        self.handle = h

    def _check(self, rc):
        if rc == -5:                                        # BM_EUNSUPPORTED
            raise NotImplementedError(self._lib.bm_last_error().decode('utf-8', 'replace'))
        check(rc)

    def pin(self, Xs):
        """The members' training sets [n, rows, n_visible] in page-locked memory, in the format each member's own `pin` would
        feed with the same values: bytes when every value is an integer in 0..255, bfloat16 for engines that round their input
        to it anyway, float32 otherwise."""
        X = np.ascontiguousarray(np.stack([e._batch(x) for e, x in zip(self.engines, Xs)]))
        P = pinned_empty(X.shape, np.uint8)
        if as_bytes(X, out=P) is not None:
            return P
        pinned_free(P)
        if all(e.feeds_bf16() for e in self.engines):
            return as_bf16(X, out=pinned_empty(X.shape, np.uint16))
        return pinned_copy(X)

    def unpin(self, P):
        pinned_free(np.asarray(P))

    def train_epoch(self, X, batch, lr, momentum, k, seed, tick0, metrics, every, iter0):
        """One epoch of every member: member m trains on X[m] exactly as engines[m].train_epoch(X[m], batch, lr[m], ...) would.
        Per-member lists: lr, momentum, seed, tick0, metrics (names), every, iter0.  Returns one {metric: [values]} per member."""
        n = len(self.engines)
        byte_valued = X.dtype == np.uint8 and not isinstance(X, Bf16Array)
        fn = (self._lib.bm_rbm_group_train_epoch_u8 if byte_valued else
              self._lib.bm_rbm_group_train_epoch_bf16 if isinstance(X, Bf16Array) else self._lib.bm_rbm_group_train_epoch)
        if X.ndim != 3 or X.shape[0] != n or X.shape[2] != self.engines[0].V or not X.flags['C_CONTIGUOUS']:
            raise ValueError('training sets have shape {0}, expected ({1}, rows, {2})'.format(X.shape, n, self.engines[0].V))
        nb = (X.shape[1] + batch - 1) // batch
        out = np.zeros((n, nb, 4), dtype=np.float64)
        arr = lambda v, dt: np.ascontiguousarray(v, dtype=dt)
        lr, momentum = arr(lr, np.float64), arr(momentum, np.float64)
        seeds = arr([int(s) & (2 ** 64 - 1) for s in seed], np.uint64)
        ticks, masks = arr(tick0, np.uint32), arr([_mask(m) for m in metrics], np.uint32)
        every, iter0 = arr(every, np.int32), arr(iter0, np.int64)
        self._check(fn(self.handle, X.ctypes.data, X.shape[1], int(batch), lr.ctypes.data, momentum.ctypes.data, int(k),
                       seeds.ctypes.data, ticks.ctypes.data, masks.ctypes.data, every.ctypes.data, iter0.ctypes.data,
                       out.ctypes.data))
        res = []
        for g in range(n):
            rep = [i for i in range(nb) if every[g] and (iter0[g] + i + 1) % every[g] == 0]
            res.append({m: [float(out[g, i, METRIC_SLOTS[m]]) for i in rep] for m in metrics[g]})
        return res

    def close(self):
        if getattr(self, 'handle', None):
            self._lib.bm_rbm_group_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _sfx(i):
    return '' if i == 0 else '_{0}'.format(i)


class CudaDBM(object):
    """Engine object for ``DBM``: a ``bm_dbm`` handle."""

    def __init__(self, cfg, ctx=None):
        self._lib = load_library()
        self.ctx = ctx or Context.default()
        self.cfg = dict(cfg)
        self.V = int(cfg['n_visible'])
        self.Hs = [int(h) for h in cfg['n_hiddens']]
        self.L = len(self.Hs)
        self.M, self.B = int(cfg['n_particles']), int(cfg['batch_size'])
        self.dt = np.dtype(cfg.get('dtype', 'float32'))
        i32arr = lambda xs: (C.c_int32 * len(xs))(*[int(x) for x in xs])
        dblarr = lambda xs: (C.c_double * len(xs))(*[float(x) for x in xs])
        c = DbmCfg()
        c.n_layers, c.n_visible = self.L, self.V
        self._keep = [i32arr(self.Hs), i32arr([UNIT_KINDS[k] for k in cfg.get('h_kinds', ['bernoulli'] * self.L)]),
                      dblarr(cfg.get('h_n_samples', [100.] * self.L)), i32arr(cfg.get('sample_h', [True] * self.L)),
                      dblarr(cfg.get('sparsity_target', [0.1] * self.L)), dblarr(cfg.get('sparsity_cost', [0.] * self.L))]
        c.n_hiddens, c.h_kinds, c.h_n_samples, c.sample_h, c.sparsity_target, c.sparsity_cost = self._keep
        c.v_kind = UNIT_KINDS[cfg.get('v_kind', 'bernoulli')]
        c.dtype = DTYPES[self.dt.name]
        # float32 models with Bernoulli hidden layers (binary or Gaussian visibles) run on the tensor-core engine
        # (csrc/bm_dbm_tc.cuh: bf16 operands, fp32 accumulation) -- the same rule as DbmTC::supports(); compute='fp32'
        # (or BM_DBM_COMPUTE / BM_COMPUTE = fp32) selects the storage-precision CUDA-core engine, which every other
        # model uses anyway.  Multinomial hidden layers run on the tensor-core engine as well, but only when the caller asks
        # for it by name: compute='bf16' or BM_DBM_COMPUTE=bf16 (BM_COMPUTE alone leaves them on the fp32 engine).
        compute = 'fp32'
        h_kinds = cfg.get('h_kinds', ['bernoulli'] * self.L)
        tc_ok = (self.dt == np.float32 and cfg.get('v_kind', 'bernoulli') in ('bernoulli', 'gaussian') and
                 all(k in ('bernoulli', 'multinomial') for k in h_kinds))
        if tc_ok and all(k == 'bernoulli' for k in h_kinds):
            compute = cfg.get('compute') or os.environ.get('BM_DBM_COMPUTE') or os.environ.get('BM_COMPUTE') or 'bf16'
        elif tc_ok:
            compute = cfg.get('compute') or os.environ.get('BM_DBM_COMPUTE') or 'fp32'
        self.compute = compute
        c.compute = COMPUTE[compute]
        c.n_particles, c.batch_size = self.M, self.B
        c.max_mf_updates = int(cfg.get('max_mf_updates', 10))
        c.sample_v = int(cfg.get('sample_v', True))
        c.mf_tol = float(cfg.get('mf_tol', 1e-7))
        c.l2 = float(cfg.get('l2', 0.))
        mn = float(cfg.get('max_norm', np.inf))
        c.max_norm = mn if np.isfinite(mn) else 1e300
        c.sparsity_damping = float(cfg.get('sparsity_damping', 0.9))
        self._sigma = None
        if cfg.get('sigma', None) is not None:
            self._sigma = np.ascontiguousarray(np.broadcast_to(np.asarray(cfg['sigma'], dtype=np.float64), (self.V,)))
            c.sigma = self._sigma.ctypes.data_as(C.POINTER(C.c_double))
        # parallel tempering: the ladder of inverse temperatures (None: off).  The engine validates it; its refusals of the
        # option (messages starting 'parallel tempering') surface as NotImplementedError (BM_EUNSUPPORTED) or ValueError
        # (BM_EINVAL), every other failure of bm_dbm_create as RuntimeError, as without tempering
        betas = cfg.get('pt_betas', None)
        self.pt_betas = None if betas is None else np.ascontiguousarray(np.asarray(betas, dtype=np.float64).ravel())
        self.T = 1 if self.pt_betas is None else len(self.pt_betas)
        if self.pt_betas is not None:
            c.n_temps = len(self.pt_betas)
            c.betas = self.pt_betas.ctypes.data_as(C.POINTER(C.c_double))
        # classification DBM: a one-of-n_classes label layer above the last hidden layer (0: none; tensor-core engine only)
        self.C = int(cfg.get('n_classes', 0) or 0)
        c.n_classes = self.C
        if self.C:
            self.compute = cfg.get('compute') or 'bf16'
            c.compute = COMPUTE[self.compute]
        # centering: data-mean offsets and offset-centred gradients (tensor-core engine only, which it asks for unless the
        # caller names a compute mode); the variables v_offset, h_offset..., offsets_set
        self.centering = bool(cfg.get('centering', False))
        if self.centering:
            c.centering = 1
            c.offset_rate = float(cfg.get('offset_rate', 0.01))
            self.compute = cfg.get('compute') or 'bf16'
            c.compute = COMPUTE[self.compute]
        h = C.c_void_p()
        rc = self._lib.bm_dbm_create(self.ctx.handle, C.byref(c), C.byref(h))
        if rc in (-1, -5):
            err = self._lib.bm_last_error().decode('utf-8', 'replace')
            if err.startswith('parallel tempering') or err.startswith('classification DBM') or err.startswith('centering'):
                raise (NotImplementedError if rc == -5 else ValueError)('libbm: ' + err)
        check(rc)
        self.handle = h
        self._shapes = {'vb': (self.V,), 'dvb': (self.V,), 'v': (self.M, self.V)}
        sizes = [self.V] + self.Hs
        for i in range(self.L):
            s = _sfx(i)
            self._shapes.update({'W' + s: (sizes[i], sizes[i + 1]), 'dW' + s: (sizes[i], sizes[i + 1]),
                                 'hb' + s: (self.Hs[i],), 'dhb' + s: (self.Hs[i],), 'mu' + s: (self.B, self.Hs[i]),
                                 'q_means' + s: (self.Hs[i],), 'mu_means' + s: (self.Hs[i],), 'h' + s: (self.M, self.Hs[i])})
        if self.T > 1:                     # the tempered slots 1..T-1 of the particles
            self._shapes['v_pt'] = (self.T - 1, self.M, self.V)
            for i in range(self.L):
                self._shapes['h_pt' + _sfx(i)] = (self.T - 1, self.M, self.Hs[i])
        if self.centering:
            self._shapes.update({'v_offset': (self.V,), 'offsets_set': (1,)})
            for i in range(self.L):
                self._shapes['h_offset' + _sfx(i)] = (self.Hs[i],)
        if self.C:
            Cn, H = self.C, self.Hs[-1]
            self._shapes.update({'U': (Cn, H), 'dU': (Cn, H), 'yb': (Cn,), 'dyb': (Cn,), 'y': (self.M, Cn),
                                 'mu_y': (self.B, Cn)})
        self._out2 = (C.c_double * 2)()

    def pt_counts(self):
        """(accepted, proposed): int64 arrays of T-1 swap counts between slots m and m+1 since the engine was created."""
        acc, prop = np.zeros(self.T - 1, dtype=np.int64), np.zeros(self.T - 1, dtype=np.int64)
        check(self._lib.bm_dbm_pt_counts(self.handle, acc.ctypes.data, prop.ctypes.data))
        return acc, prop

    def set_params(self, d):
        for k, v in d.items():
            if k == 'sigma':
                continue
            a = np.ascontiguousarray(v, dtype=self.dt).reshape(self._shapes[k])
            check(self._lib.bm_dbm_set_param(self.handle, k.encode(), a.ctypes.data, a.nbytes))

    def get_params(self, names=None):
        out = {}
        for k in (names or list(self._shapes)):
            a = np.empty(self._shapes[k], dtype=self.dt)
            check(self._lib.bm_dbm_get_param(self.handle, k.encode(), a.ctypes.data, a.nbytes))
            out[k] = a
        return out

    def init_particles(self, seed):
        check(self._lib.bm_dbm_init_particles(self.handle, int(seed) & (2 ** 64 - 1)))

    def _batch(self, X):
        X = np.ascontiguousarray(X, dtype=self.dt)
        if X.ndim != 2 or X.shape[1] != self.V:
            raise ValueError('batch has shape {0}, expected (rows, {1})'.format(X.shape, self.V))
        return X

    def train_step(self, X, lr, momentum, k, seed, tick, metrics=(), labels=None):
        """``labels`` (classification DBMs): [rows] ints in [-1, n_classes), -1 for an unlabelled row."""
        X = self._batch(X)
        if labels is None:
            check(self._lib.bm_dbm_train_step(self.handle, X.ctypes.data, X.shape[0], lr, momentum, int(k), int(seed),
                                              int(tick), 1 if metrics else 0, self._out2))
        else:
            y = np.ascontiguousarray(labels, dtype=np.int32).reshape(-1)
            if y.shape[0] != X.shape[0]:
                raise ValueError('{0} labels for {1} rows'.format(y.shape[0], X.shape[0]))
            check(self._lib.bm_dbm_train_step_labeled(self.handle, X.ctypes.data, y.ctypes.data, X.shape[0], lr, momentum,
                                                      int(k), int(seed), int(tick), 1 if metrics else 0, self._out2))
        return {'msre': float(self._out2[0]), 'n_mf_updates': float(self._out2[1])} if metrics else None

    def predict_proba(self, X):
        """classification DBMs: softmax(yb + mu_L U^T) [rows, n_classes] (float32) after the E-step with y free"""
        X = self._batch(X)
        out = np.empty((X.shape[0], self.C), dtype=np.float32)
        check(self._lib.bm_dbm_predict_proba(self.handle, X.ctypes.data, X.shape[0], out.ctypes.data))
        return out

    def val_metrics(self, X, k, seed, tick):
        X = self._batch(X)
        check(self._lib.bm_dbm_val_metrics(self.handle, X.ctypes.data, X.shape[0], int(k), int(seed), int(tick), self._out2))
        return {'msre': float(self._out2[0]), 'n_mf_updates': float(self._out2[1])}

    def transform(self, X):
        X = self._batch(X)
        out = np.empty((X.shape[0], self.Hs[-1]), dtype=self.dt)
        check(self._lib.bm_dbm_transform(self.handle, X.ctypes.data, X.shape[0], out.ctypes.data))
        return out

    def reconstruct(self, X):
        X = self._batch(X)
        out = np.empty((X.shape[0], self.V), dtype=self.dt)
        check(self._lib.bm_dbm_reconstruct(self.handle, X.ctypes.data, X.shape[0], out.ctypes.data))
        return out

    def log_proba(self, X):
        X = self._batch(X)
        out = np.empty(X.shape[0], dtype=np.float64)
        check(self._lib.bm_dbm_log_proba(self.handle, X.ctypes.data, X.shape[0], out.ctypes.data))
        return out

    def sample_v(self, k, seed, tick):
        out = np.empty((self.M, self.V), dtype=self.dt)
        check(self._lib.bm_dbm_sample_v(self.handle, int(k), int(seed), int(tick), out.ctypes.data))
        return out

    def fill(self, X, mask, labels=None, row0=0, k=1, seed=0, tick=0):
        """Clamped Gibbs chains (DESIGN.md §5.9): the visible means of X's rows after ``k`` sweeps with the units where
        ``mask`` is 1 held at X; these are rows row0.. of the caller's call.  ``labels`` (classification DBMs): [rows] ints
        in [-1, n_classes), -1 leaving the label free.  Leaves every variable as it was."""
        X = self._batch(X)
        m = np.ascontiguousarray(mask, dtype=np.uint8)
        if m.shape != X.shape:
            raise ValueError('mask has shape {0}, expected {1}'.format(m.shape, X.shape))
        y, yp = None, None
        if labels is not None:
            y = np.ascontiguousarray(labels, dtype=np.int32).reshape(-1)
            if y.shape[0] != X.shape[0]:
                raise ValueError('{0} labels for {1} rows'.format(y.shape[0], X.shape[0]))
            yp = y.ctypes.data
        out = np.empty(X.shape, dtype=self.dt)
        check(self._lib.bm_dbm_fill(self.handle, X.ctypes.data, m.ctypes.data, yp, X.shape[0], int(row0), int(k), int(seed),
                                    int(tick), out.ctypes.data))
        return out

    def debug_last_fill(self, name, rows):
        """one chain state of the last ``fill`` (include/bm.h bm_dbm_debug_last_fill): float32 values widened from the bf16
        operands on the tensor-core engine, the model dtype on the CUDA-core engine"""
        base = name[:-5] if name.endswith('_prev') else name
        sizes = {'v': self.V, 'mean': self.V, 'y': self.C}
        sizes.update({'h' + _sfx(i): self.Hs[i] for i in range(self.L)})
        width = sizes[base]
        tc = self.compute == 'bf16' and self.dt == np.float32 and self._is_tc()
        a = np.empty((int(rows), width), dtype=np.uint16 if tc else self.dt)
        check(self._lib.bm_dbm_debug_last_fill(self.handle, name.encode(), a.ctypes.data, a.nbytes))
        return (a.astype(np.uint32) << 16).view(np.float32) if tc else a

    def debug_last_sample_v(self, name):
        """one sweep of the last ``sample_v``'s uncommitted half (include/bm.h bm_dbm_debug_last_sample_v): "v", "h", "h_1", ...
        for its last sweep, + "_prev" for the sweep before; [n_particles, n], float32 widened from bf16 on the tensor-core
        engine, the model dtype on the CUDA-core engine"""
        base = name[:-5] if name.endswith('_prev') else name
        sizes = {'v': self.V}
        sizes.update({'h' + _sfx(i): self.Hs[i] for i in range(self.L)})
        tc = self.compute == 'bf16' and self.dt == np.float32 and self._is_tc()
        a = np.empty((self.M, sizes[base]), dtype=np.uint16 if tc else self.dt)
        check(self._lib.bm_dbm_debug_last_sample_v(self.handle, name.encode(), a.ctypes.data, a.nbytes))
        return (a.astype(np.uint32) << 16).view(np.float32) if tc else a

    def _is_tc(self):
        """the engine bm_dbm_create picked is the tensor-core one (the rule of DbmTC::supports)"""
        h_kinds = self.cfg.get('h_kinds', ['bernoulli'] * self.L)
        return (self.cfg.get('v_kind', 'bernoulli') in ('bernoulli', 'gaussian') and
                all(k in ('bernoulli', 'multinomial') for k in h_kinds))

    def ais(self, n_runs, n_betas, k, seed, first_run=None, base=None):
        """log Z estimates of ``n_runs`` AIS runs.  ``first_run=None``: the whole ladder (sharded over the ranks of
        the context's communicator, if any); an integer: runs [first_run, first_run + n_runs) of it, computed here.
        ``base``: None, or one entry per unit layer (v, h_1 .. h_L), each None or the layer's base-rate biases -- the ladder
        then starts from that factorial model (bm_dbm_ais_base, DESIGN.md §5.4d)."""
        out = np.empty(int(n_runs), dtype=np.float64)
        bp, keep = None, []
        if base is not None:
            if len(base) != self.L + 1:
                raise ValueError('base needs one entry per unit layer (v, h_1 .. h_L): {0}'.format(self.L + 1))
            bp = (C.c_void_p * len(base))()
            for j, a in enumerate(base):
                if a is None:
                    continue
                a = np.ascontiguousarray(a, dtype=np.float32).ravel()
                if a.size != ([self.V] + self.Hs)[j]:
                    raise ValueError('base of layer {0} has {1} entries, the layer {2}'.format(j, a.size, ([self.V] + self.Hs)[j]))
                keep.append(a)
                bp[j] = a.ctypes.data
        if first_run is None:
            check(self._lib.bm_dbm_ais_base(self.handle, int(n_runs), int(n_betas), int(k), int(seed), bp, out.ctypes.data))
        else:
            check(self._lib.bm_dbm_ais_base_rows(self.handle, int(n_runs), int(n_betas), int(k), int(seed), int(first_run), bp,
                                                 out.ctypes.data))
        return out

    def exact(self, X=None):
        """Exact log p*(v) of X's rows (None: no rows) and log Z of a binary DBM with at most 32 odd-layer units, from one
        enumeration of the odd layers' states (bm_dbm_exact, DESIGN.md §5.4f).  Returns (log_p_star [rows] float64 or None,
        log_Z).  Refusals of the engine (BM_EUNSUPPORTED) raise NotImplementedError, bad arguments RuntimeError."""
        lz = C.c_double(0.0)
        if X is None:
            rc = self._lib.bm_dbm_exact(self.handle, None, 0, None, C.byref(lz))
            lp = None
        else:
            X = np.ascontiguousarray(X, dtype=np.float32)
            if X.ndim != 2 or X.shape[1] != self.V:
                raise ValueError('batch has shape {0}, expected (rows, {1})'.format(X.shape, self.V))
            lp = np.empty(X.shape[0], dtype=np.float64)
            rc = self._lib.bm_dbm_exact(self.handle, X.ctypes.data if len(X) else None, X.shape[0],
                                        lp.ctypes.data if len(X) else None, C.byref(lz))
        if rc == -5:                                  # BM_EUNSUPPORTED: the message names the reason
            raise NotImplementedError('libbm: ' + self._lib.bm_last_error().decode('utf-8', 'replace'))
        check(rc)
        return lp, lz.value

    def ais_clamped(self, X, n_runs, n_betas, k, seed, row0=0):
        """Per-run AIS estimates of log p*(v) for the rows of X with v clamped (bm_dbm_ais_clamped, DESIGN.md §5.4g):
        [rows, n_runs] float64, log Z_0 and b_v.v included; the rows are rows row0.. of the caller's data.  Refusals of the
        engine (BM_EUNSUPPORTED) raise NotImplementedError, bad arguments RuntimeError."""
        X = np.ascontiguousarray(X, dtype=np.float32)
        if X.ndim != 2 or X.shape[1] != self.V:
            raise ValueError('batch has shape {0}, expected (rows, {1})'.format(X.shape, self.V))
        out = np.empty((X.shape[0], max(int(n_runs), 0)), dtype=np.float64)
        rc = self._lib.bm_dbm_ais_clamped(self.handle, X.ctypes.data if X.size else None, X.shape[0], int(row0), int(n_runs),
                                          int(n_betas), int(k), int(seed), out.ctypes.data if out.size else None)
        if rc == -5:                                  # BM_EUNSUPPORTED: the message names the reason
            raise NotImplementedError('libbm: ' + self._lib.bm_last_error().decode('utf-8', 'replace'))
        check(rc)
        return out

    def debug_exact_chunk(self, log2_states):
        """states per launch of `exact`'s enumeration, 2^log2_states (0: the default) -- a test hook"""
        check(self._lib.bm_dbm_debug_exact_chunk(self.handle, int(log2_states)))

    def close(self):
        if getattr(self, 'handle', None):
            self._lib.bm_dbm_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CudaCRBM(object):
    """Engine object for ``ClassificationRBM``: a ``bm_crbm`` handle (csrc/bm_crbm_tc.cuh, tensor cores only).

    cfg: n_visible, n_hidden, n_classes, alpha, beta (labels of -1 mark unlabelled rows when beta > 0), l2, sample_v,
    sample_h, max_batch, and dtype / compute / dropout /
    sparsity_cost / dbm_first / dbm_last, which the engine refuses unless they are float32 / bf16 / None / 0 / False /
    False."""

    def __init__(self, cfg, ctx=None):
        self._lib = load_library()
        self.ctx = ctx or Context.default()
        self.cfg = dict(cfg)
        self.V, self.H, self.C = int(cfg['n_visible']), int(cfg['n_hidden']), int(cfg['n_classes'])
        self.dt = np.dtype(cfg.get('dtype', 'float32'))
        c = CrbmCfg()
        c.n_visible, c.n_hidden, c.n_classes = self.V, self.H, self.C
        c.dtype = DTYPES[self.dt.name]
        c.compute = COMPUTE[cfg.get('compute') or os.environ.get('BM_COMPUTE') or 'bf16']
        c.sample_v, c.sample_h = int(cfg.get('sample_v', False)), int(cfg.get('sample_h', True))
        c.max_batch = int(cfg['max_batch'])
        c.alpha, c.l2 = float(cfg.get('alpha', 0.01)), float(cfg.get('l2', 0.))
        keep = cfg.get('dropout', None)
        c.dropout_keep = -1.0 if keep is None else float(keep)
        c.sparsity_cost = float(cfg.get('sparsity_cost', 0.))
        c.dbm_first, c.dbm_last = int(bool(cfg.get('dbm_first', False))), int(bool(cfg.get('dbm_last', False)))
        c.beta = float(cfg.get('beta', 0.))
        h = C.c_void_p()
        rc = self._lib.bm_crbm_create(self.ctx.handle, C.byref(c), C.byref(h))
        if rc == -5:                                  # BM_EUNSUPPORTED: the message names the option
            raise NotImplementedError(self._lib.bm_last_error().decode('utf-8', 'replace'))
        check(rc)
        self.handle = h
        V, H, Cn = self.V, self.H, self.C
        self._shapes = {'W': (V, H), 'U': (Cn, H), 'vb': (V,), 'hb': (H,), 'yb': (Cn,),
                        'dW': (V, H), 'dU': (Cn, H), 'dvb': (V,), 'dhb': (H,), 'dyb': (Cn,)}
        self._out2 = (C.c_double * 2)()

    def set_params(self, d):
        for k, v in d.items():
            a = np.ascontiguousarray(v, dtype=np.float32).reshape(self._shapes[k])
            check(self._lib.bm_crbm_set_param(self.handle, k.encode(), a.ctypes.data, a.nbytes))

    def get_params(self, names=None):
        out = {}
        for k in (names or list(self._shapes)):
            a = np.empty(self._shapes[k], dtype=np.float32)
            check(self._lib.bm_crbm_get_param(self.handle, k.encode(), a.ctypes.data, a.nbytes))
            out[k] = a
        return out

    def init_normal_weights(self, stddev, op_seed_w, op_seed_u):
        check(self._lib.bm_crbm_init_weights(self.handle, float(stddev), int(op_seed_w) & (2 ** 64 - 1),
                                             int(op_seed_u) & (2 ** 64 - 1)))

    def _batch(self, X):
        X = np.ascontiguousarray(X, dtype=np.float32)
        if X.ndim != 2 or X.shape[1] != self.V:
            raise ValueError('batch has shape {0}, expected (rows, {1})'.format(X.shape, self.V))
        return X

    def train_step(self, X, y, lr, momentum, k, seed, tick, metrics=False):
        """One hybrid step; with ``metrics`` returns {'nll', 'accuracy'} of the batch under the pre-update weights."""
        X = self._batch(X)
        y = np.ascontiguousarray(y, dtype=np.int32).reshape(-1)
        if y.shape[0] != X.shape[0]:
            raise ValueError('{0} labels for {1} rows'.format(y.shape[0], X.shape[0]))
        check(self._lib.bm_crbm_train_step(self.handle, X.ctypes.data, y.ctypes.data, X.shape[0], float(lr), float(momentum),
                                           int(k), int(seed) & (2 ** 64 - 1), int(tick), 1 if metrics else 0, self._out2))
        self._last_rows = X.shape[0]
        return {'nll': float(self._out2[0]), 'accuracy': float(self._out2[1])} if metrics else None

    DEBUG_WIDTHS = {'A': 'H', 'P': 'C', 'y0': None, 'G': 'H', 'h0': 'H', 'x_k': 'V', 'y_k': 'C', 'h_k': 'H', 'aH': 'H'}

    def debug_last_step(self, names=('A', 'P', 'y0', 'G')):
        """the last train_step's buffers (bm_crbm_debug_last_step): A and P float32, y0 int32, the bf16 ones widened to
        float32.  The chain's 'h0', 'x_k', 'y_k', 'h_k', 'aH' exist only when the chain ran ('h0' only at k = 1)."""
        rows = getattr(self, '_last_rows', 0)
        out = {}
        for n in names:
            w = self.DEBUG_WIDTHS[n]
            shape = (rows,) if w is None else (rows, getattr(self, w))
            a = np.empty(shape, dtype={'A': np.float32, 'P': np.float32, 'y0': np.int32}.get(n, np.uint16))
            check(self._lib.bm_crbm_debug_last_step(self.handle, n.encode(), a.ctypes.data, a.nbytes))
            out[n] = (a.astype(np.uint32) << 16).view(np.float32) if a.dtype == np.uint16 else a
        return out

    def predict_proba(self, X):
        X = self._batch(X)
        out = np.empty((X.shape[0], self.C), dtype=np.float32)
        check(self._lib.bm_crbm_predict_proba(self.handle, X.ctypes.data, X.shape[0], out.ctypes.data))
        return out

    def transform(self, X):
        X = self._batch(X)
        out = np.empty((X.shape[0], self.H), dtype=np.float32)
        check(self._lib.bm_crbm_transform(self.handle, X.ctypes.data, X.shape[0], out.ctypes.data))
        return out

    def close(self):
        if getattr(self, 'handle', None):
            self._lib.bm_crbm_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def default_factory(kind):
    load_library()
    if kind == 'dbm':
        return CudaDBM
    if kind == 'rbm':
        return CudaRBM
    if kind == 'crbm':
        return CudaCRBM
    if kind == 'rbm_group':
        return CudaRBMGroup
    raise RuntimeError("no native engine for '{0}'".format(kind))

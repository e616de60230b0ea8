"""Run-time compilation of users' environment structs (NVRTC through ctypes) into the fused rollout, env-step and
env-observe kernels of csrc/rollout_kernel.cuh, for sm_90a.

One translation unit is generated per request: csrc/user_env.cuh, the user's source, the action-space bounds as
constants, and static_asserts that tie the struct's constants to the dimensions the Python side declared.  NVRTC
instantiates the requested kernels from their name expressions (nvrtcAddNameExpression) and reports their lowered names,
which promp_env_module_load resolves in the cubin.  Cubins are cached on disk, keyed by everything that goes into them.

NVRTC: the toolkit's libnvrtc whose version equals the CUDA version the library was built with is preferred (the built-in
env types then compile to the library's own code); otherwise the one of the CUDA wheel that torch depends on.
"""
import ctypes
import glob
import hashlib
import json
import os
import sys
import tempfile
import threading

from promp_b200 import _lib

CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'csrc')
INCLUDE = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'include')
ARCH = 'sm_90a'
OPTIONS = ('-arch=' + ARCH, '-std=c++17', '-default-device', '-lineinfo', '-I' + CSRC)
# NVRTC has no C library headers; the kernels need the fixed-width integer types only
_HEADERS = {'stdint.h': ('#pragma once\ntypedef signed char int8_t; typedef short int16_t; typedef int int32_t; '
                         'typedef long long int64_t;\ntypedef unsigned char uint8_t; typedef unsigned short uint16_t; '
                         'typedef unsigned int uint32_t; typedef unsigned long long uint64_t;\n')}
# activation traits of the `hidden` argument, in the order of the module's kernel slots (include/promp_b200.h)
ACTS = ('promp::ActTanh', 'promp::ActRelu', 'promp::OutTanh<promp::ActTanh>', 'promp::OutTanh<promp::ActRelu>')
ENV = 'promp_jit::Env'

STATS = {'compiles': 0, 'cache_hits': 0}      # counted per process (tests, tools/cuda_env_time.py)
_lock = threading.Lock()


class CudaEnvCompileError(RuntimeError):
    """NVRTC rejected a user environment; `log` is the compiler's log."""

    def __init__(self, msg, log=''):
        super().__init__(msg + ('\n' + log if log else ''))
        self.log = log


# ---------------------------------------------------------------------------------------------------------- names
def _variant(hidden):
    """(v, deep) of a `hidden` argument (width | ACT_RELU | OUT_TANH | depth bits): v = the variant index of env_module.cu,
    deep = one or three hidden layers (rollout_deep_kernel)."""
    width, relu, otanh = hidden & _lib.HIDDEN_WIDTH_MASK, bool(hidden & _lib.ACT_RELU), bool(hidden & _lib.OUT_TANH)
    depth = (hidden & _lib.HIDDEN_DEPTH_MASK) >> _lib.HIDDEN_DEPTH_SHIFT
    known = _lib.HIDDEN_WIDTH_MASK | _lib.ACT_RELU | _lib.OUT_TANH | _lib.HIDDEN_DEPTH_MASK
    if width not in (32, 64) or hidden & ~known or depth > 3:
        raise ValueError("user envs run policies of hidden width 32 or 64 and 1 to 3 hidden layers (hidden argument 0x%x)"
                         % hidden)
    return (int(relu) + 2 * int(otanh)) * 2 + int(width == 64), depth not in (0, 2)


def rollout_slot(hidden, keyed):
    """Kernel slot of the rollout kernel of a `hidden` argument, as env_module.cu."""
    v, deep = _variant(hidden)
    return (_lib.ENV_SLOT_ROLLOUT_DEEP if deep else _lib.ENV_SLOT_ROLLOUT) + 2 * v + int(keyed)


def name_expressions(hiddens=()):
    """{slot: name expression}: the env-step and env-observe kernels, and both rollout kernels of every `hidden`."""
    out = {_lib.ENV_SLOT_STEP: 'promp::env_step_kernel<%s>' % ENV, _lib.ENV_SLOT_OBSERVE: 'promp::env_observe_kernel<%s>' % ENV}
    for h in hiddens:
        v, deep = _variant(h)
        for keyed in (False, True):
            out[rollout_slot(h, keyed)] = 'promp::%s<%s, %d, %s, %s>' % (
                'rollout_deep_kernel' if deep else 'rollout_kernel', ENV, h & _lib.HIDDEN_WIDTH_MASK, ACTS[v // 2],
                'true' if keyed else 'false')
    return out


def translation_unit(source, struct_name, dims, low, high):
    """The generated source: user_env.cuh + the user's source + promp_jit::Env (the struct in the warp concept)."""
    do, da, sd, td, ninfo, ends_early = dims
    fl = lambda v: ', '.join('%.9ef' % float(x) for x in v)      # noqa: E731
    checks = ''.join('static_assert(Env::%s == %d, "%s: %s does not match the declared %s (%d)");\n' % (k, v, struct_name, k, n, v)
                     for k, n, v in (('DO', 'obs_dim', do), ('DA', 'act_dim', da), ('SD', 'state_dim', sd), ('TD', 'task_dim', td)))
    return ('#include "user_env.cuh"\n#line 1 "user_env"\n%s\n#line 1 "promp_jit"\nnamespace promp_jit {\n'
            'struct Bounds {\n'
            '    static __device__ __forceinline__ float lb(int d) { const float v[%d] = {%s}; return v[d]; }\n'
            '    static __device__ __forceinline__ float ub(int d) { const float v[%d] = {%s}; return v[d]; }\n'
            '};\n'
            'using Env = promp::UserEnvOf<%s, Bounds>::type;\n%s'
            'static_assert(Env::NINFO == %d, "%s: NINFO does not match the number of info_keys (%d)");\n'
            'static_assert(Env::ENDS_EARLY == %s, "%s: ENDS_EARLY does not match ends_early");\n'
            '}\n') % (source, da, fl(low), da, fl(high), struct_name, checks, ninfo, struct_name, ninfo,
                      'true' if ends_early else 'false', struct_name)


# ---------------------------------------------------------------------------------------------------------- NVRTC
class _Nvrtc(object):
    def __init__(self, path):
        self.path = path
        self.lib = lib = ctypes.CDLL(path)
        P, c = ctypes.c_void_p, ctypes
        for name, args in (('nvrtcVersion', [c.POINTER(c.c_int), c.POINTER(c.c_int)]),
                           ('nvrtcCreateProgram', [c.POINTER(P), c.c_char_p, c.c_char_p, c.c_int, P, P]),
                           ('nvrtcAddNameExpression', [P, c.c_char_p]),
                           ('nvrtcCompileProgram', [P, c.c_int, P]),
                           ('nvrtcGetProgramLogSize', [P, c.POINTER(c.c_size_t)]),
                           ('nvrtcGetProgramLog', [P, c.c_char_p]),
                           ('nvrtcGetCUBINSize', [P, c.POINTER(c.c_size_t)]),
                           ('nvrtcGetCUBIN', [P, c.c_char_p]),
                           ('nvrtcGetLoweredName', [P, c.c_char_p, c.POINTER(c.c_char_p)]),
                           ('nvrtcDestroyProgram', [c.POINTER(P)]),
                           ('nvrtcGetErrorString', [c.c_int])):
            fn = getattr(lib, name)
            fn.argtypes = args
            fn.restype = c.c_char_p if name == 'nvrtcGetErrorString' else c.c_int
        mj, mn = c.c_int(), c.c_int()
        lib.nvrtcVersion(c.byref(mj), c.byref(mn))
        self.version = (mj.value, mn.value)

    def _check(self, st, what):
        if st != 0:
            raise CudaEnvCompileError("%s failed: %s" % (what, self.lib.nvrtcGetErrorString(st).decode()))

    def compile(self, src, name, exprs, options):
        """-> (cubin bytes, [lowered name per expression], log)"""
        c = ctypes
        prog = c.c_void_p()
        hn = list(_HEADERS)
        hdr_src = (c.c_char_p * len(hn))(*[_HEADERS[k].encode() for k in hn])
        hdr_names = (c.c_char_p * len(hn))(*[k.encode() for k in hn])
        self._check(self.lib.nvrtcCreateProgram(c.byref(prog), src.encode(), name.encode(), len(hn),
                                                c.cast(hdr_src, c.c_void_p), c.cast(hdr_names, c.c_void_p)),
                    'nvrtcCreateProgram')
        try:
            for e in exprs:
                self._check(self.lib.nvrtcAddNameExpression(prog, e.encode()), 'nvrtcAddNameExpression')
            opts = (c.c_char_p * len(options))(*[o.encode() for o in options])
            st = self.lib.nvrtcCompileProgram(prog, len(options), c.cast(opts, c.c_void_p))
            n = c.c_size_t()
            self.lib.nvrtcGetProgramLogSize(prog, c.byref(n))
            buf = c.create_string_buffer(n.value)
            self.lib.nvrtcGetProgramLog(prog, buf)
            log = buf.value.decode('utf-8', 'replace')
            if st != 0:
                raise CudaEnvCompileError("NVRTC %d.%d could not compile the environment (%s):"
                                          % (self.version + (self.lib.nvrtcGetErrorString(st).decode(),)), log)
            self._check(self.lib.nvrtcGetCUBINSize(prog, c.byref(n)), 'nvrtcGetCUBINSize')
            cubin = c.create_string_buffer(n.value)
            self._check(self.lib.nvrtcGetCUBIN(prog, cubin), 'nvrtcGetCUBIN')
            lowered = []
            for e in exprs:
                out = c.c_char_p()
                self._check(self.lib.nvrtcGetLoweredName(prog, e.encode(), c.byref(out)), 'nvrtcGetLoweredName')
                lowered.append(out.value.decode())
            return cubin.raw, lowered, log
        finally:
            self.lib.nvrtcDestroyProgram(c.byref(prog))


def _toolkit_nvrtc():
    dirs = [os.path.join(os.environ[k], 'lib64') for k in ('CUDA_HOME', 'CUDA_PATH') if os.environ.get(k)]
    from promp_b200 import _build
    try:
        dirs.append(os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(_build._nvcc()))), 'lib64'))
    except RuntimeError:
        pass
    dirs.append('/usr/local/cuda/lib64')
    return [p for d in dirs for p in sorted(glob.glob(os.path.join(d, 'libnvrtc.so.[0-9]*')))
            if os.path.basename(p).count('.') == 2]      # libnvrtc.so.<major>


def _wheel_nvrtc():
    return [os.path.join(d, 'nvidia', 'cuda_nvrtc', 'lib', 'libnvrtc.so.12') for d in sys.path
            if os.path.exists(os.path.join(d, 'nvidia', 'cuda_nvrtc', 'lib', 'libnvrtc.so.12'))]


_nvrtc = None


def nvrtc():
    """The NVRTC in use (loaded once): `.version`, `.path`."""
    global _nvrtc
    with _lock:
        if _nvrtc is None:
            build = _lib.load().promp_cuda_build_version()
            want = (build // 1000, (build % 1000) // 10)
            first = None
            for p in _toolkit_nvrtc():
                try:
                    n = _Nvrtc(p)
                except OSError:
                    continue
                if n.version == want:
                    _nvrtc = n
                    break
                first = first or n
            if _nvrtc is None:
                for p in _wheel_nvrtc():
                    try:
                        _nvrtc = _Nvrtc(p)
                        break
                    except OSError:
                        continue
            _nvrtc = _nvrtc or first
            if _nvrtc is None:
                raise CudaEnvCompileError("no NVRTC library found (CUDA toolkit lib64 or the nvidia-cuda-nvrtc wheel): user "
                                          "environments cannot be compiled")
        return _nvrtc


def matches_library():
    """True when the NVRTC in use is the CUDA version the library was built with."""
    b = _lib.load().promp_cuda_build_version()
    return nvrtc().version == (b // 1000, (b % 1000) // 10)


# ---------------------------------------------------------------------------------------------------------- cache
def cache_dir():
    """PROMP_B200_JIT_CACHE, else $XDG_CACHE_HOME/promp_b200/jit (~/.cache), else a per-user temporary directory."""
    d = os.environ.get('PROMP_B200_JIT_CACHE')
    if not d:
        base = os.environ.get('XDG_CACHE_HOME') or os.path.join(os.path.expanduser('~'), '.cache')
        d = os.path.join(base, 'promp_b200', 'jit')
    try:
        os.makedirs(d, exist_ok=True)
        if os.access(d, os.W_OK):
            return d
    except OSError:
        pass
    d = os.path.join(tempfile.gettempdir(), 'promp_b200_jit_%d' % os.getuid())
    os.makedirs(d, exist_ok=True)
    return d


def _headers_digest():
    h = hashlib.sha256()
    for p in sorted(glob.glob(os.path.join(CSRC, '*.cuh'))) + [os.path.join(INCLUDE, 'promp_b200.h')]:
        h.update(os.path.basename(p).encode())
        with open(p, 'rb') as f:
            h.update(f.read())
    return h.hexdigest()


def compile_kernels(tu, exprs):
    """Compile `tu` for sm_90a and lower `exprs` ({slot: name expression}).  -> (cubin, {slot: lowered name}); from the
    disk cache when the same source, headers, NVRTC version, options and expressions were compiled before."""
    nv = nvrtc()
    slots = sorted(exprs)
    key = hashlib.sha256(json.dumps([tu, _headers_digest(), list(nv.version), list(OPTIONS), [exprs[s] for s in slots]])
                         .encode()).hexdigest()[:40]
    d = cache_dir()
    cub, meta = os.path.join(d, key + '.cubin'), os.path.join(d, key + '.json')
    if os.path.exists(cub) and os.path.exists(meta):
        try:
            with open(meta) as f:
                names = {int(k): v for k, v in json.load(f)['lowered'].items()}
            with open(cub, 'rb') as f:
                image = f.read()
            STATS['cache_hits'] += 1
            return image, names
        except (OSError, ValueError, KeyError):
            pass
    image, lowered, log = nv.compile(tu, 'promp_user_env.cu', [exprs[s] for s in slots], list(OPTIONS))
    STATS['compiles'] += 1
    names = dict(zip(slots, lowered))
    for path, data, mode in ((cub, image, 'wb'), (meta, json.dumps(dict(
            lowered={str(k): v for k, v in names.items()}, nvrtc=list(nv.version), log=log)), 'w')):
        tmp = '%s.%d.tmp' % (path, os.getpid())      # atomic publish: concurrent builders never read a torn file
        with open(tmp, mode) as f:
            f.write(data)
        os.replace(tmp, path)
    return image, names

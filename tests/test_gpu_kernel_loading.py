"""Every kernel of the library is loaded once `dm_prepare_kernels` returns (DESIGN §7): CUDA loads kernels lazily, and
a first launch while a persistent ps serve kernel is resident can deadlock on the context-wide synchronisation the
load needs. And every instantiation of the fused step that a batch can run fits as many clusters as the ReLU one."""
import ctypes as C
import json
import os
import re
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu


def library_kernels(lib_path: str) -> dict:
    """{translation unit: [mangled kernel names]} of the library's sm_90a cubins, from the ELF symbol tables."""
    from dist_mnist_b200 import _build

    out = subprocess.run([str(_build._cuda_home() / "bin" / "cuobjdump"), "-symbols", lib_path], capture_output=True,
                         text=True, check=True).stdout
    kernels, unit = {}, None
    for line in out.splitlines():
        if line.startswith("identifier = "):
            unit = os.path.basename(line.split("=", 1)[1].strip())
            kernels[unit] = []
        elif unit is not None and (m := re.match(r"STT_FUNC\s+STB_GLOBAL\s+STO_ENTRY\s+(\S+)", line)):
            kernels[unit].append(m.group(1))
    return {u: names for u, names in kernels.items() if names}


def loading_states(lib_path: str, probes: list) -> dict:
    """{function name: loaded} over every function of the module that holds each probe kernel, after
    `dm_prepare_kernels(0)`. Runs in a process that has launched nothing. The module is found through the probe's
    context-independent kernel handle: a CUfunction handle of the probe (cudaGetFuncBySymbol) would load it."""
    lib = C.CDLL(lib_path)
    rt = C.CDLL("libcudart.so.12")   # the runtime the library links, already loaded with it
    drv = C.CDLL("libcuda.so.1")

    def cu(rc, what):
        if rc != 0:
            raise RuntimeError(f"{what} failed with {rc}")

    cu(lib.dm_prepare_kernels(0), "dm_prepare_kernels")
    states = {}
    for probe in probes:
        kernel, library, mod, n = C.c_void_p(), C.c_void_p(), C.c_void_p(), C.c_uint()
        cu(rt.cudaGetKernel(C.byref(kernel), C.cast(getattr(lib, probe), C.c_void_p)), "cudaGetKernel")
        cu(drv.cuKernelGetLibrary(C.byref(library), kernel), "cuKernelGetLibrary")
        cu(drv.cuLibraryGetModule(C.byref(mod), library), "cuLibraryGetModule")
        cu(drv.cuModuleGetFunctionCount(C.byref(n), mod), "cuModuleGetFunctionCount")
        fns = (C.c_void_p * n.value)()
        cu(drv.cuModuleEnumerateFunctions(fns, n, mod), "cuModuleEnumerateFunctions")
        for f in fns:
            name, state = C.c_char_p(), C.c_int()
            cu(drv.cuFuncGetName(C.byref(name), C.c_void_p(f)), "cuFuncGetName")
            cu(drv.cuFuncIsLoaded(C.byref(state), C.c_void_p(f)), "cuFuncIsLoaded")
            states[name.value.decode()] = state.value == 1   # CU_FUNCTION_LOADING_STATE_LOADED
    return states


def driver_version() -> int:
    v = C.c_int(0)
    C.CDLL("libcuda.so.1").cuDriverGetVersion(C.byref(v))
    return v.value


def test_every_kernel_is_loaded_after_prepare():
    from dist_mnist_b200 import _native as N

    N.lib()
    if driver_version() < 12050:
        pytest.skip(f"driver {driver_version()} cannot report whether a function is loaded (needs 12.5)")
    lib_path = str(N.lib_path())
    kernels = library_kernels(lib_path)
    probes = [names[0] for names in kernels.values()]   # one kernel per module
    # a fresh process, so that nothing has been launched or loaded before dm_prepare_kernels
    r = subprocess.run([sys.executable, __file__, lib_path, *probes], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, CUDA_MODULE_LOADING="LAZY"))
    assert r.returncode == 0, r.stderr
    states = json.loads(r.stdout.splitlines()[-1])
    assert sorted(states) == sorted(n for names in kernels.values() for n in names)
    assert [n for n, loaded in states.items() if not loaded] == []


def test_fused_lane_cap_is_that_of_the_relu_kernel_for_every_instantiation():
    """The clip, L2 and activation instantiations have the shared memory and (<= 255) registers of the plain ReLU one
    at each batch: the same cluster count fits on the device, and so the same lanes beside the ps serve kernel."""
    from dist_mnist_b200 import _native as N

    lib = N.lib()
    N.ensure_prepared(0)

    def lanes(B, clip, l2, act):
        out = C.c_int(0)
        N.check(lib.dm_fused_max_lanes(0, B, clip, l2, act, C.byref(out)))
        return out.value

    for B in (1, 32, 33, 256):
        relu = lanes(B, 0, 0, N.ACT_RELU)
        assert relu > 0
        for clip in (0, 1):
            for l2 in (0, 1):
                for act in range(N.ACT_TANH + 1):
                    assert lanes(B, clip, l2, act) == relu, (B, clip, l2, act)


if __name__ == "__main__":
    print(json.dumps(loading_states(sys.argv[1], sys.argv[2:])))

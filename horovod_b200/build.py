"""In-tree native build: `python -m horovod_b200.build [--force] [--no-torch]`.

Produces (next to this file, git-ignored):
  lib/libhvd_core.so   C++ runtime + sm_90a CUDA kernels (g++ / nvcc, no torch headers: compiles in seconds)
  lib/_hvd_torch.so    pybind11/ATen binding linked against libhvd_core.so

Role parity: the reference's CMakeLists.txt + setup.py CMake driver
(horovod/CMakeLists.txt, cmake/build_utils.py:93-118 for the -gencode list).
Here the only device target is sm_90a (H100).
"""
import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "csrc")
OUT = os.path.join(ROOT, "lib")
OBJ = os.path.join(ROOT, "build", "obj")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.path.join(CUDA_HOME, "bin", "nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

CORE_DIRS = ["common", "common/optim", "transport", "ops", "symm", "kernels"]


def _sources():
    cc, cu = [], []
    for d in CORE_DIRS:
        p = os.path.join(CSRC, d)
        for f in sorted(os.listdir(p)):
            if f.endswith(".cc"):
                cc.append(os.path.join(p, f))
            elif f.endswith(".cu"):
                cu.append(os.path.join(p, f))
    return cc, cu


def _header_digest():
    h = hashlib.sha1()
    for base, _, files in sorted(os.walk(CSRC)):
        for f in sorted(files):
            if f.endswith((".h", ".cuh")):
                with open(os.path.join(base, f), "rb") as fh:
                    h.update(fh.read())
    return h.hexdigest()[:12]


def _src_stamp(src, header_stamp):
    """Content hash of the translation unit + every header: staleness never depends on file mtimes (a snapshot copied to
    another machine keeps the contents but not necessarily the timestamps)."""
    with open(src, "rb") as fh:
        return hashlib.sha1(fh.read() + header_stamp.encode()).hexdigest()[:16]


def _needs(src, obj, stamp):
    return not (os.path.exists(obj) and os.path.exists(obj + "." + stamp))


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + "\n")
        raise RuntimeError("build failed: " + os.path.basename(cmd[-1] if cmd else ""))
    return r.stdout


def _compile(src, stamp, force, verbose, cxx=None):
    """Compiles one source into build/obj unless its content stamp is unchanged.  `cxx`: the compiler command for a .cc
    file without its input and output (default: the runtime's)."""
    rel = os.path.relpath(src, CSRC).replace("/", "__")
    obj = os.path.join(OBJ, rel + ".o")
    stamp = _src_stamp(src, stamp)
    if not force and not _needs(src, obj, stamp):
        return obj
    inc = ["-I" + os.path.join(CUDA_HOME, "include"), "-I/usr/include"]
    if src.endswith(".cu"):
        cmd = [NVCC] + ARCH + ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"] + inc + ["-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
    elif cxx is not None:
        cmd = cxx + ["-c", src, "-o", obj]
    else:
        # the host reduction / scaling loops of ops/ want the vectoriser (-O3); the rest of the runtime is control flow
        opt = "-O3" if os.sep + "ops" + os.sep in src else "-O2"
        cmd = ["g++", opt, "-g1", "-std=c++17", "-fPIC", "-Wall", "-Wno-unused-function", "-pthread"] + inc + ["-c", src, "-o", obj]
    out = _run(cmd)
    if verbose and out.strip():
        print(out)
    for f in os.listdir(OBJ):
        if f.startswith(rel + ".o.") and f != rel + ".o." + stamp:
            os.remove(os.path.join(OBJ, f))
    open(obj + "." + stamp, "w").close()
    return obj


def build_core(force=False, verbose=False):
    os.makedirs(OUT, exist_ok=True)
    os.makedirs(OBJ, exist_ok=True)
    stamp = _header_digest()
    cc, cu = _sources()
    with ThreadPoolExecutor(max_workers=max(2, os.cpu_count() or 4)) as ex:
        objs = list(ex.map(lambda s: _compile(s, stamp, force, verbose), cu + cc))
    lib = os.path.join(OUT, "libhvd_core.so")
    # the stamps of the runtime's objects only (build_torch keeps the binding's torch__*.o next to them)
    link_stamp = hashlib.sha1("".join(sorted(f for f in os.listdir(OBJ) if ".o." in f and not f.startswith("torch__")))
                              .encode()).hexdigest()[:16]
    stamp_file = os.path.join(OBJ, "core_link.stamp")
    old = open(stamp_file).read() if os.path.exists(stamp_file) else ""
    if force or not os.path.exists(lib) or old != link_stamp:
        _run([NVCC] + ARCH + ["-shared", "-o", lib] + objs + ["-cudart", "static", "-lpthread", "-ldl", "-lrt"])
        # libcuda is resolved lazily with dlsym (a CPU-only box must be able to load the library): a direct reference to a
        # driver entry point would only fail at dlopen time on such a box, so fail the build instead
        undef = [l.split()[-1] for l in _run(["nm", "-D", "--undefined-only", lib]).splitlines() if l.split()]
        direct = sorted(u for u in undef if u.startswith("cu") and len(u) > 2 and u[2].isupper() and not u.startswith("cuda"))
        if direct:
            os.remove(lib)
            raise RuntimeError("libhvd_core.so references CUDA driver symbols directly (use dlsym): " + ", ".join(direct))
        with open(stamp_file, "w") as f:
            f.write(link_stamp)
    return lib


def build_torch(force=False):
    import torch
    from torch.utils import cpp_extension

    tdir = os.path.join(CSRC, "torch")
    srcs = [os.path.join(tdir, f) for f in sorted(os.listdir(tdir)) if f.endswith(".cc")]
    lib = os.path.join(OUT, "_hvd_torch.so")
    os.makedirs(OBJ, exist_ok=True)
    stamp_file = os.path.join(OBJ, "torch_binding.stamp")
    core_stamp = os.path.join(OBJ, "core_link.stamp")
    # the binding's sources are compiled against the torch headers: a torch upgrade rebuilds every object
    hstamp = _header_digest() + torch.__version__
    src_stamps = "".join(_src_stamp(s, hstamp) for s in srcs)
    stamp = hashlib.sha1(src_stamps.encode()).hexdigest()[:16] + "-" + torch.__version__ + "-" + (
        open(core_stamp).read() if os.path.exists(core_stamp) else "")
    old = open(stamp_file).read() if os.path.exists(stamp_file) else ""
    if not force and os.path.exists(lib) and old == stamp:
        return lib
    inc = ["-I" + p for p in cpp_extension.include_paths()] + ["-I" + os.path.join(CUDA_HOME, "include"),
                                                               "-I" + sysconfig.get_paths()["include"]]
    tlib = os.path.join(os.path.dirname(torch.__file__), "lib")
    abi = int(torch._C._GLIBCXX_USE_CXX11_ABI) if hasattr(torch._C, "_GLIBCXX_USE_CXX11_ABI") else 1
    cxx = ["g++", "-O2", "-std=c++17", "-fPIC", "-pthread", "-DTORCH_EXTENSION_NAME=_hvd_torch",
           "-DTORCH_API_INCLUDE_EXTENSION_H", "-D_GLIBCXX_USE_CXX11_ABI=%d" % abi, "-Wno-deprecated-declarations"] + inc
    with ThreadPoolExecutor(max_workers=max(2, os.cpu_count() or 4)) as ex:
        objs = list(ex.map(lambda s: _compile(s, hstamp, force, False, cxx), srcs))
    _run(["g++", "-shared", "-pthread"] + objs + [
        "-o", lib, "-L" + OUT, "-lhvd_core", "-L" + tlib, "-lc10", "-lc10_cuda", "-ltorch_cpu", "-ltorch", "-ltorch_python",
        "-L" + os.path.join(CUDA_HOME, "lib64"), "-lcudart", "-Wl,-rpath,$ORIGIN", "-Wl,-rpath," + tlib])
    with open(stamp_file, "w") as f:
        f.write(stamp)
    return lib


def build_all(force=False, verbose=False, with_torch=True):
    libs = [build_core(force, verbose)]
    if with_torch:
        libs.append(build_torch(force))
    return libs


def clean():
    shutil.rmtree(os.path.join(ROOT, "build"), ignore_errors=True)
    shutil.rmtree(OUT, ignore_errors=True)


def build_tsan_selftest(force=False, sanitizer="thread"):
    """ThreadSanitizer build of the C++ runtime + its native self-test (N engines in one process over the loopback
    transport: controller, response cache, fusion, CPU ops, process sets, join, error paths) as a stand-alone executable.
    The sm_90a kernel objects are linked as they are (device code is not instrumented).  The reference has no sanitizer
    build at all (SURVEY.md 5.2).  `sanitizer="address,undefined"` builds the AddressSanitizer + UBSan flavour of the same binary."""
    build_core()
    tag = "tsan" if sanitizer == "thread" else "san_" + "".join(c if c.isalnum() else "_" for c in sanitizer)
    odir = os.path.join(os.path.dirname(OBJ), "obj_" + tag)
    os.makedirs(odir, exist_ok=True)
    hstamp = _header_digest()
    cc, _ = _sources()
    main = os.path.join(odir, "selftest_main.cc")
    with open(main, "w") as f:
        f.write('#include <cstdio>\nextern "C" int hvd_selftest(int nranks, char* log, int log_len);\n'
                'int main() { static char log[1 << 16]; int rc = hvd_selftest(4, log, sizeof log); std::fputs(log, stdout); return rc; }\n')
    inc = ["-I" + os.path.join(CUDA_HOME, "include")]

    def one(src):
        rel = os.path.relpath(src, CSRC).replace("/", "__") if src.startswith(CSRC) else os.path.basename(src)
        obj = os.path.join(odir, rel + ".o")
        stamp = _src_stamp(src, hstamp + tag)
        if force or _needs(src, obj, stamp):
            _run(["g++", "-O1", "-g", "-std=c++17", "-fsanitize=" + sanitizer, "-fno-omit-frame-pointer", "-fPIC", "-pthread"] + inc + ["-c", src, "-o", obj])
            for f in os.listdir(odir):
                if f.startswith(rel + ".o.") and f != rel + ".o." + stamp:
                    os.remove(os.path.join(odir, f))
            open(obj + "." + stamp, "w").close()
        return obj
    with ThreadPoolExecutor(max_workers=max(2, os.cpu_count() or 4)) as ex:
        objs = list(ex.map(one, cc + [main]))
    kernels = [os.path.join(OBJ, f) for f in sorted(os.listdir(OBJ)) if f.startswith("kernels__") and f.endswith(".o")]
    exe = os.path.join(os.path.dirname(OBJ), "selftest_" + tag)
    _run(["g++", "-fsanitize=" + sanitizer, "-pthread"] + objs + kernels + ["-o", exe, "-L" + os.path.join(CUDA_HOME, "lib64"),
                                                                      "-lcudart_static", "-ldl", "-lrt", "-lpthread"])
    return exe


if __name__ == "__main__":
    if "--clean" in sys.argv:
        clean()
    if "--tsan" in sys.argv:
        print("built", build_tsan_selftest(force="--force" in sys.argv))
        sys.exit(0)
    libs = build_all(force="--force" in sys.argv, verbose="-v" in sys.argv, with_torch="--no-torch" not in sys.argv)
    for l in libs:
        print("built", l)

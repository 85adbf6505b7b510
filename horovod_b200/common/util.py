"""Small shared helpers (reference horovod/common/util.py)."""
import os
import warnings
from contextlib import contextmanager


@contextmanager
def env(**kwargs):
    """Temporarily set environment variables (None deletes)."""
    backup = {}
    for k, v in kwargs.items():
        backup[k] = os.environ.get(k)
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = str(v)
    try:
        yield
    finally:
        for k, v in backup.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def split_list(l, n):
    """Splits list l into n approximately even sized chunks."""
    d, r = divmod(len(l), n)
    return [l[i * d + min(i, r):(i + 1) * d + min(i + 1, r)] for i in range(n)]


def num_rank_is_power_2(num_rank):
    return num_rank != 0 and (num_rank & (num_rank - 1)) == 0


def is_iterable(x):
    try:
        iter(x)
    except TypeError:
        return False
    return True


def resolve_op(op, average, Average, Sum):
    """`op` supersedes the legacy `average=` kwarg (reference common/util.py:214-232)."""
    if op is not None:
        if average is not None:
            raise ValueError('The op parameter supersedes average. Please provide only one of them.')
        return op
    if average is not None:
        warnings.warn('Parameter `average` has been replaced with `op` and will be removed', DeprecationWarning)
        return Average if average else Sum
    return Average


def is_version_greater_equal_than(ver, target):
    from packaging import version
    return version.parse(ver) >= version.parse(target)


# ---- build / availability queries (role parity: horovod/common/util.py extension_available, gpu_available, *_built,
# check_installed_version).  There is one native library for all front ends, so "is the <framework> extension
# available" reduces to "is the native runtime built and is that framework importable".
_FRAMEWORK_MODULE = {'torch': 'torch', 'tensorflow': 'tensorflow', 'mxnet': 'mxnet', 'keras': 'tensorflow', 'numpy': 'numpy'}


def _native_lib():
    from horovod_b200.common.basics import load_library
    return load_library()


def extension_available(ext_base_name, verbose=False):
    """True when `horovod_b200.<ext_base_name>` can be used in this environment."""
    import importlib.util
    mod = _FRAMEWORK_MODULE.get(ext_base_name, ext_base_name)
    if importlib.util.find_spec(mod) is None:
        if verbose:
            print('%s is not installed' % mod)
        return False
    try:
        _native_lib()
        return True
    except Exception as e:  # noqa: BLE001
        if verbose:
            print('native runtime unavailable: %s' % e)
        return False


def gpu_available(ext_base_name='torch', verbose=False):
    """True when the native runtime sees at least one CUDA device (the P2P kernels are sm_90a only)."""
    if not extension_available(ext_base_name, verbose):
        return False
    try:
        import torch
        return bool(torch.cuda.is_available())
    except ImportError:
        return False


def _built(query, verbose=False):
    try:
        return bool(getattr(_native_lib(), query)())
    except Exception as e:  # noqa: BLE001
        if verbose:
            print('%s: %s' % (query, e))
        return False


def mpi_built(verbose=False):
    return False  # there is no MPI data or control plane in this runtime


def gloo_built(verbose=False):
    return _built('hvd_gloo_built', verbose)  # the native TCP/shm mesh fills Gloo's role


def nccl_built(verbose=False):
    return _built('hvd_nccl_built', verbose)


def ddl_built(verbose=False):
    return False


def ccl_built(verbose=False):
    return False


def check_installed_version(name, version, exception=None):
    """Warns when the running `name` differs from the version the package was built against (the native binding is
    compiled against torch headers; other front ends go through DLPack and have no build-time version)."""
    import warnings
    try:
        from horovod_b200.build import ROOT
        import os
        stamp = os.path.join(ROOT, 'build', 'obj', 'torch_binding.stamp')
        built = open(stamp).read().split('-')[1] if name == 'torch' and os.path.exists(stamp) else None
    except Exception:  # noqa: BLE001
        built = None
    if built and built != version:
        msg = ('horovod_b200 was built against %s %s but %s is running; rebuild with `python -m horovod_b200.build`' % (name, built, version))
        if exception is not None:
            raise type(exception)(msg)
        warnings.warn(msg)
        return False
    return True


def get_average_backwards_compatibility_fun(reduce_ops):
    """Returns f(op, average) implementing the deprecated `average=` argument for a front end's ReduceOps namespace."""
    def impl(op, average):
        return resolve_op(op, average, reduce_ops.Average, reduce_ops.Sum)
    return impl


EXTENSIONS = ['torch', 'tensorflow', 'mxnet', 'numpy']


class HorovodVersionMismatchError(ImportError):
    """The native binding was built against another version of the framework than the one that is running."""

    def __init__(self, name, version, installed_version):
        super().__init__(get_version_mismatch_message(name, version, installed_version))
        self.name, self.version, self.installed_version = name, version, installed_version


def get_version_mismatch_message(name, version, installed_version):
    return ('Framework %s installed with version %s but found version %s.\n'
            '             This can result in unexpected behavior including runtime errors.\n'
            '             Rebuild the native libraries with `python -m horovod_b200.build --force` to build against the running version.'
            % (name, installed_version, version))


def get_extension_full_path(pkg_path=None, *args):
    """Path of the shared object that serves a front end.  All front ends share ONE binding (`lib/_hvd_torch.so`) on top of
    `lib/libhvd_core.so`; the arguments of the reference's per-framework lookup are accepted and ignored."""
    import os
    from horovod_b200.common.basics import lib_dir
    return os.path.join(lib_dir(), '_hvd_torch.so')


def get_ext_suffix():
    """File suffix of Python extension modules of the running interpreter (reference common/util.py:26-35)."""
    import sysconfig
    return sysconfig.get_config_var('EXT_SUFFIX') or sysconfig.get_config_var('SO') or '.so'


def check_extension(ext_name, ext_env_var=None, pkg_path=None, *args):
    """Raises ImportError with a build hint when the native library behind `ext_name` (e.g. 'horovod.torch') is missing
    (reference common/util.py:38-46; `ext_env_var` named the HOROVOD_WITH_* switch of the reference's per-framework builds —
    here every front end shares one library, built by `python -m horovod_b200.build`)."""
    import os
    full_path = get_extension_full_path(pkg_path, *args)
    if not os.path.exists(full_path):
        raise ImportError('Extension %s has not been built: %s not found.\nRun `python -m horovod_b200.build` (or '
                          '`python setup.py build_ext --inplace`) to build the native runtime.' % (ext_name, full_path))


def _parse_cpulist(text):
    cpus = set()
    for part in text.strip().split(','):
        if not part:
            continue
        if '-' in part:
            a, b = part.split('-', 1)
            cpus.update(range(int(a), int(b) + 1))
        else:
            cpus.add(int(part))
    return cpus


def gpu_numa_cpus(pci_domain, pci_bus, pci_device, sysfs='/sys'):
    """CPUs local to the NUMA node of a GPU given its PCI address, or None (no NUMA information / single node)."""
    import os
    dev = os.path.join(sysfs, 'bus/pci/devices/%04x:%02x:%02x.0' % (pci_domain, pci_bus, pci_device))
    try:
        with open(os.path.join(dev, 'numa_node')) as f:
            node = int(f.read().strip())
        if node < 0:
            return None
        with open(os.path.join(sysfs, 'devices/system/node/node%d/cpulist' % node)) as f:
            return _parse_cpulist(f.read()) or None
    except (OSError, ValueError):
        return None


def bind_to_gpu_numa(device_index, sysfs='/sys'):
    """Restricts the calling thread (and every thread it creates afterwards, e.g. the runtime's cycle thread) to the CPUs
    of the NUMA node the GPU hangs off — SURVEY C14 ("default: pin near GPU's NUMA node").  With 8 ranks on a two-socket
    box, unbound rank processes bounce between sockets and the pinned-memory H2D copies of GPUs 4-7 cross the socket
    interconnect.  No-op when the process already runs with a restricted affinity the user chose that does not overlap,
    when sysfs has no NUMA data, or with HVD_NUMA_BIND=0.  Returns the CPU set applied, or None."""
    import os
    if os.environ.get('HVD_NUMA_BIND', '1') == '0' or not hasattr(os, 'sched_setaffinity'):
        return None
    try:
        import torch
        if not torch.cuda.is_available() or device_index >= torch.cuda.device_count():
            return None
        prop = torch.cuda.get_device_properties(device_index)
        local = gpu_numa_cpus(getattr(prop, 'pci_domain_id', 0), prop.pci_bus_id, prop.pci_device_id, sysfs)
        if not local:
            return None
        current = os.sched_getaffinity(0)
        target = current & local
        if not target or target == current:
            return None
        os.sched_setaffinity(0, target)
        return target
    except Exception:  # noqa: BLE001 - binding is an optimisation, never a reason to fail init
        return None

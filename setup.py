"""pip / setuptools entry point.  `pip install -e .` (or `python setup.py build_ext --inplace`) compiles the native
runtime IN-TREE for sm_90a through horovod_b200/build.py (g++ + nvcc, no CMake needed; a CMakeLists.txt for the core
library is provided as well).  Role parity: the reference's setup.py (CMake extension driver)."""
import os
import sys

from setuptools import Command, find_packages, setup
from setuptools.command.build_ext import build_ext as _build_ext
from setuptools.command.build_py import build_py as _build_py

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)


def _native_build(force=False):
    from horovod_b200 import build
    return build.build_all(force=force, with_torch=os.environ.get('HVD_WITHOUT_PYTORCH', '0') != '1')


class build_ext(_build_ext):
    def run(self):
        for lib in _native_build(force=bool(os.environ.get('HVD_FORCE_REBUILD'))):
            print('built', lib)


class build_py(_build_py):
    def run(self):
        self.run_command('build_ext')
        super().run()


class native_selftest(Command):
    description = 'run the native (C++) self-test of the runtime'
    user_options = []

    def initialize_options(self):
        pass

    def finalize_options(self):
        pass

    def run(self):
        import ctypes
        _native_build()
        lib = ctypes.CDLL(os.path.join(HERE, 'horovod_b200', 'lib', 'libhvd_core.so'))
        buf = ctypes.create_string_buffer(1 << 16)
        rc = lib.hvd_selftest(4, buf, len(buf))
        print(buf.value.decode(errors='replace'))
        if rc != 0:
            raise SystemExit(rc)


setup(
    name='horovod_b200',
    version='0.1.0',
    description='Hopper-native (H100) data-parallel collective library with the capabilities of Horovod',
    packages=find_packages(include=['horovod_b200', 'horovod_b200.*', 'horovod']),
    package_data={'horovod_b200': ['lib/*.so', 'csrc/**/*']},
    scripts=['bin/hvdrun', 'bin/horovodrun'],
    python_requires='>=3.9',
    install_requires=['torch', 'numpy', 'psutil', 'pyyaml', 'cloudpickle'],
    extras_require={'spark': ['pyspark', 'pyarrow', 'pandas'], 'ray': ['ray'], 'tensorflow': ['tensorflow'], 'mxnet': ['mxnet']},
    cmdclass={'build_ext': build_ext, 'build_py': build_py, 'selftest': native_selftest},
    entry_points={'console_scripts': ['horovodrun = horovod_b200.runner.launch:run_commandline']},
)

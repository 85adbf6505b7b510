"""Sanitizer jobs (SURVEY.md 5.2: the reference has none).

* ThreadSanitizer build of the C++ runtime running the native self-test (4 engines in one process) — CPU.
* compute-sanitizer memcheck over the P2P kernels in the single-GPU simulation and the fused optimizer kernels — GPU.
"""
import os
import shutil
import subprocess
import sys

import pytest

from conftest import REPO


def test_native_selftest_under_thread_sanitizer():
    if shutil.which('g++') is None:
        pytest.skip('no g++')
    from horovod_b200 import build
    exe = build.build_tsan_selftest()
    env = dict(os.environ, TSAN_OPTIONS='halt_on_error=0 report_signal_unsafe=0 exitcode=66', HOROVOD_LOG_LEVEL='error')
    # second pass: tiny ring chunks (the reducer thread of the pipelined ring runs for every ring step of the self-test's
    # 400 KB allreduce) and the log-depth bit reduction instead of the star
    for extra in ({}, {'HVD_RING_CHUNK_BYTES': '4096', 'HVD_BITS_TREE_MIN_RANKS': '2'}, {'HVD_TCP_ALLTOALL_CONCURRENT': '0', 'HVD_TCP_SPIN_US': '0'}):
        p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=dict(env, **extra), timeout=600)
        err = p.stderr.decode(errors='replace')
        if 'FATAL: ThreadSanitizer' in err and 'unexpected memory mapping' in err:
            pytest.skip('ThreadSanitizer cannot run in this container (ASLR / memory layout)')
        assert 'WARNING: ThreadSanitizer' not in err, (extra, err[-6000:])
        assert p.returncode == 0, (extra, p.returncode, p.stdout.decode()[-2000:], err[-2000:])


def test_native_selftest_under_address_and_ub_sanitizers():
    """The same self-test built with -fsanitize=address,undefined (found a memcpy(nullptr, p, 0) in the wire codec): no report
    of either sanitizer, in the default configuration and with tiny ring chunks + log-depth bit reduction."""
    if shutil.which('g++') is None:
        pytest.skip('no g++')
    from horovod_b200 import build
    try:
        exe = build.build_tsan_selftest(sanitizer='address,undefined')
    except Exception as e:  # noqa: BLE001 - toolchain without libasan / libubsan
        pytest.skip('cannot build with -fsanitize=address,undefined here: %s' % str(e)[-300:])
    env = dict(os.environ, ASAN_OPTIONS='detect_leaks=0 exitcode=67', UBSAN_OPTIONS='print_stacktrace=1', HOROVOD_LOG_LEVEL='error')
    for extra in ({}, {'HVD_RING_CHUNK_BYTES': '4096', 'HVD_BITS_TREE_MIN_RANKS': '2'}, {'HVD_TCP_ALLTOALL_CONCURRENT': '0', 'HVD_TCP_SPIN_US': '0'}):
        p = subprocess.run([exe], stdout=subprocess.PIPE, stderr=subprocess.PIPE, env=dict(env, **extra), timeout=900)
        err = p.stderr.decode(errors='replace')
        if 'AddressSanitizer' in err and ('Shadow memory range interleaves' in err or 'failed to allocate' in err):
            pytest.skip('AddressSanitizer cannot run in this container (address space layout)')
        assert 'runtime error:' not in err and 'ERROR: AddressSanitizer' not in err, (extra, err[-6000:])
        assert p.returncode == 0, (extra, p.returncode, p.stdout.decode()[-2000:], err[-2000:])


@pytest.mark.gpu
@pytest.mark.skipif(os.environ.get('HVD_RUN_COMPUTE_SANITIZER', '0') != '1',
                    reason='opt-in (HVD_RUN_COMPUTE_SANITIZER=1): memcheck instruments every kernel of the process, minutes per run')
def test_p2p_kernels_under_compute_sanitizer_memcheck():
    cs = shutil.which('compute-sanitizer') or '/usr/local/cuda/bin/compute-sanitizer'
    if not os.path.exists(cs):
        pytest.skip('compute-sanitizer not installed')
    script = os.path.join(REPO, 'tests', 'sanitizer_target.py')
    p = subprocess.run([cs, '--tool', 'memcheck', '--error-exitcode', '77', '--launch-timeout', '0', sys.executable, script],
                       stdout=subprocess.PIPE, stderr=subprocess.STDOUT, timeout=600, env=dict(os.environ, PYTHONPATH=REPO))
    out = p.stdout.decode(errors='replace')
    assert p.returncode == 0 and 'SANITIZER TARGET OK' in out and 'ERROR SUMMARY: 0 errors' in out, out[-5000:]

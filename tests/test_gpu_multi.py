"""Multi-GPU runs of the op matrix over the NVLink P2P kernels (and the NCCL baseline). Needs >= 2 GPUs:
`python -m pytest tests/test_gpu_multi.py -m gpu` on a machine with several GPUs."""
import pytest
import torch

from conftest import run_parallel

pytestmark = pytest.mark.gpu


def _ngpu():
    return torch.cuda.device_count() if torch.cuda.is_available() else 0


NEW_CHECKS = "graphed_step,adasum_stability,adasum_whole_model,hierarchical_allreduce,fake_hosts_topology"


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_ops_matrix_p2p(native_built):
    n = 2 if _ngpu() < 4 else (4 if _ngpu() < 8 else 8)
    # checks added after the last multi-GPU validation run in the gated test below
    rc, out = run_parallel("ops_worker.py", np=n, timeout=420, args=["--device", "cuda", "--skip", NEW_CHECKS],
                           env={"HOROVOD_LOG_LEVEL": "info"})
    assert "ALL OK" in out, out[-4000:]
    assert "symmetric team" in out, out[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_ops_matrix_new_checks(native_built):
    n = 2 if _ngpu() < 4 else (4 if _ngpu() < 8 else 8)
    rc, out = run_parallel("ops_worker.py", np=n, timeout=420, args=["--device", "cuda", "--only", NEW_CHECKS])
    assert "ALL OK" in out, out[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_ops_matrix_variants(native_built):
    for variant in ("oneshot", "twoshot"):
        rc, out = run_parallel("ops_worker.py", np=2, timeout=300, env={"HVD_ALLREDUCE_VARIANT": variant},
                               args=["--device", "cuda", "--only", "allreduce_sum_avg,allreduce_async_fused,allreduce_mixed_dtype_fusion,optimizer"])
        assert "ALL OK" in out, (variant, out[-3000:])


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_nccl_baseline_backend(native_built):
    rc, out = run_parallel("ops_worker.py", np=2, timeout=300, env={"HVD_GPU_BACKEND": "nccl"},
                           args=["--device", "cuda", "--only", "allreduce_sum_avg,allreduce_async_fused,optimizer"])
    assert "ALL OK" in out, out[-3000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_wire_compression_env(native_built):
    # bf16 on the wire (fp32 gradients cast inside the pack / unpack phases of the fused kernel)
    rc, out = run_parallel("ops_worker.py", np=2, timeout=300, env={"HVD_WIRE_DTYPE": "bf16"},
                           args=["--device", "cuda", "--only", "wire_dtype_env"])
    assert "ALL OK" in out, out[-3000:]


@pytest.mark.skipif(_ngpu() < 4, reason="needs >= 4 GPUs (2 fake hosts x 2)")
def test_hierarchical_allreduce_fake_hosts(native_built):
    """The box's GPUs presented as 2 hosts: intra-host reduce-scatter/allgather kernels + cross-host CPU transport."""
    n = 4 if _ngpu() < 8 else 8
    rc, out = run_parallel("ops_worker.py", np=n, timeout=300,
                           env={"HVD_TEST_FAKE_HOSTS": "2", "HOROVOD_LOG_LEVEL": "info", "HVD_SYMM_BUFFER_BYTES": str(2 << 20)},
                           args=["--device", "cuda", "--only", "fake_hosts_topology,hierarchical_allreduce,allreduce_sum_avg,"
                                 "allreduce_async_fused,allgather,broadcast,optimizer,barrier_join"])
    assert "ALL OK" in out, out[-4000:]
    assert "hierarchical allreduce over 2 hosts" in out, out[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_extra_reference_cases_cuda(native_built):
    rc, out = run_parallel("ops_worker_extra.py", np=2, timeout=300, args=["--device", "cuda"])
    assert "EXTRA ALL OK" in out, out[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_op_api_edge_cases_cuda(native_built):
    rc, out = run_parallel("edge_worker.py", np=2, timeout=300, args=["cuda"], env={"HOROVOD_FUSION_THRESHOLD": "65536"})
    assert "EDGE OK" in out, out[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_collectives_as_cuda_graph_nodes(native_built):
    """hvd.captured_allreduce_ inside torch.cuda.graph, hvd.GraphedStep with the gradient allreduces captured into the
    step's graph, model.zero_grad() with zero-copy buckets, hvd.join() against a cached zero-copy response."""
    n = 2 if _ngpu() < 4 else (4 if _ngpu() < 8 else 8)
    rc, out = run_parallel("graph_comm_worker.py", np=n, timeout=420, env={"HOROVOD_LOG_LEVEL": "warning"})
    assert "GRAPH COMM OK" in out, out[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_fused_collectives_and_large_allreduce(native_built):
    """Fused allgather / reducescatter / broadcast responses (one launch each) and the three-phase allreduce of large
    plain tensors."""
    n = 2 if _ngpu() < 4 else (4 if _ngpu() < 8 else 8)
    rc, out = run_parallel("ops_worker.py", np=n, timeout=420,
                           args=["--device", "cuda", "--only", "fused_other_collectives,allgather,broadcast,reducescatter,"
                                 "allreduce_sum_avg,allreduce_async_fused,large_allreduce"])
    assert "ALL OK" in out, out[-4000:]


@pytest.mark.skipif(_ngpu() < 2, reason="needs >= 2 GPUs")
def test_elastic_rank_failure_on_gpus(native_built, tmp_path):
    """Elastic recovery with the NVLink data plane (reference test/integration/test_elastic_torch.py:33-49): two workers
    on two GPUs of ONE peer-mapped team; rank 1 is SIGKILLed in the middle of epoch 1.  The survivor's collective (its
    kernel may be spinning at the flag barrier of a peer that no longer exists) must end through the abort flag, the job
    re-forms at size 1, restores the last commit and finishes."""
    from test_integration_elastic import _run_elastic
    rc, out, recs = _run_elastic(tmp_path, [(None, ['localhost:1', '127.0.0.1:1'])], 2, 1, 2,
                                 exit_schedule={'1,2': [1]}, exit_mode='kill', main_args=['--device', 'cuda'], timeout=400,
                                 env_extra={'HVD_TEST_ONE_HOST': '1', 'HVD_KERNEL_TIMEOUT_SECONDS': '15', 'HOROVOD_LOG_LEVEL': 'info'})
    done = recs[-1]
    assert done.get('done') and done['size'] == 1, (done, out[-3000:])
    sizes_by_epoch = {}
    for r in recs:
        if 'epoch' in r:
            sizes_by_epoch.setdefault(r['epoch'], set()).add(r['size'])
    assert sizes_by_epoch[0] == {2} and sizes_by_epoch[2] == {1}, sizes_by_epoch
    assert 'symmetric team of 2 GPUs' in out, out[-3000:]

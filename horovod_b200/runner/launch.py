"""`hvdrun` — the command line launcher.

    hvdrun -np 8 python train.py
    hvdrun -np 16 -H server1:8,server2:8 python train.py
    hvdrun -np 8 --min-np 4 --max-np 8 --host-discovery-script ./discover.sh python train_elastic.py

Role parity: horovod/runner/launch.py (parse_args :286, _run_static :596, _run_elastic :689, run_controller :747,
run_commandline :830).  Controllers: the native mesh (flag name `--gloo` kept for script compatibility), `--mpi`
(builds an mpirun command line) and `--jsrun` on LSF.
"""
import argparse
import logging
import os
import sys
import textwrap

import yaml

import horovod_b200
from horovod_b200.runner.common.util import config_parser, hosts, safe_shell_exec, secret, settings as hvd_settings
from horovod_b200.runner.util import cache, lsf, network


# Cached information of horovodrun functions be stored in this directory
CACHE_FOLDER = os.path.join(os.path.expanduser('~'), '.horovod_b200')
# Cache entries will be stale if they are older than this number of minutes
CACHE_STALENESS_THRESHOLD_MINUTES = 60
# Number of attempts for sshing into the hosts
SSH_ATTEMPTS = 5
SSH_CONNECT_TIMEOUT_S = 10


def check_all_hosts_ssh_successful(host_addresses, ssh_port=None, ssh_identity_file=None, fn_cache=None):
    """Checks that passwordless ssh works to every remote host (results cached on disk)."""
    from horovod_b200.runner.mesh_run import get_ssh_command
    from horovod_b200.runner.util import threads

    def exec_command(command):
        exit_code = 1
        output_msg = ''
        for _ in range(SSH_ATTEMPTS):
            from horovod_b200.runner.common.util import tiny_shell_exec
            res = tiny_shell_exec.execute(command)
            if res is not None:
                output_msg, exit_code = res
                if exit_code == 0:
                    break
        return exit_code, output_msg

    args_list = [[get_ssh_command('true', host=h, port=ssh_port, identity_file=ssh_identity_file,
                                  timeout_s=SSH_CONNECT_TIMEOUT_S)] for h in host_addresses]
    ssh_exit_codes = threads.execute_function_multithreaded(exec_command, args_list)
    ssh_successful_to_all_hosts = True
    for index, ssh_status in ssh_exit_codes.items():
        exit_code, output_msg = ssh_status[0], ssh_status[1]
        if exit_code != 0:
            print('ssh not successful for host {host}:\n{msg_output}'.format(host=host_addresses[index], msg_output=output_msg))
            ssh_successful_to_all_hosts = False
    if not ssh_successful_to_all_hosts:
        return False
    return True


def check_build(verbose):
    def get_check(value):
        return 'X' if value else ' '
    from horovod_b200.common.basics import HorovodBasics
    b = HorovodBasics()
    output = '''{verbose_newline}\
    horovod_b200 v{version}:

    Available Frameworks:
        [{tensorflow}] TensorFlow
        [{torch}] PyTorch
        [{mxnet}] MXNet

    Available Controllers:
        [{mpi}] MPI
        [{gloo}] Native mesh (TCP + shared memory; fills Gloo's role)

    Available Tensor Operations:
        [{p2p}] NVLink P2P (sm_90a one-shot / two-shot / NVLS kernels)
        [{nccl_ops}] NCCL (baseline)
        [{ddl_ops}] DDL
        [{ccl_ops}] CCL
        [{mpi_ops}] MPI
        [{gloo_ops}] Native CPU ops (shared-memory slots on one host, shm + rings across hosts, TCP ring / tree otherwise)\
    '''.format(verbose_newline='\n' if verbose else '', version=horovod_b200.__version__, tensorflow=get_check(False),
               torch=get_check(True), mxnet=get_check(False), mpi=get_check(b.mpi_built()), gloo=get_check(b.gloo_built()),
               p2p=get_check(b.p2p_built()), nccl_ops=get_check(b.nccl_built()), ddl_ops=get_check(b.ddl_built()),
               mpi_ops=get_check(b.mpi_built()), ccl_ops=get_check(b.ccl_built()), gloo_ops=get_check(b.gloo_built()))
    print(textwrap.dedent(output))
    os._exit(0)


def make_check_build_action(np_arg):
    class CheckBuildAction(argparse.Action):
        def __call__(self, parser, args, values, option_string=None):
            # If -cb is specified, make -np optional and run the check
            np_arg.required = False
            args.check_build = True
    return CheckBuildAction


def make_override_action(override_args):
    class StoreOverrideAction(argparse.Action):
        def __init__(self, option_strings, dest, default=None, type=None, choices=None, required=False, help=None):
            super(StoreOverrideAction, self).__init__(option_strings=option_strings, dest=dest, nargs=1, default=default,
                                                      type=type, choices=choices, required=required, help=help)

        def __call__(self, parser, args, values, option_string=None):
            override_args.add(self.dest)
            setattr(args, self.dest, values[0])
    return StoreOverrideAction


def make_override_bool_action(override_args, bool_value):
    class StoreOverrideBoolAction(argparse.Action):
        def __init__(self, option_strings, dest, required=False, help=None):
            super(StoreOverrideBoolAction, self).__init__(option_strings=option_strings, dest=dest, const=bool_value,
                                                          nargs=0, default=None, required=required, help=help)

        def __call__(self, parser, args, values, option_string=None):
            override_args.add(self.dest)
            setattr(args, self.dest, self.const)
    return StoreOverrideBoolAction


def make_override_true_action(override_args):
    return make_override_bool_action(override_args, True)


def make_override_false_action(override_args):
    return make_override_bool_action(override_args, False)


def make_deprecated_bool_action(override_args, bool_value, replacement_option):
    class StoreOverrideBoolAction(argparse.Action):
        def __init__(self, option_strings, dest, required=False, help=None):
            super(StoreOverrideBoolAction, self).__init__(option_strings=option_strings, dest=dest, const=bool_value,
                                                          nargs=0, default=None, required=required, help=help)

        def __call__(self, parser, args, values, option_string=None):
            sys.stderr.write('WARNING: %s is deprecated, use %s instead\n' % (option_string, replacement_option))
            override_args.add(self.dest)
            setattr(args, self.dest, self.const)
    return StoreOverrideBoolAction


def parse_args():
    override_args = set()
    parser = argparse.ArgumentParser(description='hvdrun: launch a horovod_b200 job (Horovod-compatible launcher).')
    parser.add_argument('-v', '--version', action='version', version=horovod_b200.__version__, help='Shows the version.')
    np_arg = parser.add_argument('-np', '--num-proc', action='store', dest='num_proc', type=int, required=not lsf.LSFUtils.using_lsf(),
                                 help='Total number of training processes. In elastic mode, the number of processes required '
                                      'before training can start.')
    parser.add_argument('-cb', '--check-build', action=make_check_build_action(np_arg), nargs=0,
                        help='Shows which frameworks and libraries have been built into this package.')
    parser.add_argument('--disable-cache', action='store_true', dest='disable_cache',
                        help='If the flag is not set, hvdrun will perform the initialization checks only once every 60 '
                             'minutes -- if the checks pass -- and cache the result.')
    parser.add_argument('--start-timeout', action='store', dest='start_timeout', type=int,
                        help='Workers must start and rendezvous within this many seconds (default 30; env HOROVOD_START_TIMEOUT).')
    parser.add_argument('--network-interface', '--network-interfaces', action='store', dest='nics',
                        help='Network interfaces that can be used for communication separated by comma.')
    parser.add_argument('--output-filename', action='store',
                        help='For the native mesh: writes rank.N/stdout and rank.N/stderr below this directory. For MPI: '
                             'forwarded to mpirun --output-filename.')
    parser.add_argument('--verbose', action='store_true', dest='verbose', help='If this flag is set, extra messages will be printed.')
    parser.add_argument('command', nargs=argparse.REMAINDER, help='Command to be executed.')
    parser.add_argument('--config-file', action='store', dest='config_file',
                        help='Path to YAML file containing runtime parameter configuration. Command line wins over the file.')

    group_ssh = parser.add_argument_group('SSH arguments')
    group_ssh.add_argument('-p', '--ssh-port', action='store', dest='ssh_port', type=int, help='SSH port on all the hosts.')
    group_ssh.add_argument('-i', '--ssh-identity-file', action='store', dest='ssh_identity_file', help='File on the driver from which the identity (private key) is read.')

    group_params = parser.add_argument_group('tuneable parameter arguments')
    group_params.add_argument('--fusion-threshold-mb', action=make_override_action(override_args), type=int,
                              help='Fusion buffer threshold in MB: maximum bytes fused into one collective (default 128).')
    group_params.add_argument('--cycle-time-ms', action=make_override_action(override_args), type=float,
                              help='Upper bound in ms on how long an idle rank waits before joining a negotiation cycle (default 1).')
    group_params.add_argument('--cache-capacity', action=make_override_action(override_args), type=int,
                              help='Maximum number of tensor names kept in the response cache (default 1024, 0 disables).')
    group_hier = group_params.add_mutually_exclusive_group()
    group_hier.add_argument('--hierarchical-allreduce', action=make_override_true_action(override_args),
                            help='Two-level (intra-node NVLink, inter-node TCP) allreduce for multi-node jobs.')
    group_hier.add_argument('--no-hierarchical-allreduce', dest='hierarchical_allreduce', action=make_override_false_action(override_args))
    group_torus = group_params.add_mutually_exclusive_group()
    group_torus.add_argument('--torus-allreduce', action=make_override_true_action(override_args),
                             help='2-D allreduce for multi-node jobs (here: the same two-level schedule as --hierarchical-allreduce).')
    group_torus.add_argument('--no-torus-allreduce', dest='torus_allreduce', action=make_override_false_action(override_args))
    group_hiera = group_params.add_mutually_exclusive_group()
    group_hiera.add_argument('--hierarchical-allgather', action=make_override_true_action(override_args))
    group_hiera.add_argument('--no-hierarchical-allgather', dest='hierarchical_allgather', action=make_override_false_action(override_args))
    group_params.add_argument('--thread-affinity', action=make_override_action(override_args), type=str,
                              help='Comma separated core ids: background thread of local rank i is pinned to the i-th entry.')
    group_params.add_argument('--num-nccl-streams', action=make_override_action(override_args), type=int)

    group_autotune = parser.add_argument_group('autotune arguments')
    ga = group_autotune.add_mutually_exclusive_group()
    ga.add_argument('--autotune', action=make_override_true_action(override_args),
                    help='Tune fusion threshold, cycle time and the NVLink kernel variant crossovers at runtime.')
    ga.add_argument('--no-autotune', dest='autotune', action=make_override_false_action(override_args))
    group_autotune.add_argument('--autotune-log-file', action=make_override_action(override_args), help='CSV log of the autotuner samples.')
    group_autotune.add_argument('--autotune-warmup-samples', action=make_override_action(override_args), type=int)
    group_autotune.add_argument('--autotune-steps-per-sample', action=make_override_action(override_args), type=int)
    group_autotune.add_argument('--autotune-bayes-opt-max-samples', action=make_override_action(override_args), type=int)
    group_autotune.add_argument('--autotune-gaussian-process-noise', action=make_override_action(override_args), type=float)

    group_elastic = parser.add_argument_group('elastic arguments')
    group_elastic.add_argument('--min-np', '--min-num-proc', action='store', dest='min_num_proc', type=int,
                               help='Minimum number of processes running for training to continue (default: -np).')
    group_elastic.add_argument('--max-np', '--max-num-proc', action='store', dest='max_num_proc', type=int,
                               help='Maximum number of training processes (default: -np).')
    group_elastic.add_argument('--slots-per-host', action='store', dest='slots', type=int,
                               help='Slots per discovered host when the discovery script does not print `host:slots`.')
    group_elastic.add_argument('--elastic-timeout', action='store', dest='elastic_timeout', type=int,
                               help='Seconds to wait for the required number of slots after a re-scale event (default 600).')
    group_elastic.add_argument('--reset-limit', action='store', dest='reset_limit', type=int,
                               help='Maximum number of resets (rank re-assignments) before the job is aborted.')
    group_elastic.add_argument('--blacklist-cooldown-range', action='store', dest='cooldown_range', type=int, nargs=2,
                               help='Range (in seconds) a failing host stays blacklisted; exponential back-off inside the range.')

    group_timeline = parser.add_argument_group('timeline arguments')
    group_timeline.add_argument('--timeline-filename', action=make_override_action(override_args), help='JSON file for the Horovod Timeline.')
    gt = group_timeline.add_mutually_exclusive_group()
    gt.add_argument('--timeline-mark-cycles', action=make_override_true_action(override_args))
    gt.add_argument('--no-timeline-mark-cycles', dest='timeline_mark_cycles', action=make_override_false_action(override_args))

    group_stall = parser.add_argument_group('stall check arguments')
    gs = group_stall.add_mutually_exclusive_group()
    gs.add_argument('--no-stall-check', action=make_override_true_action(override_args))
    gs.add_argument('--stall-check', dest='no_stall_check', action=make_override_false_action(override_args))
    group_stall.add_argument('--stall-check-warning-time-seconds', action=make_override_action(override_args), type=int)
    group_stall.add_argument('--stall-check-shutdown-time-seconds', action=make_override_action(override_args), type=int)

    group_lib = parser.add_argument_group('library arguments')
    gl = group_lib.add_mutually_exclusive_group()
    gl.add_argument('--mpi-threads-disable', action=make_override_true_action(override_args))
    gl.add_argument('--no-mpi-threads-disable', dest='mpi_threads_disable', action=make_override_false_action(override_args))
    group_lib.add_argument('--gloo-timeout-seconds', action=make_override_action(override_args), type=int,
                           help='Seconds a rank waits for its peers during bootstrap / rendezvous before giving up (default 60); when given, '
                                'a socket receive of a running job that makes no progress for this long fails as well.')
    group_lib.add_argument('--mpi-args', action='store', dest='mpi_args', help='Extra MPI arguments to pass to mpirun.')
    group_lib.add_argument('--tcp', action='store_true', dest='tcp_flag', help='If this flag is set, only TCP is used for communication.')
    group_lib.add_argument('--binding-args', action='store', dest='binding_args', help='Process binding arguments.')
    group_lib.add_argument('--gpu-backend', action=make_override_action(override_args), choices=['p2p', 'nccl', 'cpu'],
                           help='GPU data path: NVLink P2P kernels (default), NCCL baseline, or host staging.')
    group_lib.add_argument('--allreduce-variant', action=make_override_action(override_args), choices=['auto', 'oneshot', 'twoshot', 'nvls'])
    group_lib.add_argument('--wire-dtype', action=make_override_action(override_args), choices=['none', 'bf16', 'fp16'],
                           help='In-kernel compression of fp32 gradient sums on the wire.')
    group_lib.add_argument('--comm-ctas', action=make_override_action(override_args), type=int, help='CTAs per communication kernel.')
    group_lib.add_argument('--num-nccl-streams-deprecated', action='store', type=int, help=argparse.SUPPRESS)

    group_log = parser.add_argument_group('logging arguments')
    group_log.add_argument('--log-level', action=make_override_action(override_args), choices=config_parser.LOG_LEVELS,
                           help='Minimum level to log to stderr from the native runtime (default WARNING).')
    glh = group_log.add_mutually_exclusive_group()
    glh.add_argument('--log-hide-timestamp', '--log-without-timestamp', dest='log_hide_timestamp', action=make_override_true_action(override_args))
    glh.add_argument('--no-log-hide-timestamp', '--log-with-timestamp', dest='log_hide_timestamp', action=make_override_false_action(override_args))
    group_log.add_argument('-prefix-timestamp', '--prefix-output-with-timestamp', action='store_true', dest='prefix_output_with_timestamp',
                           help='Timestamp every line of the forwarded worker output.')

    group_hosts_parent = parser.add_argument_group('host arguments')
    group_hosts = group_hosts_parent.add_mutually_exclusive_group()
    group_hosts.add_argument('-H', '--hosts', action='store', dest='hosts',
                             help='List of host names and the number of available slots: host1:2,host2:4. Default: localhost:<np>.')
    group_hosts.add_argument('-hostfile', '--hostfile', action='store', dest='hostfile',
                             help='File with one `hostname slots=N` line per host.')
    group_hosts.add_argument('--host-discovery-script', action=make_override_action(override_args),
                             help='Elastic: executable that prints the currently available hosts (`host[:slots]` per line).')

    group_ctrl_parent = parser.add_argument_group('controller arguments')
    group_ctrl = group_ctrl_parent.add_mutually_exclusive_group()
    group_ctrl.add_argument('--gloo', action='store_true', dest='use_gloo', help='Run with the native mesh controller (default).')
    group_ctrl.add_argument('--mpi', action='store_true', dest='use_mpi', help='Launch through mpirun.')
    group_ctrl.add_argument('--jsrun', action='store_true', dest='use_jsrun', help='Launch through jsrun (LSF).')

    args = parser.parse_args()
    if args.config_file:
        with open(args.config_file, 'r') as f:
            config = yaml.load(f, Loader=yaml.FullLoader)
        config_parser.set_args_from_config(args, config, override_args)
    config_parser.validate_config_args(args)
    args.run_func = None
    if getattr(args, 'check_build', False):
        check_build(args.verbose)
    return args


def _is_elastic(args):
    return args.host_discovery_script is not None or args.min_num_proc is not None


def _build_settings(args, elastic=False):
    tmout = args.start_timeout if args.start_timeout else int(os.getenv('HOROVOD_START_TIMEOUT', '30'))
    nics = set(args.nics.split(',')) if args.nics else None
    return hvd_settings.Settings(verbose=2 if args.verbose else 0, ssh_port=args.ssh_port,
                                 ssh_identity_file=args.ssh_identity_file, extra_mpi_args=args.mpi_args,
                                 tcp_flag=args.tcp_flag, binding_args=args.binding_args, key=secret.make_secret_key(),
                                 start_timeout=tmout, num_proc=args.num_proc, hosts=getattr(args, 'hosts', None),
                                 output_filename=args.output_filename, run_func_mode=args.run_func is not None, nics=nics,
                                 elastic=elastic, prefix_output_with_timestamp=args.prefix_output_with_timestamp)


def _run_static(args):
    # horovodrun has to finish all the checks before this timeout runs out.
    if args.hostfile:
        args.hosts = hosts.parse_host_files(args.hostfile)
    if not args.hosts:
        if lsf.LSFUtils.using_lsf():
            args.hosts = ','.join('{host}:{np}'.format(host=host, np=lsf.LSFUtils.get_num_gpus()) for host in lsf.LSFUtils.get_compute_hosts())
        else:
            args.hosts = 'localhost:{np}'.format(np=args.num_proc)
    if args.num_proc is None:
        args.num_proc = sum(h.slots for h in hosts.parse_hosts(args.hosts))
    all_host_names, _ = hosts.parse_hosts_and_slots(args.hosts)
    settings = _build_settings(args)
    fn_cache = None
    if not args.disable_cache:
        params = ''
        if args.np if hasattr(args, 'np') else args.num_proc:
            params += str(args.num_proc) + ' '
        if args.hosts:
            params += str(args.hosts) + ' '
        if args.ssh_port:
            params += str(args.ssh_port)
        if args.ssh_identity_file:
            params += args.ssh_identity_file
        parameters_hash = __import__('hashlib').md5(params.encode('utf-8')).hexdigest()
        fn_cache = cache.Cache(CACHE_FOLDER, CACHE_STALENESS_THRESHOLD_MINUTES, parameters_hash)
    remote_host_names = network.filter_local_addresses(all_host_names)
    if remote_host_names:
        if settings.verbose >= 2:
            print('Checking ssh on all remote hosts.')
        check = fn_cache.use_cache()(check_all_hosts_ssh_successful) if fn_cache else check_all_hosts_ssh_successful
        if not check(remote_host_names, args.ssh_port, args.ssh_identity_file):
            raise RuntimeError('could not connect to some hosts via ssh')
        if settings.verbose >= 2:
            print('SSH was successful into all the remote hosts.')
    nics = settings.nics
    if remote_host_names and not nics:
        from horovod_b200.runner.driver import driver_service
        nics = driver_service.get_common_interfaces(settings, all_host_names, remote_host_names, fn_cache)
    if args.run_func:
        return _run_func_static(args, settings, nics)
    command = args.command
    _launch_job(args, settings, nics, command)
    return None


def _run_func_static(args, settings, nics):
    """Run-func mode: the pickled function travels through a KV store, results come back per rank."""
    from horovod_b200.runner.http.http_server import KVStoreServer
    import cloudpickle
    kvstore = KVStoreServer(verbose=settings.verbose)
    port = kvstore.start_server()
    driver_ip = network.get_driver_ip(nics)
    kvstore.put('runfunc', 'func', cloudpickle.dumps(args.run_func))
    command = [sys.executable, '-m', 'horovod_b200.runner.run_task', str(driver_ip), str(port)]
    try:
        _launch_job(args, settings, nics, command)
        results = [None] * args.num_proc
        for i in range(args.num_proc):
            raw = kvstore.get('runfunc_result', str(i))
            if raw is None:
                raise RuntimeError(f'hvdrun: rank {i} did not return a result')
            results[i] = cloudpickle.loads(raw)
        return results
    finally:
        kvstore.shutdown_server()


def _run_elastic(args):
    from horovod_b200.runner.elastic import discovery
    from horovod_b200.runner.mesh_run import elastic_run
    # construct host discovery component
    if args.host_discovery_script:
        disc = discovery.HostDiscoveryScript(args.host_discovery_script, args.slots)
    elif args.hosts:
        _, available_host_slots = hosts.parse_hosts_and_slots(args.hosts)
        if len(available_host_slots) < 2:
            print('Elastic training is running on a single fixed host: no fault tolerance against host failure.')
        disc = discovery.FixedHosts(available_host_slots)
    elif args.hostfile:
        _, available_host_slots = hosts.parse_hosts_and_slots(hosts.parse_host_files(args.hostfile))
        disc = discovery.FixedHosts(available_host_slots)
    else:
        raise ValueError('One of --host-discovery-script, --hosts, or --hostfile must be provided')
    settings = _build_settings(args, elastic=True)
    settings.discovery = disc
    settings.min_num_proc = args.min_num_proc or args.num_proc
    settings.max_num_proc = args.max_num_proc or args.num_proc
    settings.elastic_timeout = args.elastic_timeout or int(os.getenv('HOROVOD_ELASTIC_TIMEOUT', '600'))
    settings.reset_limit = args.reset_limit
    settings.cooldown_range = args.cooldown_range
    if args.use_mpi or args.use_jsrun:
        raise ValueError('elastic training is only supported with the native mesh controller')
    env = os.environ.copy()
    config_parser.set_env_from_args(env, args)
    os.environ.update({k: v for k, v in env.items() if k.startswith(('HOROVOD_', 'HVD_'))})
    if not args.run_func:
        return elastic_run(settings, env, args.command, disc, settings.min_num_proc, settings.max_num_proc,
                           settings.elastic_timeout, settings.reset_limit, settings.cooldown_range)
    # run-func mode: the pickled function travels through a KV store; every worker of the FINAL round uploads its return
    # value under the rank it held then (hvd.init rewrites HOROVOD_RANK on every elastic reset)
    from horovod_b200.runner.http.http_server import KVStoreServer
    import cloudpickle
    kvstore = KVStoreServer(verbose=settings.verbose)
    port = kvstore.start_server()
    try:
        kvstore.put('runfunc', 'func', cloudpickle.dumps(args.run_func))
        command = [args.executable or sys.executable, '-m', 'horovod_b200.runner.run_task', str(network.get_driver_ip(settings.nics)), str(port)]
        elastic_run(settings, env, command, disc, settings.min_num_proc, settings.max_num_proc,
                    settings.elastic_timeout, settings.reset_limit, settings.cooldown_range)
        results = []
        while True:
            raw = kvstore.get('runfunc_result', str(len(results)))
            if raw is None:
                break
            results.append(cloudpickle.loads(raw))
        if len(results) < settings.min_num_proc:
            raise RuntimeError('hvdrun: only %d of at least %d workers returned a result' % (len(results), settings.min_num_proc))
        return results
    finally:
        kvstore.shutdown_server()


def is_gloo_used(use_gloo=None, use_mpi=None, use_jsrun=None):
    # determines whether run_controller will run gloo in the case all flags are None
    return use_gloo or (not use_mpi and not use_jsrun)


def run_controller(use_gloo, gloo_run, use_mpi, mpi_run, use_jsrun, js_run, verbosity):
    """Picks the launcher back end (reference launch.py:747-779)."""
    from horovod_b200.runner import mpi_run as mpi_mod
    if use_gloo:
        gloo_run()
    elif use_mpi:
        if not mpi_mod.mpi_available():
            raise ValueError('MPI support has not been found (no mpirun on PATH); use the native mesh controller.')
        mpi_run()
    elif use_jsrun:
        if not lsf.LSFUtils.using_lsf():
            raise ValueError('jsrun is only available inside an LSF allocation.')
        js_run()
    else:
        if lsf.LSFUtils.using_lsf() and mpi_mod.mpi_available():
            js_run()
        else:
            gloo_run()


def _launch_job(args, settings, nics, command):
    env = os.environ.copy()
    config_parser.set_env_from_args(env, args)
    # workers inherit the launcher's environment when spawned locally
    os.environ.update({k: v for k, v in env.items() if k.startswith(('HOROVOD_', 'HVD_'))})

    def gloo_run_fn():
        from horovod_b200.runner.mesh_run import mesh_run
        driver_ip = network.get_driver_ip(nics) if network.filter_local_addresses(hosts.parse_hosts_and_slots(settings.hosts)[0]) else '127.0.0.1'
        mesh_run(settings, nics, env, driver_ip, command)

    def mpi_run_fn():
        from horovod_b200.runner.mpi_run import mpi_run
        mpi_run(settings, nics, env, command)

    def js_run_fn():
        from horovod_b200.runner.js_run import js_run
        js_run(settings, nics, env, command)

    run_controller(args.use_gloo, gloo_run_fn, args.use_mpi, mpi_run_fn, args.use_jsrun, js_run_fn, args.verbose)


def _run(args):
    # if hosts are not specified, either parse from hostfile, or default as localhost
    if _is_elastic(args):
        return _run_elastic(args)
    return _run_static(args)


def run_commandline():
    args = parse_args()
    if not args.command:
        sys.stderr.write('hvdrun: no command given\n')
        sys.exit(2)
    try:
        _run(args)
    except (RuntimeError, ValueError) as e:
        sys.stderr.write(str(e) + '\n')
        sys.exit(1)


if __name__ == '__main__':
    run_commandline()

"""Per-node launcher: spawn one worker per local GPU with RANK/LOCAL_RANK/WORLD_SIZE/MASTER_* set, babysit them,
tear the whole tree down when one dies.  Reference: ``launcher/launch.py`` (``main :133``)."""
import argparse
import base64
import json
import os
import signal
import subprocess
import sys
import time
from collections import defaultdict

from deepspeed_b200.utils.logging import logger

PID_FILE_BASEPATH = "/tmp"


def parse_args(argv=None):
    p = argparse.ArgumentParser(description="DeepSpeed-H100 per-node process launcher")
    p.add_argument("--node_rank", type=int, default=0)
    p.add_argument("--master_addr", default="127.0.0.1", type=str)
    p.add_argument("--master_port", default=29500, type=int)
    p.add_argument("--world_info", default="None", type=str, help="base64(json {host: [gpu ids]})")
    p.add_argument("--module", action="store_true")
    p.add_argument("--no_python", action="store_true")
    p.add_argument("--enable_elastic_training", action="store_true")
    p.add_argument("--min_elastic_nodes", type=int, default=-1)
    p.add_argument("--max_elastic_nodes", type=int, default=-1)
    p.add_argument("--no_local_rank", action="store_true")
    p.add_argument("--save_pid", type=int, default=0, nargs="?", const=1)
    p.add_argument("--enable_each_rank_log", default="None", type=str)
    p.add_argument("--bind_cores_to_rank", action="store_true")
    p.add_argument("--bind_core_list", type=str, default=None)
    p.add_argument("training_script", type=str)
    p.add_argument("training_script_args", nargs=argparse.REMAINDER)
    return p.parse_args(argv)


def terminate_process_tree(pid):
    """Kill exactly the subtree rooted at ``pid`` (children first)."""
    try:
        import psutil
        parent = psutil.Process(pid)
        procs = parent.children(recursive=True) + [parent]
        for p in procs:
            try:
                p.terminate()
            except psutil.NoSuchProcess:
                pass
        _, alive = psutil.wait_procs(procs, timeout=30)
        for p in alive:
            p.kill()
    except Exception:
        try:
            os.kill(pid, signal.SIGTERM)
        except ProcessLookupError:
            pass


def _core_binding(local_rank, n_local, core_list):
    """numactl prefix pinning this rank to an equal share of the host cores (feeds the CPU-offload optimizer)."""
    import shutil
    if shutil.which("numactl") is None:
        return []
    if core_list:
        cores = []
        for part in core_list.split(","):
            a, _, b = part.partition("-")
            cores += list(range(int(a), int(b or a) + 1))
    else:
        cores = sorted(os.sched_getaffinity(0))
    per = max(1, len(cores) // n_local)
    mine = cores[local_rank * per:(local_rank + 1) * per]
    return ["numactl", "-C", ",".join(map(str, mine))] if mine else []


def build_rank_env_and_cmds(args, world_info):
    hosts = list(world_info.keys())
    node = hosts[args.node_rank]
    local_gpus = world_info[node]
    offsets, total = {}, 0
    for h in hosts:
        offsets[h] = total
        total += len(world_info[h])
    base_env = os.environ.copy()
    base_env["MASTER_ADDR"] = args.master_addr
    base_env["MASTER_PORT"] = str(args.master_port)
    base_env["WORLD_SIZE"] = str(total)
    base_env["CROSS_RANK"] = str(args.node_rank)
    base_env["CROSS_SIZE"] = str(len(hosts))
    base_env["LOCAL_SIZE"] = base_env["LOCAL_WORLD_SIZE"] = str(len(local_gpus))
    base_env.setdefault("CUDA_VISIBLE_DEVICES", ",".join(map(str, local_gpus)))
    out = []
    for lr, gpu in enumerate(local_gpus):
        env = dict(base_env)
        env["RANK"] = str(offsets[node] + lr)
        env["LOCAL_RANK"] = str(lr)
        cmd = []
        if args.bind_cores_to_rank:
            cmd += _core_binding(lr, len(local_gpus), args.bind_core_list)
            env.setdefault("OMP_NUM_THREADS", str(max(1, len(os.sched_getaffinity(0)) // len(local_gpus))))
        if not args.no_python:
            cmd += [sys.executable, "-u"]
            if args.module:
                cmd.append("-m")
        elif args.module:
            raise ValueError("Don't use both the '--no_python' flag and the '--module' flag at the same time.")
        cmd.append(args.training_script)
        if not args.no_local_rank:
            cmd.append(f"--local_rank={lr}")
        cmd += args.training_script_args
        out.append((env, cmd))
    return out


def main(argv=None):
    args = parse_args(argv)
    if args.world_info == "None":
        raise ValueError("world_info can not be None")
    world_info = json.loads(base64.urlsafe_b64decode(args.world_info))
    logger.info(f"WORLD INFO DICT: {world_info}")
    if args.enable_elastic_training:
        return _elastic_main(args, world_info)
    launches = build_rank_env_and_cmds(args, world_info)
    log_dir = None if args.enable_each_rank_log == "None" else args.enable_each_rank_log
    if log_dir:
        os.makedirs(log_dir, exist_ok=True)
    procs = []
    for env, cmd in launches:
        if log_dir:
            f = open(os.path.join(log_dir, f"rank{env['RANK']}.log"), "w")
            p = subprocess.Popen(cmd, env=env, stdout=f, stderr=f)
        else:
            p = subprocess.Popen(cmd, env=env)
        logger.info(f"process {p.pid} spawned with command: {cmd}")
        procs.append(p)
    pid_file = None
    if args.save_pid:
        pid_file = os.path.join(PID_FILE_BASEPATH, f"{args.save_pid}.deepspeed")
        with open(pid_file, "w") as f:
            json.dump([p.pid for p in procs] + [os.getpid()], f)

    def _sig(signum, frame):
        for p in procs:
            logger.info(f"Killing subprocess {p.pid}")
            terminate_process_tree(p.pid)
        if pid_file and os.path.isfile(pid_file):
            os.remove(pid_file)
        sys.exit(1)

    signal.signal(signal.SIGINT, _sig)
    signal.signal(signal.SIGTERM, _sig)
    alive = set(procs)
    rc_final = 0
    while alive:
        done = [p for p in alive if p.poll() is not None]
        for p in done:
            alive.discard(p)
            if p.returncode != 0:
                logger.error(f"{p.args} exits with return code = {p.returncode}")
                rc_final = p.returncode
                for q in alive:
                    terminate_process_tree(q.pid)
                alive.clear()
                break
            logger.info(f"Process {p.pid} exits successfully.")
        time.sleep(0.5)
    if pid_file and os.path.isfile(pid_file):
        os.remove(pid_file)
    sys.exit(rc_final)


def _elastic_main(args, world_info):
    from torch.distributed.elastic.agent.server.api import WorkerSpec
    from torch.distributed.elastic.rendezvous import RendezvousParameters
    import torch.distributed.elastic.rendezvous.registry as rdzv_registry
    from deepspeed_b200.elasticity import DSElasticAgent
    hosts = list(world_info.keys())
    n_local = len(world_info[hosts[args.node_rank]])
    lo = args.min_elastic_nodes if args.min_elastic_nodes > 0 else 1
    hi = args.max_elastic_nodes if args.max_elastic_nodes > 0 else len(hosts)
    params = RendezvousParameters(backend="c10d", endpoint=f"{args.master_addr}:{args.master_port}",
                                  run_id=os.environ.get("ELASTIC_RUN_ID", "123456789"), min_nodes=lo, max_nodes=hi)
    cmd = [sys.executable, "-u"] + (["-m"] if args.module else []) + [args.training_script] + args.training_script_args
    spec = WorkerSpec(role="trainer", local_world_size=n_local, entrypoint=cmd[0], args=tuple(cmd[1:]),
                      rdzv_handler=rdzv_registry.get_rendezvous_handler(params), max_restarts=100, monitor_interval=5,
                      master_addr=args.master_addr, master_port=args.master_port)
    agent = DSElasticAgent(spec, dict(os.environ))
    agent.run()


if __name__ == "__main__":
    main()

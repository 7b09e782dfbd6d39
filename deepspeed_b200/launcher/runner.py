"""``deepspeed`` command: resolve resources (hostfile, --include/--exclude, --num_nodes/--num_gpus), then either
exec the per-node launcher locally or fan out through a multi-node runner (pdsh / mpi flavours / slurm).

CLI parity: reference ``launcher/runner.py`` (``parse_args :48``, ``fetch_hostfile :213``,
``parse_resource_filter :293``, ``encode_world_info :384``, ``main :419``).
"""
import argparse
import base64
import collections
import json
import os
import re
import shlex
import signal
import subprocess
import sys
from copy import deepcopy
from typing import Dict, List, Tuple

from deepspeed_b200.utils.logging import logger
from . import constants as K
from .multinode_runner import RUNNERS


def parse_args(args=None):
    p = argparse.ArgumentParser(description="DeepSpeed-H100 runner: launch single- or multi-node training jobs")
    p.add_argument("-H", "--hostfile", type=str, default=K.DLTS_HOSTFILE,
                   help="Hostfile path (MPI style): lines of `hostname slots=N`")
    p.add_argument("-i", "--include", type=str, default="",
                   help="Resources to use, e.g. `worker-0@worker-1:0,2` = all of worker-0, GPUs 0 and 2 of worker-1")
    p.add_argument("-e", "--exclude", type=str, default="", help="Resources NOT to use (mutually exclusive with -i)")
    p.add_argument("--num_nodes", type=int, default=-1)
    p.add_argument("--min_elastic_nodes", type=int, default=-1)
    p.add_argument("--max_elastic_nodes", type=int, default=-1)
    p.add_argument("--num_gpus", "--num_accelerators", type=int, default=-1)
    p.add_argument("--master_port", default=K.TORCH_DISTRIBUTED_DEFAULT_PORT, type=int)
    p.add_argument("--master_addr", default="", type=str)
    p.add_argument("--node_rank", default=-1, type=int)
    p.add_argument("--launcher", default=K.PDSH_LAUNCHER, type=str,
                   help="multi-node backend: pdsh, openmpi, mpich, impi, slurm, mvapich")
    p.add_argument("--launcher_args", default="", type=str)
    p.add_argument("--module", action="store_true", help="run the user script as `python -m`")
    p.add_argument("--no_python", action="store_true", help="exec the user script directly")
    p.add_argument("--no_local_rank", action="store_true", help="do not pass --local_rank to the user script")
    p.add_argument("--no_ssh", action="store_true", help="launch on every node independently (needs --node_rank)")
    p.add_argument("--no_ssh_check", action="store_true")
    p.add_argument("--force_multi", action="store_true")
    p.add_argument("--save_pid", action="store_true")
    p.add_argument("--enable_each_rank_log", default="None", type=str)
    p.add_argument("--autotuning", default="", choices=["tune", "run", ""], type=str)
    p.add_argument("--elastic_training", action="store_true")
    p.add_argument("--bind_cores_to_rank", action="store_true")
    p.add_argument("--bind_core_list", type=str, default=None)
    p.add_argument("--ssh_port", type=int, default=None)
    p.add_argument("user_script", type=str, help="training script, followed by its arguments")
    p.add_argument("user_args", nargs=argparse.REMAINDER)
    return p.parse_args(args=args)


def fetch_hostfile(path):
    if not os.path.isfile(path):
        logger.warning("Unable to find hostfile, will proceed with training with local resources only.")
        return None
    with open(path) as f:
        return _parse_hostfile(f.readlines())


_HOST_RE = re.compile(r"^(\S+)\s+slots=(\d+)")


def _parse_hostfile(lines):
    pool = collections.OrderedDict()
    for raw in lines:
        line = raw.strip()
        if not line or line.startswith("#"):
            continue
        m = _HOST_RE.match(line)
        if not m:
            raise ValueError(f"Hostfile contains a bad entry: {line}, unable to proceed with training")
        host, slots = m.group(1), int(m.group(2))
        if host in pool:
            raise ValueError(f"Hostfile contains multiple entries for {host}, unable to proceed with training")
        pool[host] = slots
    if not pool:
        raise ValueError("Hostfile is empty or not formatted correctly, unable to proceed with training.")
    return pool


def _dedup(xs):
    seen, out = set(), []
    for x in xs:
        if x not in seen:
            seen.add(x)
            out.append(x)
    return out


def parse_node_config(node_config: str) -> Tuple[str, List[int]]:
    host, _, slots = node_config.partition(":")
    if not slots:
        return host, []
    return host, [int(s) for s in slots.split(",")]


def parse_node_config_list(items: List[str]) -> Dict[str, List[int]]:
    return {h: s for h, s in (parse_node_config(i) for i in items)}


def parse_resource_filter(host_info, include_str="", exclude_str=""):
    """``host_info``: {host: [slot ids]}.  String grammar: NODE_SPEC[@NODE_SPEC...], NODE_SPEC = NAME[:SLOT[,SLOT...]]"""
    if include_str and exclude_str:
        raise ValueError("include_str and exclude_str are mutually exclusive.")
    if not include_str and not exclude_str:
        return host_info
    spec = include_str or exclude_str
    result = collections.OrderedDict() if include_str else deepcopy(host_info)
    for node in spec.split("@"):
        host, slots = parse_node_config(node)
        if host not in host_info:
            raise ValueError(f"Hostname '{host}' not found in hostfile")
        for s in slots:
            if s not in host_info[host]:
                raise ValueError(f"No slot '{s}' specified on host '{host}'")
        if include_str:
            result[host] = _dedup(result.get(host, []) + (slots or list(host_info[host])))
        elif slots:
            result[host] = [s for s in result[host] if s not in slots]
        else:
            result.pop(host, None)
    ordered = collections.OrderedDict()
    for h in host_info:  # keep hostfile order
        if h in result and result[h]:
            ordered[h] = sorted(_dedup(result[h]))
    return ordered


def parse_inclusion_exclusion(resource_pool, inclusion, exclusion):
    active = collections.OrderedDict((h, list(range(n))) for h, n in resource_pool.items())
    return parse_resource_filter(active, include_str=inclusion, exclude_str=exclusion)


def encode_world_info(world_info):
    return base64.urlsafe_b64encode(json.dumps(world_info).encode("utf-8")).decode("utf-8")


def decode_world_info(s):
    return json.loads(base64.urlsafe_b64decode(s))


def parse_num_nodes(str_num_nodes: str, elastic_training: bool):
    parts = str(str_num_nodes).split(":")
    if len(parts) == 1:
        return int(parts[0]), -1
    if len(parts) == 2 and elastic_training:
        lo, hi = int(parts[0]), int(parts[1])
        if lo <= 0 or hi < lo:
            raise RuntimeError("MIN:MAX format of num_nodes requires 0 < MIN <= MAX")
        return lo, hi
    if len(parts) == 2:
        raise RuntimeError("MIN:MAX format is only supported in elastic training")
    raise RuntimeError(f"num_nodes {str_num_nodes} is not in MIN:MAX format")


def _local_gpu_count():
    try:
        import torch
        n = torch.cuda.device_count()
    except Exception:
        n = 0
    if n == 0:
        vis = os.environ.get("CUDA_VISIBLE_DEVICES")
        if vis:
            n = len([v for v in vis.split(",") if v])
    return n


def run_autotuning(args, active_resources):
    from deepspeed_b200.autotuning import Autotuner
    tuner = Autotuner(args, active_resources)
    logger.info("[Start] Running autotuning")
    tuner.tune()
    tuner.print_tuning_results()
    logger.info("[End] Running autotuning")
    tuner.write_optimal_config()
    if args.autotuning == "run":
        tuner.run_after_tuning()


def build_launch_cmd(args, world_info_b64, node_rank=0):
    cmd = [sys.executable, "-u", "-m", "deepspeed_b200.launcher.launch", f"--world_info={world_info_b64}",
           f"--master_addr={args.master_addr}", f"--master_port={args.master_port}", f"--node_rank={node_rank}"]
    for flag in ("no_python", "module", "no_local_rank", "save_pid", "bind_cores_to_rank"):
        if getattr(args, flag):
            cmd.append(f"--{flag}")
    if args.enable_each_rank_log != "None":
        cmd.append(f"--enable_each_rank_log={args.enable_each_rank_log}")
    if args.bind_core_list:
        cmd.append(f"--bind_core_list={args.bind_core_list}")
    if args.elastic_training:
        cmd += ["--enable_elastic_training", f"--max_elastic_nodes={args.max_elastic_nodes}",
                f"--min_elastic_nodes={args.min_elastic_nodes}"]
    return cmd + [args.user_script] + list(args.user_args)


def main(args=None):
    args = parse_args(args)
    if (args.num_nodes >= 0 or args.num_gpus >= 0) and (args.include != "" or args.exclude != ""):
        raise ValueError("Cannot specify num_nodes/gpus with include/exclude")
    if args.elastic_training:
        assert args.master_addr != "", "Master Addr is required when elastic training is enabled"
    resource_pool = fetch_hostfile(args.hostfile)
    if not resource_pool and (args.include or args.exclude):
        # single node: filters apply to localhost
        pass
    multi_node = bool(resource_pool) and (len(resource_pool) > 1 or args.force_multi)
    if not resource_pool:
        n = _local_gpu_count()
        if n == 0:
            raise RuntimeError("Unable to proceed, no GPU resources available")
        resource_pool = collections.OrderedDict(localhost=n)
        args.master_addr = args.master_addr or "127.0.0.1"
    active = parse_inclusion_exclusion(resource_pool, args.include, args.exclude)
    if args.num_nodes > 0:
        active = collections.OrderedDict(list(active.items())[:args.num_nodes])
    if args.num_gpus > 0:
        active = collections.OrderedDict((h, s[:args.num_gpus]) for h, s in active.items())
    multi_node = multi_node and len(active) > 1 or args.force_multi and "localhost" not in active
    if not args.master_addr:
        first = next(iter(active))
        if multi_node and not args.no_ssh:
            ssh = ["ssh"] + (["-p", str(args.ssh_port)] if args.ssh_port else []) + [first, "hostname -I"]
            out = subprocess.check_output(ssh).decode("utf-8").split()
            args.master_addr = out[0]
        else:
            args.master_addr = "127.0.0.1"
    if args.autotuning:
        run_autotuning(args, active)
        return
    world_info = encode_world_info(active)
    env = os.environ.copy()
    kill_cmd = None
    if args.elastic_training:
        cfg = _find_ds_config(args.user_args)
        if cfg:
            with open(cfg) as f:
                env["DEEPSPEED_ELASTICITY_CONFIG"] = json.dumps(json.load(f).get("elasticity", {}))
    if not multi_node or args.no_ssh:
        node_rank = max(args.node_rank, 0)
        cmd = build_launch_cmd(args, world_info, node_rank)
    else:
        cls = RUNNERS.get(args.launcher.lower())
        if cls is None:
            raise NotImplementedError(f"Unknown launcher {args.launcher}")
        runner = cls(args, world_info, active)
        if not runner.backend_exists():
            raise RuntimeError(f"launcher '{args.launcher}' not installed.")
        for var, val in os.environ.items():
            if any(var.startswith(p) for p in K.EXPORT_ENVS):
                runner.add_export(var, val)
        for d in K.DEEPSPEED_ENVIRONMENT_PATHS:
            f = os.path.join(os.path.expanduser(d), K.DEEPSPEED_ENVIRONMENT_NAME)
            if os.path.isfile(f):
                with open(f) as fh:
                    for line in fh:
                        if "=" in line:
                            k, v = line.strip().split("=", 1)
                            runner.add_export(k, v)
        got = runner.get_cmd(env, active)
        if isinstance(got, tuple):  # pdsh: (command, what to run on the workers on interrupt, environment)
            cmd, kill_cmd, env = got
        else:
            cmd = got
    logger.info(f"cmd = {' '.join(map(shlex.quote, cmd))}")
    proc = subprocess.Popen(cmd, env=env)

    def _forward(sig, frame):
        proc.send_signal(sig)
        if kill_cmd is not None:
            try:
                subprocess.Popen(kill_cmd, env=env).wait(timeout=30)
            except Exception:
                pass
        try:
            proc.wait(timeout=30)
        except subprocess.TimeoutExpired:
            proc.kill()
        sys.exit(1)

    signal.signal(signal.SIGINT, _forward)
    signal.signal(signal.SIGTERM, _forward)
    proc.wait()
    if proc.returncode != 0:
        sys.exit(proc.returncode)


def _find_ds_config(user_args):
    for i, a in enumerate(user_args):
        if a in ("--deepspeed_config", "--deepspeed-config") and i + 1 < len(user_args):
            return user_args[i + 1]
        if a.startswith("--deepspeed_config="):
            return a.split("=", 1)[1]
    return None


if __name__ == "__main__":
    main()

"""Autotuner: find the ZeRO stage / micro-batch size / ZeRO knobs that maximise throughput (or minimise latency).

Flow parity with reference ``autotuning/autotuner.py`` (``tune :404``): (1) model-info profiling run, (2) for each
ZeRO stage that fits in memory (estimator below), sweep micro-batch sizes, (3) tune the stage's knob space with
the chosen tuner around the best micro-batch size, (4) write the optimal config + a results table.  Memory
arithmetic uses H100's 80 GB HBM via ``torch.cuda.mem_get_info`` when a GPU is visible.
"""
import copy
import json
import os
import shutil

from deepspeed_b200.utils.logging import logger
from . import constants as K
from .config import DeepSpeedAutotuningConfig
from .scheduler import ResourceManager
from .tuner import GridSearchTuner, ModelBasedTuner, RandomTuner
from .utils import canonical_name, get_all_configs, memory_to_string, number_to_string, replace_dict

ZERO_SPACES = {0: K.DEFAULT_TUNING_SPACE_ZERO_0, 1: K.DEFAULT_TUNING_SPACE_ZERO_1, 2: K.DEFAULT_TUNING_SPACE_ZERO_2,
               3: K.DEFAULT_TUNING_SPACE_ZERO_3}


class Autotuner:

    def __init__(self, args, active_resources, runner=None):
        self.args = args
        self.user_config = self._get_user_config(args.user_args)
        assert self.user_config is not None, "DeepSpeed configuration is not provided"
        self.autotuning_config = DeepSpeedAutotuningConfig(**(self.user_config.get(K.AUTOTUNING) or {}))
        self.results_dir, self.exps_dir = self.autotuning_config.results_dir, self.autotuning_config.exps_dir
        if self.autotuning_config.overwrite:
            for d in (self.results_dir, self.exps_dir):
                shutil.rmtree(d, ignore_errors=True)
        os.makedirs(self.results_dir, exist_ok=True)
        os.makedirs(self.exps_dir, exist_ok=True)
        self.exp_num_nodes = len(active_resources)
        self.exp_num_gpus = min(len(v) for v in active_resources.values())
        self.rm = ResourceManager(args, list(active_resources.keys()), self.exp_num_gpus, self.results_dir, self.exps_dir,
                                  self.autotuning_config.arg_mappings, runner=runner)
        self.records = {}
        self.optimal_cmd = None
        self.optimal_ds_config = None
        self.model_info = self.autotuning_config.model_info

    # ---- config plumbing
    def _get_user_config(self, user_args):
        path = None
        for i, a in enumerate(user_args):
            if a in ("--deepspeed_config", "--deepspeed-config") and i + 1 < len(user_args):
                path = user_args[i + 1]
            elif a.startswith("--deepspeed_config="):
                path = a.split("=", 1)[1]
        if path is None:
            return None
        assert os.path.isfile(path), f"DeepSpeed configuration file: {path} is not an existing file"
        self.user_config_path = path
        with open(path) as f:
            return json.load(f)

    def metric(self):
        return self.autotuning_config.metric

    def fast_enabled(self):
        return self.autotuning_config.fast

    def mp_size(self):
        return self.autotuning_config.mp_size

    def get_gpu_memory_info(self):
        try:
            import torch
            if torch.cuda.is_available():
                return torch.cuda.get_device_properties(0).total_memory
        except Exception:
            pass
        return 80 * (1 << 30)

    def get_model_num_params(self):
        return (self.model_info or {}).get(K.MODEL_INFO_NUM_PARAMS)

    def get_instantiation_memory_required_per_gpu(self, zero_stage):
        """params(2B) + grads(2B) + optimizer(12B: fp32 master + 2 moments), divided per the stage's sharding."""
        n = self.get_model_num_params() or 0
        g = self.exp_num_gpus * self.exp_num_nodes // self.mp_size()
        p, gr, o = 2 * n, 2 * n, 12 * n
        if zero_stage >= 1:
            o /= g
        if zero_stage >= 2:
            gr /= g
        if zero_stage >= 3:
            p /= g
        return (p + gr + o) / self.mp_size()

    # ---- phases
    def model_info_profile_run(self):
        if self.model_info and self.model_info.get(K.MODEL_INFO_NUM_PARAMS):
            return self.model_info
        cfg = copy.deepcopy(self.user_config)
        replace_dict(cfg, K.DEFAULT_MIN_MEM_CONFIG)
        cfg.setdefault(K.AUTOTUNING, {})["model_info"] = {K.MODEL_INFO_PROFILE: True}
        exp = {"name": "profile_model_info", "ds_config": cfg, "num_gpus": self.exp_num_gpus, "num_nodes": self.exp_num_nodes}
        self.rm.schedule_experiments_dicts([exp])
        self.rm.run()
        p = os.path.join(exp["result_dir"], "model_info.json")
        if os.path.exists(p):
            with open(p) as f:
                self.model_info = json.load(f)
        self.rm.clear()
        return self.model_info

    def _mbs_candidates(self, stage):
        c = self.autotuning_config
        lo, hi = c.min_train_micro_batch_size_per_gpu, c.max_train_micro_batch_size_per_gpu
        user = self.user_config.get("train_micro_batch_size_per_gpu")
        if isinstance(user, int):
            return [user]
        out, m = [], max(1, lo)
        while m <= hi and len(out) < max(1, c.num_tuning_micro_batch_sizes):
            out.append(m)
            m *= 2
        return out

    def _exp(self, space_name, ds_config):
        name = canonical_name(ds_config, ["stage", "train_micro_batch_size_per_gpu", "overlap_comm", "b200_unit_prefetch",
                                          "reduce_bucket_size", "stage3_param_persistence_threshold"], prefix=space_name)
        return {"name": name, "ds_config": ds_config, "num_gpus": self.exp_num_gpus, "num_nodes": self.exp_num_nodes}

    def tune_space(self, stage):
        space_name = f"{K.TUNING_MICRO_BATCH_SIZE_PREFIX}{stage}"
        base = copy.deepcopy(self.user_config)
        base.pop(K.AUTOTUNING, None)
        # 1) micro-batch sweep with the first value of every knob
        from .utils import get_first_config
        first = get_first_config(ZERO_SPACES[stage])
        best_mbs, best_val = None, None
        for mbs in self._mbs_candidates(stage):
            cfg = replace_dict(copy.deepcopy(base), first)
            cfg["train_micro_batch_size_per_gpu"] = mbs
            cfg.pop("train_batch_size", None)
            exp = self._exp(space_name, cfg)
            self.rm.schedule_experiments_dicts([exp])
            self.rm.run()
            val = self.rm.metric_of(exp, self.metric())
            self.update_records(space_name, exp, val, 1)
            self.rm.clear()
            if val is None:
                break  # larger batches will not fit either
            if best_val is None or (val < best_val if self.metric() == "latency" else val > best_val):
                best_mbs, best_val = mbs, val
            elif self.fast_enabled():
                break  # throughput plateaued
        if best_mbs is None:
            return None
        if self.fast_enabled():
            return self.get_best_space_record(space_name)
        # 2) knob space around the best micro batch
        exps = []
        for cfg_knobs in get_all_configs(ZERO_SPACES[stage]):
            cfg = replace_dict(copy.deepcopy(base), cfg_knobs)
            cfg["train_micro_batch_size_per_gpu"] = best_mbs
            cfg.pop("train_batch_size", None)
            exps.append(self._exp(space_name, cfg))
        t = self.autotuning_config.tuner_type
        tuner_cls = {K.AUTOTUNING_TUNER_GRIDSEARCH: GridSearchTuner, K.AUTOTUNING_TUNER_RANDOM: RandomTuner,
                     K.AUTOTUNING_TUNER_MODELBASED: ModelBasedTuner}[t]
        tuner = tuner_cls(exps, self.rm, self.metric())
        n = tuner.tune(sample_size=1, n_trials=self.autotuning_config.tuner_num_trials,
                       early_stopping=self.autotuning_config.tuner_early_stopping)
        if tuner.best_exp is not None:
            self.update_records(space_name, tuner.best_exp, tuner.best_metric_val, n)
        return self.get_best_space_record(space_name)

    def tune(self):
        self.model_info_profile_run()
        gpu_mem = self.get_gpu_memory_info()
        n = self.get_model_num_params()
        if n:
            logger.info(f"The model has {number_to_string(n)} parameters; device memory {memory_to_string(gpu_mem, 'B')}")
        stages = self.autotuning_config.zero_stages
        user_stage = self.user_config.get("zero_optimization", {}).get("stage")
        if stages is None:
            stages = [user_stage] if isinstance(user_stage, int) else [0, 1, 2, 3]
        for s in stages:
            need = self.get_instantiation_memory_required_per_gpu(s) if n else 0
            if need > gpu_mem:
                logger.info(f"ZeRO stage {s}: needs {memory_to_string(need, 'B')} per GPU for model states alone, skipping")
                continue
            self.tune_space(s)
        best = self.get_best_space_records()
        if best.get(K.GLOBAL_TUNING_SPACE):
            exp, val, _ = best[K.GLOBAL_TUNING_SPACE]
            self.optimal_ds_config = exp["ds_config"]
        return best

    # ---- config accessors and micro-batch search helpers (reference ``autotuner.py:200-300, :640-1075``) -------------
    def max_train_batch_size(self):
        return self.autotuning_config.max_train_batch_size

    def max_train_micro_batch_size_per_gpu(self):
        c = self.autotuning_config
        cap = c.max_train_micro_batch_size_per_gpu
        if self.max_train_batch_size():
            gpus = self.exp_num_gpus * self.exp_num_nodes // max(1, self.mp_size())
            cap = min(cap, max(1, self.max_train_batch_size() // max(1, gpus)))
        return cap

    def min_train_micro_batch_size_per_gpu(self):
        return self.autotuning_config.min_train_micro_batch_size_per_gpu

    def num_tuning_micro_batch_sizes(self):
        return self.autotuning_config.num_tuning_micro_batch_sizes

    def fp16_enabled(self):
        return bool((self.user_config.get("fp16") or {}).get("enabled", False))

    def get_activation_memory_per_gpu(self):
        return (self.model_info or {}).get("activation_mem_per_gpu")

    def get_val_from_user_args(self, ds_name):
        """Numeric value the user script was given for the argument mapped to config key ``ds_name``."""
        arg = (self.autotuning_config.arg_mappings or {}).get(ds_name)
        ua = list(self.args.user_args)
        if arg in ua and ua.index(arg) + 1 < len(ua) and str(ua[ua.index(arg) + 1]).isnumeric():
            return ua[ua.index(arg) + 1]
        return None

    def get_gas_from_user_config(self):
        gas = self.user_config.get("gradient_accumulation_steps", 1)
        if gas == "auto":
            gas = int(self.get_val_from_user_args("gradient_accumulation_steps") or 1)
        elif not isinstance(gas, int):
            logger.info("Specifying a list of gradient_accumulation_steps to tune is not supported. 1 would be used.")
            gas = 1
        assert gas > 0, "Gradient accumulation steps must be positive."
        return gas

    def get_tuning_micro_batch_size_list(self, min_micro_batch_size, max_micro_batch_size, num_tuning_micro_batch_sizes):
        """``(candidates, max_train_batch_size)``: up to ``num_tuning_micro_batch_sizes`` values spread evenly over
        ``[min, max]`` (both ends included), capped so that ``mbs * gas * gpus`` stays under ``max_train_batch_size``."""
        if min_micro_batch_size <= 0 or max_micro_batch_size <= 0:
            return [], 0
        gpus = self.exp_num_gpus * self.exp_num_nodes // max(1, self.mp_size())
        gas = self.get_gas_from_user_config()
        cap = self.max_train_batch_size()
        if cap:
            max_micro_batch_size = min(max_micro_batch_size, max(1, cap // (gas * gpus)))
        if min_micro_batch_size > max_micro_batch_size:
            return [], 0
        n = max(1, num_tuning_micro_batch_sizes)
        if n == 1 or min_micro_batch_size == max_micro_batch_size:
            vals = [max_micro_batch_size]
        else:
            step = (max_micro_batch_size - min_micro_batch_size) / (n - 1)
            vals = sorted({int(round(min_micro_batch_size + i * step)) for i in range(n)})
        return vals, max_micro_batch_size * gas * gpus

    def run_ds_config(self, ds_config, exp_name):
        """Run ONE configuration now; returns its metric value (``None`` if the run produced none, e.g. OOM)."""
        exp = {"name": exp_name, "ds_config": ds_config, "num_gpus": self.exp_num_gpus, "num_nodes": self.exp_num_nodes,
               "hostfile": getattr(self.args, "hostfile", None)}
        with open(os.path.join(self.exps_dir, f"{exp_name}.json"), "w") as f:
            json.dump(exp, f)
        self.rm.schedule_experiments_dicts([exp])
        self.rm.run()
        val = self.rm.metric_of(exp, self.metric())
        self.rm.clear()
        return val

    def get_plateau_mbs(self, tuning_space_name):
        """Largest micro batch before the metric stopped improving by more than 5 % (0 if the space has no records)."""
        recs = sorted((r for r in self.records.get(tuning_space_name, []) if r[1] is not None),
                      key=lambda r: r[0]["ds_config"]["train_micro_batch_size_per_gpu"])
        prev_val, prev_mbs = None, 0
        for exp, val, _ in recs:
            if prev_val and (val < prev_val or (val - prev_val) / prev_val < 0.05):
                break
            prev_val, prev_mbs = val, exp["ds_config"]["train_micro_batch_size_per_gpu"]
        return prev_mbs

    def get_min_max_micro_batch_size(self, stage, min_micro_batch_size, calculated_max_micro_batch_size):
        """Probe by running: the smallest micro batch that runs at all, then binary search for the largest that still fits
        under ``calculated_max_micro_batch_size``.  ``(-1, -1)`` when nothing runs."""
        if min_micro_batch_size > calculated_max_micro_batch_size:
            return -1, -1
        space = f"{K.TUNING_MICRO_BATCH_SIZE_PREFIX}{stage}"
        base = copy.deepcopy(self.user_config)
        base.pop(K.AUTOTUNING, None)
        base.pop("train_batch_size", None)
        base.setdefault("zero_optimization", {})["stage"] = stage
        base["gradient_accumulation_steps"] = self.get_gas_from_user_config()

        def fits(mbs):
            cfg = copy.deepcopy(base)
            cfg["train_micro_batch_size_per_gpu"] = mbs
            name = f"{space}_gas{cfg['gradient_accumulation_steps']}_tmbspg{mbs}"
            val = self.run_ds_config(cfg, name)
            self.update_records(space, {"name": name, "ds_config": cfg}, val, 1)
            return val is not None

        lo = max(1, min_micro_batch_size)
        if not fits(lo):
            return -1, -1
        hi = calculated_max_micro_batch_size
        if hi > lo and fits(hi):
            return lo, hi
        best, left, right = lo, lo + 1, hi - 1
        while left <= right:
            mid = (left + right) // 2
            if fits(mid):
                best, left = mid, mid + 1
            else:
                right = mid - 1
        return lo, best

    def run_tuning_micro_batch_sizes(self, tuning_micro_batch_sizes, max_train_batch_size_per_gpu, min_gas, max_gas, stage):
        """Run the listed micro batches (gas fixed to the user's value) and return the fastest one."""
        space = f"{K.TUNING_MICRO_BATCH_SIZE_PREFIX}{stage}"
        base = copy.deepcopy(self.user_config)
        base.pop(K.AUTOTUNING, None)
        base.pop("train_batch_size", None)
        base.setdefault("zero_optimization", {})["stage"] = stage
        gas = min(max(self.get_gas_from_user_config(), min_gas or 1), max_gas or 10**9)
        for mbs in tuning_micro_batch_sizes:
            if max_train_batch_size_per_gpu and mbs * gas > max_train_batch_size_per_gpu:
                continue
            cfg = copy.deepcopy(base)
            cfg["train_micro_batch_size_per_gpu"], cfg["gradient_accumulation_steps"] = mbs, gas
            name = f"{space}_gas{gas}_tmbspg{mbs}"
            self.update_records(space, {"name": name, "ds_config": cfg}, self.run_ds_config(cfg, name), 1)
        rec = self.get_best_space_record(space)
        return rec[0]["ds_config"]["train_micro_batch_size_per_gpu"] if rec else 0

    # ---- records / reporting
    def update_records(self, space_name, exp, metric_val, num_exps):
        self.records.setdefault(space_name, []).append((exp, metric_val, num_exps))

    def get_best_space_record(self, space_name):
        recs = [r for r in self.records.get(space_name, []) if r[1] is not None]
        if not recs:
            return None
        key = (lambda r: -r[1]) if self.metric() != "latency" else (lambda r: r[1])
        best = sorted(recs, key=key)[0]
        return (best[0], best[1], sum(r[2] for r in self.records[space_name]))

    def get_best_space_records(self):
        out, glob = {}, None
        for name in self.records:
            b = self.get_best_space_record(name)
            if b is None:
                continue
            out[name] = b
            if glob is None or (b[1] < glob[1] if self.metric() == "latency" else b[1] > glob[1]):
                glob = b
        if glob is not None:
            out[K.GLOBAL_TUNING_SPACE] = glob
        return out

    def print_tuning_results(self):
        best = self.get_best_space_records()
        rows = [(name, n, val, exp["name"]) for name, (exp, val, n) in best.items()]
        try:
            from tabulate import tabulate
            print(tabulate(rows, headers=["tuning_space", "num_experiments", "best_metric_val", "best_exp_name"],
                           tablefmt="pipe"))
        except Exception:
            for r in rows:
                print(r)
        if K.GLOBAL_TUNING_SPACE in best:
            exp, val, n = best[K.GLOBAL_TUNING_SPACE]
            print(f"\nTuning completed. Best {self.metric()} = {val} from {exp['name']} after {n} experiments.")

    def write_optimal_config(self):
        best = self.get_best_space_records().get(K.GLOBAL_TUNING_SPACE)
        if not best:
            return
        exp, _, _ = best
        cfg = copy.deepcopy(exp["ds_config"])
        cfg.pop(K.AUTOTUNING, None)
        path = os.path.join(self.results_dir, "ds_config_optimal.json")
        with open(path, "w") as f:
            json.dump(cfg, f, indent=2)
        user_args = list(self.args.user_args)
        for i, a in enumerate(user_args):
            if a in ("--deepspeed_config", "--deepspeed-config") and i + 1 < len(user_args):
                user_args[i + 1] = path
        self.optimal_cmd = ["deepspeed", self.args.user_script] + user_args
        with open(os.path.join(self.results_dir, "cmd_optimal.txt"), "w") as f:
            f.write(" ".join(self.optimal_cmd))
        self.optimal_ds_config = cfg
        logger.info(f"Wrote optimal config to {path}")

    def run_after_tuning(self):
        if self.optimal_cmd:
            import subprocess
            import sys
            cmd = [sys.executable, "-m", "deepspeed_b200.launcher.runner"] + self.optimal_cmd[1:]
            subprocess.Popen(cmd).wait()
        else:
            logger.info("No optimal DeepSpeed configuration found by autotuning.")

"""``ds_report``: environment + op compatibility report (reference ``env_report.py``)."""
import argparse
import importlib
import importlib.util
import os
import shutil
import subprocess
import sys

GREEN, RED, YELLOW, END = "\033[92m", "\033[91m", "\033[93m", "\033[0m"
OKAY, FAIL, WARN = f"{GREEN}[OKAY]{END}", f"{RED}[FAIL]{END}", f"{YELLOW}[WARNING]{END}"
YES, NO = f"{GREEN}[YES]{END}", f"{YELLOW}[NO]{END}"


def op_report(verbose=True):
    from deepspeed_b200.op_builder import ALL_OPS
    print("-" * 50 + "\nDeepSpeed-H100 native op report\n" + "-" * 50)
    print("NOTE: native ops are built in-tree into deepspeed_b200/lib (sm_90a only); 'installed' means the shared\n"
          "      object is present and up to date, 'compatible' means the toolchain can (re)build it here.\n" + "-" * 50)
    print(f"{'op name':<24}{'installed':<22}{'compatible'}\n" + "-" * 50)
    for name, builder in ALL_OPS.items():
        b = builder()
        inst = YES if b.installed() else NO
        comp = OKAY if b.is_compatible(verbose) else FAIL
        print(f"{name:<24}{inst:<31}{comp}")


def nvcc_version():
    nvcc = shutil.which("nvcc") or os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "nvcc")
    try:
        out = subprocess.check_output([nvcc, "-V"], universal_newlines=True)
        rel = [l for l in out.splitlines() if "release" in l]
        return rel[0].split("release")[1].split(",")[0].strip() if rel else "unknown"
    except Exception:
        return f"{RED}[FAIL] cannot find nvcc{END}"


def ninja_installed():
    """True when the ``ninja`` build tool the JIT op loader needs is importable."""
    return importlib.util.find_spec("ninja") is not None


def human_readable_size(size):
    """Bytes → ``"12.34 GB"`` (binary units)."""
    units = ["B", "KB", "MB", "GB", "TB", "PB"]
    v, i = float(size), 0
    while v >= 1024 and i < len(units) - 1:
        v, i = v / 1024, i + 1
    return f"{v:.2f} {units[i]}"


def get_shm_size():
    """(size string, [warnings]) for ``/dev/shm``: NCCL's intra-node transports fall back to sockets when it is tiny
    (reference ``env_report.py:110``)."""
    try:
        total = shutil.disk_usage("/dev/shm").total
    except OSError:
        return "UNKNOWN", []
    warn = []
    if total < 512 * 1024**2:
        warn.append(f" {YELLOW} [WARNING] /dev/shm size might be too small, if running in docker increase to at least "
                    f"--shm-size='1gb' {END}")
        try:
            import torch
            if torch.cuda.is_available():
                warn.append(f" {YELLOW} [WARNING] see more details about NCCL requirements: "
                            f"https://docs.nvidia.com/deeplearning/nccl/user-guide/docs/troubleshooting.html#sharing-data {END}")
        except ImportError:
            pass
    return human_readable_size(total), warn


def debug_report():
    import torch
    import deepspeed_b200
    rows = [("torch install path", torch.__path__), ("torch version", torch.__version__),
            ("deepspeed_b200 install path", deepspeed_b200.__path__), ("deepspeed_b200 info", deepspeed_b200.__version__),
            ("torch cuda version", torch.version.cuda), ("nvcc version", nvcc_version()),
            ("cuda available", torch.cuda.is_available())]
    if torch.cuda.is_available():
        p = torch.cuda.get_device_properties(0)
        rows += [("device", f"{p.name} sm_{p.major}{p.minor} x{torch.cuda.device_count()}"),
                 ("device memory", f"{p.total_memory / 2**30:.1f} GiB"), ("SM count", p.multi_processor_count)]
    try:
        rows.append(("nccl version", ".".join(map(str, torch.cuda.nccl.version()))))
    except Exception:
        pass
    import psutil
    shm, shm_warn = get_shm_size()
    rows.append(("shared memory (/dev/shm) size", shm))
    rows.append(("host memory", f"{psutil.virtual_memory().total / 2**30:.1f} GiB"))
    print("DeepSpeed-H100 general environment info:")
    for k, v in rows:
        print(f"{k} {'.' * (40 - len(k))} {v}")
    for w in shm_warn:
        print(w)


def parse_arguments():
    p = argparse.ArgumentParser()
    p.add_argument("--hide_operator_status", action="store_true")
    p.add_argument("--hide_errors_and_warnings", action="store_true")
    return p.parse_args()


def main(hide_operator_status=False, hide_errors_and_warnings=False):
    if not hide_operator_status:
        op_report(verbose=not hide_errors_and_warnings)
    debug_report()


def cli_main():
    a = parse_arguments()
    main(a.hide_operator_status, a.hide_errors_and_warnings)


if __name__ == "__main__":
    cli_main()


def installed_cann_path():
    """Ascend toolkits are not a target of this build (single-vendor: NVIDIA sm_90a)."""
    return None


def installed_cann_version():
    return None

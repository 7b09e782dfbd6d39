"""Native build system: nvcc / g++ -> in-tree shared libraries loaded with ctypes.

Parity target: reference ``op_builder/builder.py`` (``OpBuilder.load :523``, ``jit_load :542``,
``CUDAOpBuilder.compute_capability_args :610``).  Design differences:

* One arch only: ``-gencode arch=compute_90a,code=sm_90a`` (the ``a`` suffix is required for
  ``wgmma`` / ``setmaxnreg`` / ``multimem``).  No arch sweep, no ``TORCH_CUDA_ARCH_LIST``.
* Kernels expose a C ABI and never include torch headers, so a full rebuild is seconds and the
  ``.so`` files live in ``deepspeed_b200/lib`` (in-tree: they travel with the repo snapshot and are
  visible in ``/proc/self/maps`` of every process that uses them).
* Objects are cached by content hash of (source, headers, flags); unchanged files are not rebuilt.
* ``DS_BUILD_OPS`` / ``DSB200_BUILD_JOBS`` / ``DSB200_NVCC`` environment knobs.
"""
import concurrent.futures
import ctypes
import hashlib
import os
import shutil
import subprocess
import threading
from pathlib import Path
from typing import Dict, List, Optional

ROOT = Path(__file__).resolve().parent.parent
CSRC = ROOT / "csrc"
LIB_DIR = ROOT / "lib"
OBJ_DIR = LIB_DIR / "obj"

ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
              "--expt-relaxed-constexpr", "-DNDEBUG"]
CXX_FLAGS = ["-O3", "-std=c++17", "-fPIC", "-fopenmp", "-fvisibility=hidden", "-DNDEBUG", "-pthread"]

_lock = threading.Lock()
_loaded: Dict[str, ctypes.CDLL] = {}


class BuildError(RuntimeError):
    pass


def nvcc_path() -> Optional[str]:
    cand = os.environ.get("DSB200_NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if cand and os.path.exists(cand) else None


def cxx_path() -> str:
    """Host C++ compiler.  ``$CXX`` is deliberately NOT honoured blindly: some images export a wrapper
    without OpenMP specs; ``DSB200_CXX`` overrides, else the first ``g++`` on PATH."""
    return os.environ.get("DSB200_CXX") or shutil.which("g++") or "g++"


def cuda_home() -> str:
    n = nvcc_path()
    return str(Path(n).resolve().parent.parent) if n else os.environ.get("CUDA_HOME", "/usr/local/cuda")


def _simd_flags() -> List[str]:
    """Pick the widest x86 SIMD level the *build host* supports; the CPU kernels also carry a
    runtime dispatch so a library built with AVX-512 still runs on an AVX2-only host."""
    try:
        flags = open("/proc/cpuinfo").read()
    except OSError:
        return []
    out = []
    if " avx2" in flags:
        out += ["-mavx2", "-mfma", "-mf16c"]
    return out


def _hash(paths: List[Path], flags: List[str]) -> str:
    h = hashlib.sha256()
    for p in paths:
        h.update(str(p.name).encode())
        h.update(p.read_bytes())
    h.update(" ".join(flags).encode())
    return h.hexdigest()[:16]


def _headers() -> List[Path]:
    return sorted((CSRC / "include").glob("*"))


def _run(cmd: List[str]):
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        raise BuildError(f"command failed: {' '.join(cmd)}\n{proc.stdout}")
    return proc.stdout


class MissingCUDAException(Exception):
    pass


class CUDAMismatchException(Exception):
    pass


DEFAULT_COMPUTE_CAPABILITIES = "9.0a"


def installed_cuda_version(name=""):
    """(major, minor) of the toolkit ``nvcc`` belongs to (reference ``builder.py:47``)."""
    nv = nvcc_path()
    if nv is None:
        raise MissingCUDAException("CUDA_HOME does not exist, unable to compile CUDA op(s)")
    out = _run([nv, "-V"])
    import re
    m = re.search(r"release (\d+)\.(\d+)", out)
    if m is None:
        raise MissingCUDAException(f"cannot parse `nvcc -V` output: {out!r}")
    return int(m.group(1)), int(m.group(2))


def get_default_compute_capabilities():
    return DEFAULT_COMPUTE_CAPABILITIES


def assert_no_cuda_mismatch(name=""):
    """The toolkit must be able to target sm_90a (CUDA ≥ 12.0) and share torch's CUDA major version; minor-version skew
    is tolerated (the kernels use a C ABI, no torch headers).  ``DS_SKIP_CUDA_CHECK=1`` downgrades errors to warnings."""
    major, minor = installed_cuda_version(name)
    problems = []
    if (major, minor) < (12, 0):
        problems.append(f"CUDA {major}.{minor} cannot compile for sm_90a (needs >= 12.0)")
    try:
        import torch
        tv = torch.version.cuda
        if tv and int(tv.split(".")[0]) != major:
            problems.append(f"installed CUDA {major}.{minor} does not match the version torch was built with ({tv})")
    except ImportError:
        pass
    if problems:
        if os.environ.get("DS_SKIP_CUDA_CHECK", "0") == "1":
            print("[WARNING] " + "; ".join(problems))
            return True
        raise CUDAMismatchException(f">- DeepSpeed-H100 op builder ({name}): " + "; ".join(problems))
    return True


class OpBuilder:
    """Build one shared library from a list of sources (``.cu`` via nvcc, ``.cpp`` via g++)."""
    VERSION_CHECKED = False

    NAME = "base"
    SOURCES: List[str] = []
    EXTRA_NVCC: List[str] = []
    EXTRA_CXX: List[str] = []
    LINK_LIBS: List[str] = []
    NEEDS_CUDA = True

    def __init__(self):
        self.name = self.NAME

    # reference API surface -------------------------------------------------------------------
    def absolute_name(self):
        return f"deepspeed_b200.lib.lib{self.NAME}"

    def sources(self):
        return [str(CSRC / s) for s in self.SOURCES]

    def include_paths(self):
        return [str(CSRC / "include"), os.path.join(cuda_home(), "include")]

    def is_compatible(self, verbose=False):
        if self.NEEDS_CUDA and nvcc_path() is None and not self.lib_path().exists():
            return False
        return True

    def lib_path(self) -> Path:
        return LIB_DIR / f"lib{self.NAME}.so"

    # toolchain probes (reference ``OpBuilder`` helpers) ------------------------------------------------------------
    def builder(self):
        return self

    def extra_ldflags(self):
        return list(self.LINK_LIBS)

    def nvcc_args(self):
        return []

    def cxx_args(self):
        return CXX_FLAGS + self.EXTRA_CXX

    @staticmethod
    def validate_torch_version(torch_info=None):
        """In-tree libraries carry no torch ABI, so any installed torch is fine; kept for callers of the reference API."""
        return True

    validate_torch_op_version = validate_torch_version

    @staticmethod
    def installed_rocm_version():
        """(major, minor) of a ROCm toolchain -- there is none on this single-vendor build (reference ``builder.py:163``)."""
        return 0, 0

    @staticmethod
    def is_rocm_pytorch():
        return False

    @staticmethod
    def is_sycl_enabled():
        return False

    def hipify_extension(self):
        pass

    def sycl_extension(self):
        pass

    def strip_empty_entries(self, args):
        return [a for a in args if len(a) > 0]

    def command_exists(self, cmd):
        cmds = cmd if isinstance(cmd, (list, tuple)) else [cmd]
        ok = any(shutil.which(c) is not None for c in cmds)
        if not ok:
            self.warning(f"{self.name} requires one of {cmds}, none of which is on PATH")
        return ok

    def warning(self, msg):
        print(f"\033[93m [WARNING] \033[0m {msg}")

    def deepspeed_src_path(self, code_path):
        return str(CSRC / code_path) if not os.path.isabs(code_path) else code_path

    def has_function(self, funcname, libraries, library_dirs=None, verbose=False):
        """Can a program calling ``funcname`` be linked against ``libraries``?"""
        import tempfile
        with tempfile.TemporaryDirectory() as d:
            src = os.path.join(d, "probe.c")
            with open(src, "w") as f:
                f.write(f"#ifdef __cplusplus\nextern \"C\"\n#endif\nchar {funcname}(void);\nint main(void) {{ {funcname}(); return 0; }}\n")
            cmd = [os.environ.get("CC", "gcc"), src, "-o", os.path.join(d, "probe")] + \
                [f"-L{p}" for p in (library_dirs or [])] + [f"-l{l}" for l in libraries]
            return subprocess.run(cmd, stdout=subprocess.DEVNULL, stderr=subprocess.DEVNULL).returncode == 0

    def _cpu_flags(self):
        try:
            for line in open("/proc/cpuinfo"):
                if line.startswith("flags"):
                    return set(line.split(":", 1)[1].split())
        except OSError:
            pass
        return set()

    def cpu_arch(self):
        """``-march=native`` unless the host is not x86 (then the compiler default)."""
        import platform
        return "-march=native" if platform.machine() in ("x86_64", "AMD64") else ""

    def simd_width(self):
        """The macro the CPU kernels are compiled with: ``-D__AVX512__`` / ``-D__AVX256__`` / scalar."""
        flags = self._cpu_flags()
        if "avx512f" in flags:
            return "-D__AVX512__"
        if "avx2" in flags:
            return "-D__AVX256__"
        return "-D__SCALAR__"

    def get_cuda_compile_flag(self):
        return "-D__ENABLE_CUDA__" if nvcc_path() is not None else "-D__DISABLE_CUDA__"

    def installed(self) -> bool:
        return self.lib_path().exists()

    # build -----------------------------------------------------------------------------------
    def _compile_one(self, src: Path) -> Path:
        is_cu = src.suffix == ".cu"
        incs = [f"-I{p}" for p in self.include_paths()]
        if is_cu:
            flags = ARCH_FLAGS + NVCC_FLAGS + self.EXTRA_NVCC + incs
            tool = nvcc_path()
            if tool is None:
                raise BuildError("nvcc not found; cannot build CUDA sources")
        else:
            flags = CXX_FLAGS + _simd_flags() + self.EXTRA_CXX + incs
            tool = cxx_path()
        key = _hash([src] + _headers(), flags)
        obj = OBJ_DIR / f"{self.NAME}-{src.stem}-{key}.o"
        if obj.exists():
            return obj
        OBJ_DIR.mkdir(parents=True, exist_ok=True)
        for stale in OBJ_DIR.glob(f"{self.NAME}-{src.stem}-*.o"):
            stale.unlink(missing_ok=True)
        tmp = obj.with_suffix(f".tmp{os.getpid()}.o")
        _run([tool] + flags + ["-c", str(src), "-o", str(tmp)])
        os.replace(tmp, obj)
        return obj

    def build(self, verbose=False, jobs: Optional[int] = None) -> Path:
        srcs = [Path(s) for s in self.sources()]
        jobs = jobs or int(os.environ.get("DSB200_BUILD_JOBS", os.cpu_count() or 4))
        with concurrent.futures.ThreadPoolExecutor(max_workers=max(1, min(jobs, len(srcs)))) as ex:
            objs = list(ex.map(self._compile_one, srcs))
        stamp = hashlib.sha256(" ".join(sorted(o.name for o in objs)).encode()).hexdigest()[:16]
        stamp_file = LIB_DIR / f"lib{self.NAME}.stamp"
        out = self.lib_path()
        if out.exists() and stamp_file.exists() and stamp_file.read_text() == stamp:
            return out
        LIB_DIR.mkdir(parents=True, exist_ok=True)
        tmp = out.with_suffix(f".tmp{os.getpid()}.so")
        if self.NEEDS_CUDA:
            cmd = [nvcc_path(), "-shared"] + ARCH_FLAGS + ["-Xcompiler", "-fPIC", "-o", str(tmp)] + \
                [str(o) for o in objs] + ["-lcudart"] + self.LINK_LIBS
        else:
            cmd = [cxx_path(), "-shared", "-fPIC", "-fopenmp", "-o", str(tmp)] + \
                [str(o) for o in objs] + self.LINK_LIBS
        _run(cmd)
        os.replace(tmp, out)
        stamp_file.write_text(stamp)
        if verbose:
            print(f"[deepspeed_b200] built {out}")
        return out

    def jit_load(self, verbose=False):
        return self.load(verbose)

    def load(self, verbose=False) -> ctypes.CDLL:
        with _lock:
            if self.NAME in _loaded:
                return _loaded[self.NAME]
            path = self.lib_path()
            can_build = (nvcc_path() is not None) if self.NEEDS_CUDA else True
            if can_build and os.environ.get("DSB200_NO_JIT", "0") != "1":
                try:
                    path = self.build(verbose)
                except BuildError:
                    if not path.exists():
                        raise
            if not path.exists():
                raise BuildError(f"native library {path} is missing and cannot be built here; run "
                                 f"`python -c 'import __graft_entry__ as g; g.build()'` on a host with nvcc")
            lib = ctypes.CDLL(str(path), mode=ctypes.RTLD_GLOBAL)
            _loaded[self.NAME] = lib
            return lib


class CUDAOpBuilder(OpBuilder):
    NEEDS_CUDA = True

    def compute_capability_args(self, cross_compile_archs=None):
        return list(ARCH_FLAGS)

    def filter_ccs(self, ccs):
        """Only sm_90a is ever built: every requested capability collapses to it."""
        return [["9", "0a"]]

    def version_dependent_macros(self):
        return ["-DVERSION_GE_1_1", "-DVERSION_GE_1_3", "-DVERSION_GE_1_5"]

    def libraries_args(self):
        return ["cudart"]

    def is_compatible(self, verbose=False):
        if not super().is_compatible(verbose):
            return False
        if nvcc_path() is not None and not OpBuilder.VERSION_CHECKED:
            try:
                assert_no_cuda_mismatch(self.name)
            except (CUDAMismatchException, MissingCUDAException) as e:
                if verbose:
                    self.warning(str(e))
                return self.lib_path().exists()
            OpBuilder.VERSION_CHECKED = True
        return True

    def nvcc_args(self):
        return NVCC_FLAGS + self.EXTRA_NVCC

    def cxx_args(self):
        return CXX_FLAGS + self.EXTRA_CXX


class CPUOpBuilder(OpBuilder):
    NEEDS_CUDA = False

    def get_cuda_lib64_path(self):
        return os.path.join(cuda_home(), "lib64")

    def include_paths(self):
        return [str(CSRC / "include")]


TorchCPUOpBuilder = CPUOpBuilder  # reference name of the host-op base class

"""In-tree build of libhawq_b200.so with nvcc for sm_90a (Hopper; cross-compiles without a GPU)."""
import glob
import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")
OUT = os.path.join(_HERE, "libhawq_b200.so")

GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = GENCODE + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]
OBJ_DIR = os.path.join(_HERE, "_obj")


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found")


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def _deps():
    return sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(INCLUDE, "*.h"))


def _deps_digest():
    import hashlib
    h = hashlib.sha256()
    for d in sorted(_deps()):
        h.update(os.path.basename(d).encode())
        h.update(open(d, "rb").read())
    return h.hexdigest()


def up_to_date():
    """The library exists and was built from exactly these sources (content digest in a stamp file: file times do not survive the
    copy to a GPU box)."""
    if not os.path.isfile(OUT) or not os.path.isfile(OUT + ".stamp"):
        return False
    return open(OUT + ".stamp").read().strip() == _deps_digest()


def _includes(path, seen=None):
    """Transitive closure of the quoted #includes of a source file (for per-object staleness)."""
    import re
    seen = set() if seen is None else seen
    try:
        text = open(path).read()
    except OSError:
        return seen
    for inc in re.findall(r'#include\s+"([^"]+)"', text):
        f = os.path.normpath(os.path.join(os.path.dirname(path), inc))
        if f not in seen and os.path.isfile(f):
            seen.add(f)
            _includes(f, seen)
    return seen


def _compile_objects(force, verbose, extra_flags):
    """One object per .cu (compiled in parallel; only stale ones), so editing one kernel file does not rebuild the others."""
    from concurrent.futures import ThreadPoolExecutor
    os.makedirs(OBJ_DIR, exist_ok=True)
    tag = "_".join(extra_flags).replace("/", "_").replace("=", "_")
    jobs, objs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + (("." + tag) if tag else "") + ".o")
        objs.append(obj)
        deps = [src] + sorted(_includes(src))
        if force or not os.path.isfile(obj) or any(os.path.getmtime(d) > os.path.getmtime(obj) for d in deps):
            jobs.append((src, obj))

    def run(job):
        src, obj = job
        cmd = [_nvcc()] + NVCC_FLAGS + list(extra_flags) + ["-I", INCLUDE, "-c", "-o", obj + ".tmp.%d" % os.getpid(), src]
        if verbose:
            print(" ".join(cmd).replace(".tmp.%d" % os.getpid(), ""))
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed on %s:\n%s" % (src, r.stdout))
        os.replace(obj + ".tmp.%d" % os.getpid(), obj)
        return r.stdout

    with ThreadPoolExecutor(max_workers=max(1, min(len(jobs), os.cpu_count() or 1))) as ex:
        for out in ex.map(run, jobs):
            if verbose and out:
                print(out)
    return objs


def build_library(force=False, verbose=False, extra_flags=()):
    """Compile every .cu under csrc/ into hawq_b200/libhawq_b200.so.  Returns the path.
    Safe when several processes call it at once (one rank per GPU under torchrun): an exclusive file lock serialises them, the
    winner compiles into a temporary file and renames it into place, the others find the library up to date."""
    if not force and up_to_date():
        return OUT
    import fcntl
    with open(OUT + ".lock", "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and up_to_date():               # another process built it while we waited
                return OUT
            objs = _compile_objects(force, verbose, tuple(extra_flags))
            tmp = "%s.tmp.%d" % (OUT, os.getpid())
            cmd = [_nvcc()] + GENCODE + ["--shared", "-o", tmp] + objs
            if verbose:
                print(" ".join(cmd).replace(tmp, OUT))
            r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
            if r.returncode != 0:
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc link failed:\n" + r.stdout)
            os.replace(tmp, OUT)
            with open(OUT + ".stamp", "w") as f:
                f.write(_deps_digest())
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return OUT


RUNNER_SRC = os.path.join(os.path.dirname(_HERE), "tools", "hawq_run.c")
RUNNER = os.path.join(_HERE, "hawq_run")


def _cuda_root():
    return os.path.dirname(os.path.dirname(os.path.realpath(_nvcc())))


def build_runner(verbose=False):
    """Compile tools/hawq_run.c next to the library: the standalone runner of plan files.  It links libhawq_b200.so (found next to
    the binary) and the static CUDA runtime, and nothing of Python or torch."""
    cuda = _cuda_root()
    tmp = "%s.tmp.%d" % (RUNNER, os.getpid())
    cmd = ["gcc", "-O2", "-std=c11", "-Wall", "-I", INCLUDE, "-I", os.path.join(cuda, "include"), "-o", tmp, RUNNER_SRC, "-L", _HERE,
           "-l:libhawq_b200.so", "-Wl,-rpath,$ORIGIN", "-L", os.path.join(cuda, "lib64"), "-lcudart_static", "-lrt", "-lpthread", "-ldl"]
    if verbose:
        print(" ".join(cmd).replace(tmp, RUNNER))
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise RuntimeError("building hawq_run failed:\n" + r.stdout)
    os.replace(tmp, RUNNER)
    return RUNNER

"""In-tree build of libcrnnctc.so (sm_90a only; nvcc cross-compiles without a GPU)."""
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(ROOT, "lstm_ctc_ocr_b200", "csrc")
OUT = os.path.join(ROOT, "lstm_ctc_ocr_b200", "libcrnnctc.so")
SOURCES = ["ctc.cu", "align.cu", "lexicon.cu", "kernels.cu", "model.cu", "backward_kernels.cu", "backward.cu", "forward_x3.cu", "forward_fp8.cu", "peer.cu", "beam.cpp",
           "beam.cu"]
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-I/usr/local/cuda/include"]


def _stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "crnn_ctc.h")]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not _stale():
        return OUT
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    os.makedirs(os.path.join(ROOT, "build"), exist_ok=True)
    for src in SOURCES:
        obj = os.path.join(ROOT, "build", src + ".o")        # beam.cpp and beam.cu both exist
        cmd = [nvcc, "-c", os.path.join(CSRC, src), "-o", obj] + FLAGS + (["-Xptxas", "-v"] if verbose else [])
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(obj)
    for src, p in procs:
        out, _ = p.communicate()
        if verbose or p.returncode != 0:
            sys.stderr.write(out)
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
    cmd = [nvcc, "-shared", "-o", OUT] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    subprocess.check_call(cmd)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))

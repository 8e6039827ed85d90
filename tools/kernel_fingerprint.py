"""What the compiler made of the search and embed kernels, in a form two checkouts can be diffed on.  Needs nvcc, no GPU.

    python tools/kernel_fingerprint.py OUT_DIR [CSRC_DIR]
    git worktree add /tmp/parent HEAD~1
    python tools/kernel_fingerprint.py /tmp/fp_parent /tmp/parent/clip-retrieval_b200/csrc
    python tools/kernel_fingerprint.py /tmp/fp_branch
    diff -r /tmp/fp_parent /tmp/fp_branch

Compiles knn_scan / knn_ivf / knn_ivfpq / knn_mma (search) and gemm / attention / attention_wgmma / embed_kernels /
clip_model / text_encoder (embed path) with the flags of build.py plus -Xptxas=-v and writes, per
source, `<name>.res` (one line per kernel entry: registers, barriers, shared memory, stack frame, spill bytes) and
`<name>.sass` (cuobjdump -sass per function, addresses and encodings stripped, functions sorted by name).  A refactor
that claims to leave a kernel alone shows an empty diff for it; identical SASS settles its speed and its results.
"""
import importlib.util
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = ["knn_scan", "knn_ivf", "knn_ivfpq", "knn_mma", "latent_pool", "dwconv",
           "gemm", "attention", "attention_wgmma", "embed_kernels", "clip_model", "text_encoder"]


def _build_py():
    spec = importlib.util.spec_from_file_location("b200_build", os.path.join(ROOT, "clip-retrieval_b200", "build.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def resources(ptxas_log):
    """{kernel: 'Used ... | stack/spill ...'} from the -Xptxas=-v log."""
    out, name, frame = {}, None, ""
    for line in ptxas_log.splitlines():
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            name = m.group(1)
        elif "bytes stack frame" in line:
            frame = line.strip()
        elif name and "Used" in line:
            out[name] = "%s | %s" % (line.split(":", 1)[1].strip(), frame)
            name = None
    return out


def sass(obj, cuobjdump):
    text = subprocess.run([cuobjdump, "-sass", obj], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in text.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(.*?)\s*/\* 0x[0-9a-f]+ \*/", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


def main():
    out_dir = sys.argv[1]
    bp = _build_py()
    csrc = sys.argv[2] if len(sys.argv) > 2 else bp.CSRC
    nvcc = bp._nvcc()
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    os.makedirs(out_dir, exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        procs = []
        for name in SOURCES:
            obj = os.path.join(tmp, name + ".o")
            cmd = [nvcc, "-Xptxas=-v"] + bp.NVCC_FLAGS + ["-c", os.path.join(csrc, name + ".cu"), "-o", obj]
            procs.append((name, obj, subprocess.Popen(cmd, stderr=subprocess.PIPE, text=True)))
        for name, obj, p in procs:
            log = p.communicate()[1]
            if p.returncode != 0:
                sys.exit("nvcc failed for %s:\n%s" % (name, log))
            res = resources(log)
            with open(os.path.join(out_dir, name + ".res"), "w") as f:
                for k in sorted(res):
                    f.write("%s: %s\n" % (k, res[k]))
            funcs = sass(obj, cuobjdump)
            with open(os.path.join(out_dir, name + ".sass"), "w") as f:
                for k in sorted(funcs):
                    f.write("Function %s\n" % k)
                    f.writelines("  %s\n" % ins for ins in funcs[k])
            print("%s: %d kernel entries, %d with spills" % (
                name, len(res), sum("0 bytes spill stores, 0 bytes spill loads" not in v for v in res.values())))


if __name__ == "__main__":
    main()

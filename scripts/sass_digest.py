"""One line per kernel of a built library: its resource usage and a hash of its SASS opcode sequence.

    python scripts/sass_digest.py [tfdiffeq_b200/libb2ode.so] > digest.txt

Each line is `<mangled name> REG:.. STACK:.. SHARED:.. LOCAL:.. <hash>`, sorted by name.  The hash covers every instruction's
mnemonic with its predicate and modifiers (`@!P0 BRA`, `DFMA.RM`), operands stripped as tests/test_sass_polls_cpu.py parses
them, so register renaming and moved addresses do not count, but any added, removed or reordered instruction does.
Changed operands (a register, an immediate, a constant-bank offset) do not show either.  Two builds whose digests `diff`
equal have the same opcode sequence and resource usage in every kernel.  No GPU needed: it reads the library with
cuobjdump.
"""
import hashlib
import os
import re
import shutil
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CUOBJDUMP = shutil.which("cuobjdump") or "/usr/local/cuda/bin/cuobjdump"
RES = ("REG", "STACK", "SHARED", "LOCAL")


def cuobjdump(flag, lib):
    return subprocess.run([CUOBJDUMP, flag, lib], capture_output=True, text=True, check=True).stdout.splitlines()


def resources(lib):
    """{kernel: 'REG:n STACK:n SHARED:n LOCAL:n'} from `cuobjdump -res-usage`."""
    res, name = {}, None
    for line in cuobjdump("-res-usage", lib):
        m = re.match(r"\s*Function (\S+):\s*$", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            fields = dict(re.findall(r"(\w+):(\d+)", line))
            res[name] = " ".join("%s:%s" % (k, fields[k]) for k in RES)
            name = None
    return res


def opcode_hashes(lib):
    """{kernel: sha256 of its opcode sequence} from `cuobjdump -sass`."""
    seqs, name = {}, None
    for line in cuobjdump("-sass", lib):
        m = re.match(r"\s*Function : (\S+)\s*$", line)
        if m:
            name = m.group(1)
            seqs[name] = hashlib.sha256()
            continue
        m = re.match(r"\s*/\*([0-9a-f]{4,})\*/\s+(.*?);", line)
        if m and name:
            tok = m.group(2).split()
            op = " ".join(tok[:2]) if tok[0].startswith("@") else tok[0]
            seqs[name].update(op.encode() + b"\n")
    return {k: h.hexdigest()[:16] for k, h in seqs.items()}


def main():
    lib = sys.argv[1] if len(sys.argv) > 1 else os.path.join(ROOT, "tfdiffeq_b200", "libb2ode.so")
    res, ops = resources(lib), opcode_hashes(lib)
    for k in sorted(set(res) | set(ops)):
        print(k, res.get(k, "-"), ops.get(k, "-"))
    print("%d kernels" % len(set(res) | set(ops)), file=sys.stderr)


if __name__ == "__main__":
    main()

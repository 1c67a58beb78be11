"""Static loop report for the lane kernels, from their SASS.  CPU only.

    python tools/sass_loops.py sentencepiece_b200/lib/libspm_b200.so
    python tools/sass_loops.py engine.sm_90a.cubin --kernel encode_unigram_lane

For each kernel whose name matches --kernel (default: the lane kernels) it prints the registers and stack frame
(cuobjdump -res-usage), the local-memory instructions (LDL/STL: spills), and every loop, found by its backward
branch: the loop head, the back-branch, the static instruction count in between (head and back-branch included) and the source
lines they come from (the library is built with -lineinfo).  Any S2R, S2UR or LDC inside a loop is listed with its
source line: in these kernels such an instruction is an address or a parameter the compiler rebuilds on every trip
instead of keeping it in a register.
"""
import argparse
import glob
import os
import re
import subprocess
import sys
import tempfile

CUDA_BIN = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin")
DEFAULT_KERNELS = r"lane"

_INSN = re.compile(r"^\s*/\*([0-9a-f]{4,})\*/\s+(.*?)\s*;")
_LABEL = re.compile(r"^(\.L_x_\d+):")
_LINE = re.compile(r'^\s*//## File "([^"]+)", line (\d+)')
_FUNC = re.compile(r"^\.text\.(\S+):")
_TARGET = re.compile(r"`\((\.L_x_\d+)\)")
_PRED = r"^(?:@!?U?P\w+\s+)?"
_REMAT = re.compile(_PRED + r"(S2R|S2UR|LDC)\b")
_BRA = re.compile(_PRED + r"BRA\b")
_LOCAL = re.compile(_PRED + r"(LDL|STL)\b")


def tool(name):
    p = os.path.join(CUDA_BIN, name)
    return p if os.path.exists(p) else name


def cubins(path, tmp):
    if path.endswith(".cubin"):
        return [path]
    subprocess.run([tool("cuobjdump"), "-xelf", "all", os.path.abspath(path)], cwd=tmp, check=True,
                   stdout=subprocess.DEVNULL)
    return sorted(glob.glob(os.path.join(tmp, "*.cubin")))


def res_usage(cubin):
    out = subprocess.run([tool("cuobjdump"), "-res-usage", cubin], check=True, capture_output=True, text=True).stdout
    usage, name = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            name = m.group(1)
            continue
        if name and "REG:" in line:
            usage[name] = dict(re.findall(r"(\w+):(\d+)", line))
            name = None
    return usage


def parse(cubin):
    """{function: [(addr, text, (file, line))]} and {function: {label: addr}}"""
    out = subprocess.run([tool("nvdisasm"), "-g", "-c", cubin], check=True, capture_output=True, text=True).stdout
    funcs, labels = {}, {}
    cur, src, pending = None, None, []
    for line in out.splitlines():
        m = _FUNC.match(line)
        if m:
            cur, src = m.group(1), None
            funcs[cur], labels[cur] = [], {}
            continue
        if cur is None:
            continue
        m = _LINE.match(line)
        if m:
            src = (os.path.basename(m.group(1)), int(m.group(2)))
            continue
        m = _LABEL.match(line)
        if m:
            pending.append(m.group(1))
            continue
        m = _INSN.match(line)
        if m:
            addr = int(m.group(1), 16)
            for lab in pending:
                labels[cur][lab] = addr
            pending = []
            funcs[cur].append((addr, m.group(2), src))
    return funcs, labels


def loops(insns, labels):
    """Loops as (head index, back-branch index), one per backward branch target, outermost first.  The out-of-line
    blocks that BRA.DIV jumps to (warp-divergent shuffles and votes) sit after the kernel's body and branch back
    into it; those branches are not loops."""
    index = {a: i for i, (a, _, _) in enumerate(insns)}
    body_end = insns[-1][0] + 1
    for addr, text, _ in insns:
        m = _TARGET.search(text)
        if "BRA.DIV" in text and m and m.group(1) in labels and labels[m.group(1)] > addr:
            body_end = min(body_end, labels[m.group(1)])
    found = {}
    for i, (addr, text, _) in enumerate(insns):
        m = _TARGET.search(text)
        if addr >= body_end or not _BRA.match(text) or not m or m.group(1) not in labels:
            continue
        t = labels[m.group(1)]
        if t <= addr:
            h = index[t]
            found[h] = max(found.get(h, i), i)
    return sorted(found.items(), key=lambda hb: (hb[0], -hb[1]))


def where(src):
    return f"{src[0]}:{src[1]}" if src else "?"


def report(name, insns, labels, usage, min_len):
    u = usage.get(name, {})
    local = sum(1 for _, t, _ in insns if _LOCAL.match(t))
    print(name)
    print(f"  registers {u.get('REG', '?')}, stack {u.get('STACK', '?')} B, local-memory instructions {local}, "
          f"instructions {len(insns)}")
    spans = loops(insns, labels)
    for h, b in spans:
        if b - h + 1 < min_len:
            continue
        inner = [(h2, b2) for h2, b2 in spans if h <= h2 and b2 <= b and (h2, b2) != (h, b)]
        depth = sum(1 for h2, b2 in spans if h2 <= h and b <= b2 and (h2, b2) != (h, b))
        ind = "  " * (depth + 1)
        print(f"{ind}loop {insns[h][0]:#06x}..{insns[b][0]:#06x}  {b - h + 1:4d} instructions  "
              f"head {where(insns[h][2])}  back-branch {where(insns[b][2])}")
        # each S2R / S2UR / LDC is listed under the innermost loop that holds it
        for i in range(h, b + 1):
            a, t, s = insns[i]
            if _REMAT.match(t) and not any(h2 <= i <= b2 for h2, b2 in inner):
                print(f"{ind}  {a:#06x}  {t:<40s} {where(s)}")
    print()


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("binary", help="libspm_b200.so, an object file or a cubin")
    ap.add_argument("--kernel", default=DEFAULT_KERNELS, help="regular expression on the mangled kernel name")
    ap.add_argument("--min-len", type=int, default=16, help="omit loops with fewer instructions")
    a = ap.parse_args()
    with tempfile.TemporaryDirectory() as tmp:
        any_kernel = False
        for cb in cubins(a.binary, tmp):
            usage = res_usage(cb)
            funcs, labels = parse(cb)
            for name in sorted(funcs):
                if re.search(a.kernel, name):
                    any_kernel = True
                    report(name, funcs[name], labels[name], usage, a.min_len)
        if not any_kernel:
            sys.exit(f"no kernel matches {a.kernel!r} in {a.binary}")


if __name__ == "__main__":
    main()

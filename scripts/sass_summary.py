"""Register / spill / shared-memory / SASS summary of every kernel in the product library (CPU only: ptxas -v logs of
erasor_b200/csrc/build.sh + cuobjdump -sass of the objects).  Writes a markdown table to stdout."""
import os
import re
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BUILD = os.path.join(ROOT, "erasor_b200", "_build")


def demangle(name):
    try:
        return subprocess.run(["cu++filt", name], capture_output=True, text=True).stdout.strip() or name
    except Exception:
        return name


def short(d):
    d = re.sub(r"^void ", "", d).replace("erasor::", "").replace("(int)", "").replace("(bool)", "")
    m = re.match(r"([A-Za-z0-9_]+)(<[^(]*?>)?\(", d)
    return (m.group(1) + (m.group(2) or "")) if m else d[:60]


def ptxas(path):
    out, cur = {}, None
    for line in open(path):
        m = re.search(r"Compiling entry function '([^']+)'", line)
        if m:
            cur = m.group(1); out[cur] = dict(stack=0, spill_st=0, spill_ld=0, regs=0, smem=0, barriers=0, seen=False)
            continue
        if cur is None:
            continue
        m = re.search(r"(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads", line)
        if m and not out[cur]["seen"]:         # the entry's own line comes first; lines of its noinline callees follow
            out[cur].update(stack=int(m.group(1)), spill_st=int(m.group(2)), spill_ld=int(m.group(3)), seen=True)
        m = re.search(r"Used (\d+) registers, used (\d+) barriers(?:, (\d+) bytes cumulative stack size)?(?:, (\d+) bytes smem)?", line)
        if m:
            out[cur].update(regs=int(m.group(1)), barriers=int(m.group(2)), smem=int(m.group(4) or 0))
    return out


def sass_counts(obj):
    txt = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
    out, cur = {}, None
    for line in txt.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1); out[cur] = {}
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s+(?:@!?U?P\d\s+)?([A-Z0-9_]+)", line)
        if cur and m:
            op = m.group(1)
            out[cur]["total"] = out[cur].get("total", 0) + 1
            for k in ("MATCH", "REDUX", "ATOMS", "MUFU", "SHFL", "LDG", "STG", "BAR", "DFMA", "DMUL", "DADD", "HMMA", "UTCMMA", "UTMALDG"):
                if op.startswith(k):
                    out[cur][k] = out[cur].get(k, 0) + 1
    return out


def main():
    print("| kernel | registers | spill st / ld (B) | stack (B) | static smem (B) | SASS instructions | MUFU | SHFL | MATCH | REDUX | ATOMS | LDG | STG | BAR | FP64 (DFMA+DMUL+DADD) | tensor (HMMA / UTCMMA) | TMA (UTMALDG) |")
    print("|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|---|")
    for stem in ("kernels", "updater_kernels"):
        p = ptxas(os.path.join(BUILD, stem + ".ptxas.log"))
        s = sass_counts(os.path.join(BUILD, stem + ".o"))
        for mangled, v in sorted(p.items(), key=lambda kv: short(demangle(kv[0]))):
            c = s.get(mangled, {})
            fp64 = c.get("DFMA", 0) + c.get("DMUL", 0) + c.get("DADD", 0)
            print(f"| `{short(demangle(mangled))}` | {v['regs']} | {v['spill_st']} / {v['spill_ld']} | {v['stack']} | {v['smem']} | {c.get('total', 0)} | {c.get('MUFU', 0)} | "
                  f"{c.get('SHFL', 0)} | {c.get('MATCH', 0)} | {c.get('REDUX', 0)} | {c.get('ATOMS', 0)} | {c.get('LDG', 0)} | {c.get('STG', 0)} | {c.get('BAR', 0)} | {fp64} | "
                  f"{c.get('HMMA', 0) + c.get('UTCMMA', 0)} | {c.get('UTMALDG', 0)} |")
    print("\nNo tensor-core or TMA instructions anywhere, as `north_star` prescribes for this path (bandwidth / issue-bound indexing and reduction, no dense contraction).")


if __name__ == "__main__":
    main()

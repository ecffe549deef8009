"""Do two built libraries hold the same kernels, instruction for instruction?  sass_same.py old.so new.so

Runs `cuobjdump -sass` and `cuobjdump -res-usage` on both.  Functions are matched by demangled name without its anonymous
namespaces (nvcc names an anonymous namespace after its file, so moving a kernel to another .cu renames it).  For each function
present in both it compares every instruction and its encoding (the /*offset*/ column dropped) and the REG / STACK / SHARED /
LOCAL / CONSTANT usage.  Prints one line per differing function and per function in only one library, then
`N functions, K differ (C in their instructions)`; exits non-zero if K > 0 or the two sets of functions differ.
"""
import os, re, subprocess, sys

CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
ANON = re.compile(r"\(anonymous namespace\)::|<unnamed>::")
USAGE = re.compile(r"\b(REG|STACK|SHARED|LOCAL|CONSTANT\[\d+\]):(\d+)")


def run(*cmd, stdin=None):
    return subprocess.run(cmd, input=stdin, capture_output=True, text=True, check=True).stdout


def functions(lib):
    """{normalised name: (instruction lines, usage)}"""
    code, usage, cur = {}, {}, None
    for ln in run(f"{CUDA}/bin/cuobjdump", "-sass", lib).splitlines():
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1); code[cur] = []
        elif cur and "/*" in ln:
            code[cur].append(" ".join(re.sub(r"^\s*/\*[0-9a-f]{4,}\*/", "", ln).split()))
    cur = None
    for ln in run(f"{CUDA}/bin/cuobjdump", "-res-usage", lib).splitlines():  # a function's usage is the line after its name
        m = re.match(r"\s*Function (\S+):", ln)
        if cur: usage[cur] = " ".join(f"{k}:{v}" for k, v in USAGE.findall(ln))
        cur = m.group(1) if m else None
    names = list(code)
    plain = run(f"{CUDA}/bin/cu++filt", stdin="\n".join(names) + "\n").splitlines()
    out = {}
    for mangled, demangled in zip(names, plain):
        key = ANON.sub("", demangled)
        if key in out: sys.exit(f"{lib}: two functions are both {key}")
        out[key] = (code[mangled], usage.get(mangled, ""))
    return out


old, new = functions(sys.argv[1]), functions(sys.argv[2])
differ = code = 0
for name in sorted(set(old) | set(new)):
    if name not in new or name not in old:
        print(f"only in {sys.argv[1] if name in old else sys.argv[2]}: {name}")
    elif old[name] != new[name]:
        differ += 1
        (oc, ou), (nc, nu) = old[name], new[name]
        code += oc != nc
        what = "instructions" if oc != nc else "usage"
        print(f"differs ({what}): {name}: {ou} -> {nu}")
print(f"{len(set(old) & set(new))} functions, {differ} differ ({code} in their instructions)")
sys.exit(1 if differ or set(old) != set(new) else 0)

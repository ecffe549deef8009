"""Opcode histogram of the steady-state march loop of k_chain_fused in a built library (static count over the five unrolled
phases, i.e. per 5 march steps, rare paths included): sass_loop.py <substring of the mangled kernel name> <lib.so> [<lib.so> ...].
With several libraries the histograms are printed side by side (per march step), e.g. a parent build against a new one.
The loop is the chunk loop: the innermost backward branch that encloses the first mbarrier try-wait, from its target up to
the branch itself.  Instantiations: 'Lb1EEELb0' / 'Lb1EEELb1' are ShapeA without / with the normals outputs, 'Lb0EEELb0' /
'Lb0EEELb1' ShapeB."""
import collections, re, subprocess, sys


def loop_histogram(lib, pat):
    out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True, check=True).stdout.splitlines()
    funcs, cur = {}, None
    for ln in out:
        m = re.search(r"Function : (\S+)", ln)
        if m:
            cur = m.group(1) if "k_chain_fused" in m.group(1) and pat in m.group(1) else None
            if cur: funcs[cur] = []
            continue
        m = re.match(r"\s+/\*([0-9a-f]{4,})\*/\s+(.*?);", ln) if cur else None
        if m: funcs[cur].append((int(m.group(1), 16), m.group(2).strip()))
    if len(funcs) != 1:
        raise SystemExit(f"{lib}: '{pat}' matches {len(funcs)} k_chain_fused instantiations: {sorted(funcs)}")
    name, body = next(iter(funcs.items()))
    wait = next(a for a, t in body if "TRYWAIT" in t)
    best = None  # (target, address) of the innermost enclosing backward branch
    for a, t in body:
        # BRA 0x.., BRA.U.ANY 0x.., and forms with an operand before the target (BRA.U !UP0, 0x.. ; BRA.DIV UR4, 0x..)
        m = re.search(r"\bBRA(?:\.\S+)?\s+(?:\S+,\s*)?(0x[0-9a-f]+)$", t)
        if not m: continue
        tgt = int(m.group(1), 16)
        if tgt <= wait < a and (best is None or tgt > best[0]):
            best = (tgt, a)
    if best is None:
        raise SystemExit(f"{lib}: no backward branch encloses the mbarrier wait of {name}")
    h = collections.Counter()
    for a, t in body:
        if best[0] <= a <= best[1]:
            op = t.split()
            o = op[1] if op[0].startswith("@") else op[0]
            h[o.split(".")[0]] += 1
    return name, best, h


def main():
    if len(sys.argv) < 3:
        raise SystemExit(__doc__)
    pat, libs = sys.argv[1], sys.argv[2:]
    res = [loop_histogram(lib, pat) for lib in libs]
    for lib, (name, (lo, hi), h) in zip(libs, res):
        n = sum(h.values())
        print(f"{lib}: {name}\n  loop {lo:#x}..{hi:#x}: {n} instructions / 5 steps = {n / 5:.1f} per step")
    ops = sorted(set().union(*(h for _, _, h in res)), key=lambda o: -max(h[o] for _, _, h in res))
    print("per step " + "".join(f"{'lib' + str(i):>9}" for i in range(len(libs))))
    for o in ops:
        print(f"{o:<9}" + "".join(f"{h[o] / 5:>9.1f}" for _, _, h in res))
    print(f"{'total':<9}" + "".join(f"{sum(h.values()) / 5:>9.1f}" for _, _, h in res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python3
"""Static SASS opcode mix of the hot kernels, straight from the built library (cuobjdump -sass): which
instructions the sm_90a code consists of. usage: sass_mix.py [kernel-name-substring ...]"""
import collections, os, re, subprocess, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = os.path.join(ROOT, "monte-carlo-ray-tracer_b200", "libmcrt_b200.so")
want = sys.argv[1:] or ["k_extendIdLi2ELi2", "k_extendIdLi1ELi1", "k_shadowIdLb0ELi2ELi2", "k_shadeIdLi0ELb0ELj4294967282", "k_shadeIdLi0ELb0ELj4294967295",
                        "k_knnIdLi2ELb0ELj4294967282", "k_shade_keyId", "k_resolve_film_peers", "k_generateIdLb0"]
out = subprocess.run(["cuobjdump", "-sass", lib], capture_output=True, text=True).stdout
cur, mix = None, collections.OrderedDict()
for ln in out.splitlines():
    m = re.search(r"Function : (\S+)", ln)
    if m:
        cur = next((w for w in want if w in m.group(1)), None)
        if cur and cur not in mix:
            mix[cur] = (m.group(1), collections.Counter())
        elif cur and mix[cur][0] != m.group(1):
            cur = None
        continue
    if cur:
        m = re.match(r"\s+/\*[0-9a-f]+\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", ln)
        if m:
            mix[cur][1][m.group(1).split(".")[0]] += 1
print("Static SASS opcode mix (instruction counts in the kernel image, not execution counts), sm_90a, cuobjdump -sass of libmcrt_b200.so")
print("LDG/STG = global memory, LDL/STL = local memory (stacks, spills), DADD/DMUL/DFMA = float64 pipe, FFMA/FMNMX = the float32 box tests,")
print("REDUX/SHFL/VOTE/MATCH = warp collectives, ATOMG/RED = global atomics (queue appends, film)\n")
for key, (name, c) in mix.items():
    total = sum(c.values())
    print(f"{name}\n  {total} instructions: " + ", ".join(f"{op} {n}" for op, n in c.most_common(22)))
    groups = {"fp64": ["DADD", "DMUL", "DFMA", "DSETP", "MUFU"], "fp32": ["FFMA", "FMUL", "FADD", "FMNMX", "FSETP", "FSEL"], "global mem": ["LDG", "STG"], "local mem": ["LDL", "STL"],
              "warp collectives": ["SHFL", "VOTE", "VOTEU", "REDUX", "MATCH"], "atomics": ["ATOMG", "RED", "ATOMS", "ATOM"]}
    print("  " + ", ".join(f"{g} {sum(c[o] for o in ops)}" for g, ops in groups.items()) + "\n")

#!/usr/bin/env python3
"""Compare two builds kernel by kernel.

    python tools/sass_diff.py old.sass new.sass    # two `cuobjdump -sass libonesweep_b200.so` dumps
    python tools/sass_diff.py old.log new.log      # two ptxas reports (gpusorting_b200/csrc/build/*.ptxas.log)

Kernels are matched by name, so a different instantiation order does not count as a change.  In a SASS dump the
`identifier = <source path>` lines are dropped, so two checkouts in different directories compare equal; of a ptxas
report the registers, shared memory, stack and spills of each kernel are compared.  Prints the kernel counts and every
kernel that was added, removed or changed; exits 1 if there is any.
"""
import re
import sys


def sass_functions(text):
    out = {}
    for chunk in text.split("Function : ")[1:]:
        name, _, body = chunk.partition("\n")
        body = body.split("\nFatbin ")[0]  # the headers of the next object file follow the last function of each
        lines = [l.rstrip() for l in body.splitlines() if not re.match(r"\s*identifier\s*=", l)]
        out[name.strip()] = "\n".join(lines).strip()
    return out


def ptxas_functions(text):
    out, name = {}, None
    for line in text.splitlines():
        m = re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            name = m.group(1)
            out[name] = []
        elif name and re.search(r"Used \d+ registers|stack frame|spill", line):
            out[name].append(line.split(":", 1)[-1].strip())
    return {k: "\n".join(v) for k, v in out.items()}


def functions(path):
    text = open(path, encoding="utf-8", errors="replace").read()
    return ptxas_functions(text) if "Compiling entry function" in text else sass_functions(text)


def main(old_path, new_path):
    old, new = functions(old_path), functions(new_path)
    removed = sorted(old.keys() - new.keys())
    added = sorted(new.keys() - old.keys())
    changed = sorted(f for f in old.keys() & new.keys() if old[f] != new[f])
    print(f"{len(old)} kernels in {old_path}, {len(new)} in {new_path}")
    for label, names in (("removed", removed), ("added", added), ("changed", changed)):
        print(f"{label}: {len(names)}")
        for f in names:
            print(f"  {f}")
    return 1 if removed or added or changed else 0


if __name__ == "__main__":
    if len(sys.argv) != 3:
        sys.exit(__doc__)
    sys.exit(main(sys.argv[1], sys.argv[2]))

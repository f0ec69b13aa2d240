"""Compare the SASS of every kernel of one build of liblgrast.so with the same kernel in another (cuobjdump -sass, instruction by
instruction).  Kernels that gained a defaulted trailing flag (`DEPTH = false` of the blend kernels) or a defaulted trailing parameter
(`BlendDepth`, `BlendDepthBack`) are matched to their old names by demangling and dropping those.  Prints the kernels of the first
build that are missing from the second or whose SASS differs, and the kernels only the second has.

usage: python scripts/sass_diff.py OLD/liblgrast.so NEW/liblgrast.so"""
import re
import subprocess
import sys

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def functions(path):
    txt = subprocess.run([CUOBJDUMP, "-sass", path], capture_output=True, text=True, check=True).stdout
    out, name, body = {}, None, []
    for line in txt.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                out[name] = body
            name, body = m.group(1), []
        elif name is not None and ".section" not in line and "......" not in line:
            body.append(re.sub(r"\s+", " ", line.strip()))
    if name:
        out[name] = body
    return out


def demangle(names):
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True, check=True).stdout.split("\n")
    return dict(zip(names, r))


def normalise(d):
    d = d.replace(", (anonymous namespace)::BlendDepthBack)", ")").replace(", (anonymous namespace)::BlendDepth)", ")")
    d = re.sub(r"(blend_forward_ring_kernel<(?:(?:true|false), ){3}(?:true|false)), false>", r"\1>", d)
    return re.sub(r"(blend_backward_ring_kernel<(?:true|false)), false>", r"\1>", d)


def main(old_path, new_path):
    old, new = functions(old_path), functions(new_path)
    dn_old, dn_new = demangle(list(old)), demangle(list(new))
    old_by = {normalise(dn_old[k]): v for k, v in old.items()}
    new_by = {normalise(dn_new[k]): v for k, v in new.items()}
    missing = [k for k in old_by if k not in new_by]
    differ = [k for k in old_by if k in new_by and old_by[k] != new_by[k]]
    print(f"kernels in {old_path}: {len(old_by)}; missing in {new_path}: {len(missing)}; differing SASS: {len(differ)}")
    for k in missing:
        print("missing:", k)
    for k in differ:
        print("differs:", k)
    for k in (k for k in new_by if k not in old_by):
        print("new:", k)
    return 1 if missing or differ else 0


if __name__ == "__main__":
    sys.exit(main(*sys.argv[1:3]))

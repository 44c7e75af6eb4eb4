"""Compare the SASS of two object files (or shared libraries) kernel by kernel.

Kernels are matched by demangled name, with the row element-type template argument `float` dropped from the new
names (`genconv_aggregate_kernel<float, 4, 1, ...>` -> `genconv_aggregate_kernel<4, 1, ...>`), so the fp32
instantiations of a kernel that gained that parameter are compared with the kernel as it was.  Instruction text is
compared without addresses' encodings.

    python tools/sass_diff.py OLD.o NEW.o [name substring]
"""
import re
import subprocess
import sys

CUDA = "/usr/local/cuda/bin/"


def kernels(obj):
    out = subprocess.run([CUDA + "cuobjdump", "-sass", obj], capture_output=True, text=True, check=True).stdout
    res, name, body = {}, None, []
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            if name:
                res[name] = body
            name, body = m.group(1), []
        elif name and re.match(r"\s*/\*[0-9a-f]{4,}\*/", line):
            body.append(re.sub(r"\s*/\* 0x[0-9a-f]+ \*/\s*$", "", line).strip())
    if name:
        res[name] = body
    names = subprocess.run([CUDA + "cu++filt"], input="\n".join(res), capture_output=True, text=True).stdout.split("\n")
    return {normalise(d): res[m] for m, d in zip(res, names)}


def normalise(name):
    name = re.sub(r"^void ", "", name)
    # the trailing template flag the GENConv kernels gained last (KEEP of the aggregate: 7th argument, PRE of its
    # backward: 3rd) is false for every kernel that existed before it
    m = re.match(r"^(?:dgcn::)?genconv_aggregate(_bwd)?_kernel<([^>]*)>", name)
    if m and m.group(2).endswith(", (bool)0") and len(m.group(2).split(",")) == (3 if m.group(1) else 7):
        name = name.replace(m.group(2), m.group(2)[:-len(", (bool)0")], 1)
    name = name.replace("<float, ", "<")
    return re.sub(r"<float>\(const T1 \*, (.*), T1 \*\)", r"(const float *, \1, float *)", name)


def main():
    old, new = kernels(sys.argv[1]), kernels(sys.argv[2])
    same = [k for k in old if new.get(k) == old[k]]
    differ = [k for k in old if k in new and new[k] != old[k]]
    missing = [k for k in old if k not in new]
    for k in differ:
        print("DIFFERENT", k)
    for k in missing:
        print("MISSING  ", k)
    print("%d kernels in OLD: %d identical, %d different, %d missing; %d only in NEW"
          % (len(old), len(same), len(differ), len(missing), len(set(new) - set(old))))
    if len(sys.argv) > 3:
        import difflib
        k = next(k for k in differ if sys.argv[3] in k)
        print("\n".join(difflib.unified_diff(old[k], new[k], "OLD " + k, "NEW", lineterm="", n=1)))


if __name__ == "__main__":
    main()

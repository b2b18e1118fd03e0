"""Compare the SASS of two builds kernel by kernel:  python tools/sass_diff.py old.o new.o   (objects or libcl3d.so)

Dumps both with `cuobjdump -sass`, drops the /*address*/ prefixes and the encoding comments, and prints the kernels
found in only one file and the kernels whose instruction text differs, with the instruction count on each side.
Exit status 0 when every kernel present in both files is identical, 1 otherwise."""
import re
import subprocess
import sys


def kernels(path):
    out = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    funcs, cur = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        m = re.match(r"\s*/\*[0-9a-f]{4,}\*/\s*(.*?)\s*;", line)
        if m and cur is not None:
            cur.append(m.group(1))
    return funcs


def demangle(names):
    r = subprocess.run(["cu++filt"], input="\n".join(names), capture_output=True, text=True)
    return dict(zip(names, r.stdout.splitlines())) if r.returncode == 0 else {n: n for n in names}


def main(old_path, new_path):
    old, new = kernels(old_path), kernels(new_path)
    names = demangle(sorted(set(old) | set(new)))
    only_old = sorted(k for k in old if k not in new)
    only_new = sorted(k for k in new if k not in old)
    differ = sorted(k for k in old if k in new and old[k] != new[k])
    for title, ks in ((f"only in {old_path}", only_old), (f"only in {new_path}", only_new)):
        print(f"{title}: {len(ks)}")
        for k in ks:
            print(f"  {names[k]}")
    print(f"differ: {len(differ)} of {len(set(old) & set(new))}")
    for k in differ:
        print(f"  {names[k]}: {len(old[k])} -> {len(new[k])} instructions")
    return 1 if differ else 0


if __name__ == "__main__":
    sys.exit(main(*sys.argv[1:3]))

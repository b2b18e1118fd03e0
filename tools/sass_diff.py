"""Compare the SASS of two builds kernel by kernel:  python tools/sass_diff.py old.o new.o   (objects or libcl3d.so)

Dumps both with `cuobjdump -sass`, drops the /*address*/ prefixes and the encoding comments, and prints the kernels
found in only one file and the kernels whose instruction text differs, with the instruction count on each side.
A kernel found in only one file whose instruction text equals that of a kernel found only in the other is listed as
renamed (a template parameter added to a kernel renames its existing instance without changing its code).
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
    by_code = {}
    for k in only_new:
        by_code.setdefault(tuple(new[k]), []).append(k)
    renamed = [(k, by_code[tuple(old[k])].pop(0)) for k in only_old if by_code.get(tuple(old[k]))]
    only_old = [k for k in only_old if k not in {a for a, _ in renamed}]
    only_new = [k for k in only_new if k not in {b for _, b in renamed}]
    print(f"renamed, same instructions: {len(renamed)}")
    for a, b in renamed:
        print(f"  {names[a]}  ->  {names[b]}")
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

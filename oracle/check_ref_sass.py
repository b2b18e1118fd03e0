#!/usr/bin/env python
"""Check (container only) that the sm_90 SASS nvcc emits for the reference's distance expression is
    FADD dy ; FADD dx ; FMUL t=dy*dy ; FADD dz ; FFMA t=dx*dx+t ; FFMA t=dz*dz+t
i.e. d2 = fma(dz,dz, fma(dx,dx, dy*dy)) with d = query - support, which is what oracle/cl3d_oracle.c (ref_d2)
and closerlook3d_b200/csrc/common.cuh (ref_d2) spell out.  Needs oracle/_ref/obj (run oracle/build_ref.py).
TEST INFRASTRUCTURE ONLY."""
import os
import re
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def main():
    ok = True
    for name in ("masked_ordered_ball_query_gpu.cu.o", "masked_nearest_query_gpu.cu.o"):
        obj = os.path.join(HERE, "_ref", "obj", name)
        if not os.path.exists(obj):
            print("missing", obj, "- run oracle/build_ref.py first")
            return 2
        sass = subprocess.run(["cuobjdump", "-sass", obj], capture_output=True, text=True).stdout
        ops = re.findall(r"\b(FADD|FMUL|FFMA) (R\d+), (-?R\d+)(?:\.reuse)?, (-?R\d+)(?:\.reuse)?(?:, (-?R\d+))?", sass)
        # find the first FMUL x*x followed by two FFMA a*a+t chains
        seq = [o[0] for o in ops]
        found = False
        for i in range(len(ops) - 2):
            if ops[i][0] == "FMUL" and ops[i][2] == ops[i][3]:
                later = [o for o in ops[i + 1:i + 6] if o[0] == "FFMA" and o[2] == o[3]]
                if len(later) >= 2:
                    found = True
                    break
        print(name, "FMUL sq + 2 chained FFMA sq:", found)
        ok &= found
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())

"""Records tests/golden/geometry_order_border.npz: what UpdateSurfelActivation + one OptimizeGeometryIteration compute on the
border scene of tests/test_gpu_geometry_order.py, in depth-only, descriptor-only and combined mode, with the library of the tree
this script is run from.  The committed fixture was recorded from a checkout of commit 5e2691d, the last one whose geometry
kernels visit the surfels in the caller's order and cull nothing (copy this script and tests/test_gpu_geometry_order.py into that
checkout, build it, then run from its root):

    python tools/record_geometry_order_border.py tests/golden/geometry_order_border.npz

Stored: every placed border surfel and a seeded sample of 1000 of the scene's own, as `columns` plus, per mode "<depth><desc>",
the flags after the activation (`_flags_act`), rows 0-7 (`_rows`) and the flags (`_flags`) after the geometry iteration.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def main():
    import numpy as np
    from badslam_b200 import scene as S
    from badslam_b200.direct_ba import DirectBA
    import test_gpu_geometry_order as T
    base = S.make_scene(S.config_by_name("many"))
    sc = T.border_scene(S, base)
    n0, n = base.num_surfels, sc.num_surfels
    cols = np.sort(np.concatenate([np.random.default_rng(3).choice(n0, 1000, replace=False), np.arange(n0, n)]))
    out = {"columns": cols.astype(np.int32)}
    for use_depth, use_desc in T.MODES:
        mode = f"{int(use_depth)}{int(use_desc)}"
        flags_act, rows, flags = T.activation_and_geometry(DirectBA, sc, use_depth, use_desc)
        out[mode + "_flags_act"], out[mode + "_rows"], out[mode + "_flags"] = flags_act[cols], rows[:, cols], flags[cols]
    np.savez_compressed(sys.argv[1], **out)
    print("wrote", sys.argv[1], "columns", len(cols))


if __name__ == "__main__":
    main()

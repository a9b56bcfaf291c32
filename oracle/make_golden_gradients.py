"""TEST INFRASTRUCTURE ONLY -- tests/golden/gradients_im_function.npz: 8 frames of the UNMODIFIED reference's
scripts/gradients.py::im_function (:117-140) at 346x260, bench.py's config-2 parameters (background 127,
contrast 2, bump width 0.5, 300 px/s), sampled at 30 fps.

    V2E_REFERENCE_ROOT=<reference checkout> python oracle/make_golden_gradients.py
"""
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import ref_shim  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests", "golden",
                   "gradients_im_function.npz")


def main():
    ref_shim.load_reference()
    sys.path.insert(0, os.path.join(ref_shim.REFERENCE_ROOT, "scripts"))
    import gradients as g
    m = g.gradients.__new__(g.gradients)          # im_function only needs these attributes (gradients.py:117-140)
    m.bg, m.contrast, m.bump_width, m.w, m.h, m.speed_pps = 127, 2.0, 0.5, 346, 260, 300.0
    frames = np.stack([np.asarray(m.im_function(np.arange(260)[:, None], np.arange(346)[None, :], k / 30.0))
                       for k in range(8)])
    np.savez_compressed(OUT, frames=frames)
    print(OUT, frames.shape, frames.dtype)


if __name__ == "__main__":
    main()

"""Build check of sass_identity.py for csrc/td_vae.cu: the kernels a base revision of td_vae.cu had compile to the same SASS,
instruction for instruction, in the working tree; and the -Xptxas -v registers and spills of the kernels the tree adds.

    python tests/debug_tools/sass_identity_vae.py [--base HEAD~1]
"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import sass_identity  # noqa: E402

sass_identity.SRC = "multidiffusion_upscaler_for_automatic1111_b200/csrc/td_vae.cu"

if __name__ == "__main__":
    sass_identity.main()

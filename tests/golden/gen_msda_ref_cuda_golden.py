"""Regenerates refcuda_msda_*.npz: outputs of the reference's own CUDA forward kernel (oracle/_ref/libref_msda.so, built by
oracle/Makefile from the reference checkout) on the seeded inputs of tests/test_msda_gpu.py's reference-kernel tests,
sampled along the query axis so each file stays under 1 MB.  Needs a GPU; run from the repository root."""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import msda as O  # noqa: E402

L5_1024 = [(256, 256), (128, 128), (64, 64), (32, 32), (16, 16)]
DEC_STEP, ENC_STEP = 4, 256  # query sampling of the stored outputs


def main(out_dir=HERE):
    assert O.have_ref_cuda(), "oracle/_ref/libref_msda.so is not built"
    for dtype, tag in ((torch.float32, "f32"), (torch.float16, "f16")):
        ins = [t.to("cuda") for t in O.make_inputs(2, 900, 8, 32, L5_1024, 4, seed=3, border=True)]
        ins = [t.to(dtype) if t.is_floating_point() else t for t in ins]
        ref = O.ref_cuda(*ins)
        np.savez_compressed(os.path.join(out_dir, f"refcuda_msda_decoder_{tag}.npz"), out=ref[:, ::DEC_STEP].float().cpu().numpy())
    S = sum(h * w for h, w in L5_1024)
    ins = [t.to("cuda") for t in O.make_inputs(1, S, 8, 32, L5_1024, 4, seed=3, border=True)]
    ref = O.ref_cuda(*ins)
    np.savez_compressed(os.path.join(out_dir, "refcuda_msda_encoder_f32.npz"), out=ref[:, ::ENC_STEP].cpu().numpy())


if __name__ == "__main__":
    main(*sys.argv[1:])

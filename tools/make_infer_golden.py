"""Generates tests/golden/infer_bf16_attn.npz: the UNMODIFIED reference (ae.py) converted with `.bfloat16()` and run
without autograd exactly like its model card ("How to use": `z = vae.encoder(img).clamp(-8.0, 8.0)`,
`decz = vae.decoder(z)`), on a small seeded model with the mid-block attention and a non-square image. TEST
INFRASTRUCTURE, run where the reference tree is available; the fixture is committed.

    VQB_REFERENCE=/path/to/reference python tools/make_infer_golden.py

The reference is imported through oracle/make_golden.py (same stubs, same AttnBlock swap as the vae_attn fixture). The
weights are `seeded.fill_state_dict(..., "infer_bf16_attn")` rounded to bf16; the image is
`seeded.tensor("infer_bf16_attn/x", (1, 3, 32, 48), 1.0, "uniform")` rounded to bf16. Before writing, the oracle
restatement run in bf16 on the same bf16 weights must agree with the reference (tests/test_infer_golden.py repeats that
check); both are stored as float32 arrays holding bf16 values.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from oracle import make_golden as MG  # noqa: E402  (imports the reference with the stubs it needs)
from oracle import seeded  # noqa: E402
from oracle import vae_oracle as VO  # noqa: E402

NAME = "infer_bf16_attn"
CFG = VO.VAEConfig(resolution=32, ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=4, use_attn=True)
SHAPE = (1, 3, 32, 48)
ORACLE_TOL = 4e-2  # bf16 arithmetic: the reference's SDPA vs the oracle's explicit softmax, other summation orders (~2e-2)


def main():
    cfg = CFG
    ref = MG.ref_ae.VAE(resolution=cfg.resolution, in_channels=3, ch=cfg.ch, out_ch=3, ch_mult=list(cfg.ch_mult),
                        num_res_blocks=cfg.num_res_blocks, z_channels=cfg.z_channels, use_attn=False,
                        decoder_also_perform_hr=False, use_wavelet=False)
    c = cfg.ch * cfg.ch_mult[-1]
    ref.encoder.mid.attn_1 = MG.ref_ae.AttnBlock(c)
    ref.decoder.mid.attn_1 = MG.ref_ae.AttnBlock(c)
    sd = seeded.fill_state_dict(ref.state_dict(), NAME)
    ref.load_state_dict(sd)
    ref = ref.bfloat16().eval()
    x = seeded.tensor(NAME + "/x", SHAPE, 1.0, "uniform").bfloat16()
    with torch.no_grad():
        z = ref.encoder(x).clamp(-8.0, 8.0)
        dec = ref.decoder(z)
        sdb = {k: v.bfloat16() for k, v in sd.items()}
        oz = VO.encoder_forward(sdb, x, cfg).clamp(-8.0, 8.0)
        odec = VO.decoder_forward(sdb, oz, cfg)
    assert z.dtype == dec.dtype == torch.bfloat16
    MG.close(oz.float(), z.float(), ORACLE_TOL, NAME + " z")
    MG.close(odec.float(), dec.float(), ORACLE_TOL, NAME + " dec")
    MG.save(NAME, z=z.float(), dec=dec.float(), x=x.float(), tag=NAME)


if __name__ == "__main__":
    main()
    MG.dist.destroy_process_group()

"""CPU: the oracle restatement run in bf16 (no autograd) reproduces the reference's bf16 model-card inference
(tests/golden/infer_bf16_attn.npz, written by tools/make_infer_golden.py from the unmodified reference)."""
import torch

from helpers import golden, rel_l2, seeded_sd
from oracle import seeded
from oracle import vae_oracle as VO

CFG = VO.VAEConfig(resolution=32, ch=32, ch_mult=(1, 2), num_res_blocks=1, z_channels=4, use_attn=True)
# bf16 arithmetic on both sides, the reference's SDPA vs the oracle's explicit softmax: measured ~2e-2 when written
TOL = 4e-2


def test_oracle_bf16_matches_reference_inference_golden():
    g = golden("infer_bf16_attn")
    x = seeded.tensor("infer_bf16_attn/x", (1, 3, 32, 48), 1.0, "uniform").bfloat16()
    assert torch.equal(x.float(), torch.from_numpy(g["x"]))
    sd = {k: v.bfloat16() for k, v in seeded_sd(VO.state_dict_shapes(CFG), "infer_bf16_attn").items()}
    with torch.no_grad():
        z = VO.encoder_forward(sd, x, CFG).clamp(-8.0, 8.0)
        dec = VO.decoder_forward(sd, z, CFG)
    assert z.dtype == dec.dtype == torch.bfloat16
    assert z.shape == g["z"].shape == (1, 4, 16, 24) and dec.shape == g["dec"].shape == (1, 3, 32, 48)
    ez, ed = rel_l2(z, g["z"]), rel_l2(dec, g["dec"])
    print(f"\noracle bf16 vs reference bf16: z rel {ez:.3e}  dec rel {ed:.3e}")
    assert ez < TOL and ed < TOL

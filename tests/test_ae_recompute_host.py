"""CPU: ResnetBlock recompute of the image autoencoder (ae.enable_recompute, Trainer(..., recompute=True)) without a
device: the flags, the Trainer's default and the saved-activation prediction of tools/train_mem_bench.py."""
import inspect
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _vae(hr=False):
    import ae

    return ae.VAE(resolution=32, in_channels=3, ch=32, out_ch=3, ch_mult=[1, 2], num_res_blocks=1, z_channels=4,
                  use_attn=True, decoder_also_perform_hr=hr, use_wavelet=False)


def _blocks(m):
    import ae

    return [s for s in m.modules() if isinstance(s, ae.ResnetBlock)]


def test_enable_recompute_flags_every_resnet_block_and_nothing_else():
    import ae

    for hr in (False, True):
        torch.manual_seed(5)
        m = _vae(hr)
        torch.manual_seed(5)
        ref = _vae(hr)
        assert ae.enable_recompute(m) is m
        blocks = _blocks(m)
        levels, nrb = 2 + hr, 1
        assert len(blocks) == (2 * nrb + 2) + (2 + levels * (nrb + 1))  # encoder levels + mid, decoder mid + levels
        assert all(b._vqb_recompute for b in blocks)
        assert len(_blocks(m.decoder.up[levels - 1])) == nrb + 1  # the HR decoder's extra level (or the top level)
        others = [s for s in m.modules() if not isinstance(s, ae.ResnetBlock)]
        assert not any(hasattr(s, "_vqb_recompute") for s in others)
        sd, sr = m.state_dict(), ref.state_dict()
        assert list(sd) == list(sr) and all(torch.equal(sd[k], sr[k]) for k in sd)
        assert ae.enable_recompute(m, enabled=False) is m
        assert not any(b._vqb_recompute for b in blocks)
        ae.enable_recompute(m.decoder)
        assert all(b._vqb_recompute for b in _blocks(m.decoder))
        assert not any(b._vqb_recompute for b in _blocks(m.encoder))


def test_trainer_defaults_to_no_recompute():
    import vae_trainer as vt

    assert inspect.signature(vt.Trainer).parameters["recompute"].default is False
    kw = dict(vae_resolution=32, vae_ch=32, vae_ch_mult="1,2", vae_num_res_blocks=1, vae_z_channels=4, max_steps=10,
              decoder_also_perform_hr=True)
    plain = vt.Trainer("cpu", **kw)
    assert not any(getattr(b, "_vqb_recompute", False) for b in _blocks(plain.vae.module))
    rc = vt.Trainer("cpu", recompute=True, **kw)
    assert all(b._vqb_recompute for b in _blocks(rc.vae.module))
    assert not any(hasattr(s, "_vqb_recompute") for s in rc.discriminator.modules())
    sp, sr = plain.vae.state_dict(), rc.vae.state_dict()  # same seed, same initialisation
    assert all(torch.equal(sp[k], sr[k]) for k in sp)


def test_saved_activation_prediction_matches_a_hand_count():
    sys.path.insert(0, os.path.join(ROOT, "tools"))
    import train_mem_bench as tb

    # ch=32, ch_mult (1, 2), one block per level, z=4, batch 2; encoder 16x16, decoder 16x16 (32x32 with hr)
    N, rec = 2, 2 * 2 * 32 * 2 * 4  # two [N, 32, 2] fp32 GroupNorm records per block

    def act(c, px):
        return 2 * c * px * N

    def block(cin, cout, px, recompute):
        return act(cin, px) + rec if recompute else 2 * act(cin, px) + 2 * act(cout, px) + rec

    for recompute in (False, True):
        enc = (act(8, 256) + block(32, 32, 256, recompute) + act(32, 256) + block(32, 64, 64, recompute)
               + 2 * block(64, 64, 64, recompute) + 2 * act(64, 64))
        dec = (act(8, 64) + 2 * block(64, 64, 64, recompute) + 2 * block(64, 64, 64, recompute) + act(64, 64)
               + block(64, 32, 256, recompute) + block(32, 32, 256, recompute) + 2 * act(32, 256))
        assert tb.saved_activation_bytes(32, [1, 2], 1, 4, False, N, 16, 16, recompute) == enc + dec
        # hr: a third decoder level at ch * 4 = 128 channels; 8x8 latent -> 16x16 -> 32x32
        dec_hr = (act(8, 64) + 2 * block(128, 128, 64, recompute)
                  + 2 * block(128, 128, 64, recompute) + act(128, 64)
                  + block(128, 64, 256, recompute) + block(64, 64, 256, recompute) + act(64, 256)
                  + block(64, 32, 1024, recompute) + block(32, 32, 1024, recompute) + 2 * act(32, 1024))
        assert tb.saved_activation_bytes(32, [1, 2], 1, 4, True, N, 16, 32, recompute) == enc + dec_hr
    assert tb.saved_activation_bytes(32, [1, 2], 1, 4, False, N, 16, 16, True) < \
        tb.saved_activation_bytes(32, [1, 2], 1, 4, False, N, 16, 16, False) / 2

"""CPU: the host side of data-parallel video training (tae_trainer.train_video). The CLI parses and lists its options;
the synthetic clip stream is deterministic per (seed, rank), distinct between ranks, of the requested shape and in
[-1, 1]; bad arguments are refused before anything touches a device."""
import pytest
import torch
import torch.distributed as dist
from click.testing import CliRunner

OPTIONS = ["--vae_ch", "--vae_ch_mult", "--vae_num_res_blocks", "--vae_z_channels", "--do_ganloss", "--disc_type",
           "--use_lecam", "--learning_rate_vae", "--learning_rate_disc", "--max_steps", "--batch_size", "--load_path",
           "--run_name", "--evaluate_every_n_steps", "--clip_frames", "--resolution", "--perceptual_frames",
           "--recompute", "--no_lpips", "--seed"]


def test_help_lists_every_option():
    import tae_trainer

    res = CliRunner().invoke(tae_trainer.train_video, ["--help"])
    assert res.exit_code == 0, res.output
    missing = [o for o in OPTIONS if o not in res.output]
    assert not missing, missing


def test_cli_parses_a_full_command_line(monkeypatch):
    import tae_trainer

    seen = {}
    monkeypatch.setattr(tae_trainer, "_train_video", lambda *a: seen.update(args=a))
    monkeypatch.setattr(torch.cuda, "is_available", lambda: True)
    monkeypatch.setattr(torch.cuda, "set_device", lambda d: None)
    monkeypatch.delenv("RANK", raising=False)
    argv = ["--vae_ch", "32", "--vae_ch_mult", "1,8", "--vae_num_res_blocks", "1", "--vae_z_channels", "4",
            "--clip_frames", "4", "--resolution", "32", "--batch_size", "2", "--perceptual_frames", "2",
            "--do_ganloss", "--disc_type", "hinge", "--use_lecam", "True", "--recompute", "--no_lpips",
            "--learning_rate_vae", "3e-4", "--learning_rate_disc", "5e-4", "--max_steps", "7",
            "--evaluate_every_n_steps", "3", "--load_path", "w.pt", "--run_name", "r", "--seed", "9"]
    res = CliRunner().invoke(tae_trainer.train_video, argv)
    assert res.exit_code == 0, res.output
    rank, device = seen["args"][:2]
    assert rank == 0 and device == torch.device("cuda:0")
    assert seen["args"][2:] == (2, 4, 32, 2, True, "hinge", True, True, True, 3e-4, 5e-4, 32, [1, 8], 1, 4, 7, 3,
                                "w.pt", "r", 9)


def _clips(seed, rank, monkeypatch, **kw):
    import vae_trainer

    monkeypatch.setenv("RANK", str(rank))
    it = iter(vae_trainer.SyntheticLoader(2, 24, seed=seed, n_distinct=3, frames=5, **kw))
    return [next(it)[0].clone() for _ in range(4)]


def test_synthetic_clips_are_per_rank_and_deterministic(monkeypatch):
    r0, r0b, r1 = _clips(None, 0, monkeypatch), _clips(None, 0, monkeypatch), _clips(None, 1, monkeypatch)
    for c in r0 + r1:
        assert c.shape == (2, 3, 5, 24, 24) and c.dtype == torch.float32
        assert float(c.min()) >= -1 and float(c.max()) <= 1
    assert all(torch.equal(a, b) for a, b in zip(r0, r0b)), "the stream is not deterministic for one rank"
    assert not any(torch.equal(a, b) for a, b in zip(r0, r1)), "two ranks draw the same clips"
    assert torch.equal(r0[3], r0[0]) and not torch.equal(r0[0], r0[1])  # n_distinct=3 clips, cycled
    # the default seed is 42 + rank, the seed of the image stream
    assert all(torch.equal(a, b) for a, b in zip(r1, _clips(43, 0, monkeypatch)))
    # the image stream is unchanged by the frames argument
    import vae_trainer

    img = next(iter(vae_trainer.SyntheticLoader(2, 24, seed=5, n_distinct=1)))[0]
    g = torch.Generator().manual_seed(5)
    assert torch.equal(img, torch.rand(2, 3, 24, 24, generator=g) * 2 - 1)


@pytest.mark.parametrize("argv, match", [
    (["--clip_frames", "8", "--perceptual_frames", "9"], "perceptual_frames"),
    (["--perceptual_frames", "0"], "perceptual_frames"),
    (["--disc_type", "wgan"], "disc_type"),
    (["--vae_ch_mult", "1,x"], "vae_ch_mult"),
    (["--vae_ch_mult", "1,2,4", "--clip_frames", "6"], "multiples of 4"),
])
def test_bad_arguments_are_refused_before_device_work(argv, match, monkeypatch):
    import tae_trainer

    def device_work(*a, **k):
        raise AssertionError("device work before the arguments were checked")

    monkeypatch.setattr(torch.cuda, "is_available", device_work)
    monkeypatch.setattr(torch.cuda, "set_device", device_work)
    monkeypatch.setattr(dist, "init_process_group", device_work)
    monkeypatch.setattr(tae_trainer, "_train_video", device_work)
    res = CliRunner().invoke(tae_trainer.train_video, argv)
    assert res.exit_code == 2, (res.exit_code, res.output, res.exception)
    assert match in res.output

"""VideoToVideo_sr.enhance_frames_iter refuses the setups it does not serve before it reads the input or does any device work:
a process group of more than one rank (the streamed decode is not sharded; enhance_frames is) and a pipeline without a GPU."""
import pytest
import torch

from tests.test_pipeline_cpu import make_pipe


class Untouched(dict):
    """an input dict that fails on any read"""

    def __getitem__(self, key):
        raise AssertionError(f"input[{key!r}] was read")


class Forbidden:
    """a pipeline member that fails on any use"""

    def __init__(self, name):
        self.name = name

    def __getattr__(self, attr):
        raise AssertionError(f"{self.name}.{attr} was used")

    def __call__(self, *a, **k):
        raise AssertionError(f"{self.name} was called")


def forbidden_pipe(device):
    pipe = make_pipe()
    pipe.device = torch.device(device)
    pipe.vae, pipe.generator, pipe.text_encoder = Forbidden("vae"), Forbidden("generator"), Forbidden("text_encoder")
    return pipe


def test_iter_refuses_two_ranks_before_device_work(monkeypatch):
    from star_b200.video_to_video import video_to_video_model as M
    monkeypatch.setattr(M, "_dist_info", lambda: (2, 0))
    pipe = forbidden_pipe("cuda")
    with pytest.raises(NotImplementedError, match="enhance_frames"):
        pipe.enhance_frames_iter(Untouched(), steps=1)


def test_iter_refuses_a_pipeline_without_gpu():
    with pytest.raises(NotImplementedError, match="GPU"):
        forbidden_pipe("cpu").enhance_frames_iter(Untouched(), steps=1)

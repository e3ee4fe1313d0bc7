"""Batched panorama inference, host side (no GPU): the argument checks of split_panoramas, merge_panoramas, finish_panoramas and
infer_panoramas fail with MogeError before any device work, and the C library's batch limit is the Python one."""
import pytest
import torch

from moge_b200 import capi
from moge_b200 import panorama as P
from moge_b200.capi import MogeError


def test_split_panoramas_checks():
    assert capi.PANORAMA_MAX_BATCH == P.MAX_BATCH == 64
    imgs = torch.zeros(2, 64, 128, 3, dtype=torch.uint8)
    with pytest.raises(MogeError, match="CUDA"):
        P.split_panoramas(imgs)
    with pytest.raises(MogeError, match="uint8"):
        P.split_panoramas(imgs.float())
    with pytest.raises(MogeError, match=r"\(P, H, W, 3\)"):
        P.split_panoramas(imgs[0])
    with pytest.raises(MogeError, match=r"\(P, H, W, 3\)"):
        P.split_panoramas(imgs[..., :2])
    with pytest.raises(MogeError, match=r"outside \[1, 64\]"):
        P.split_panoramas(imgs[:0])
    with pytest.raises(MogeError, match=r"batch of 65 panoramas is outside \[1, 64\]"):
        P.split_panoramas(torch.zeros(65, 2, 2, 3, dtype=torch.uint8))
    with pytest.raises(MogeError, match="outside"):
        P.split_panoramas(torch.zeros(2, 1, 128, 3, dtype=torch.uint8))


def test_merge_panoramas_checks():
    dist, mask = torch.ones(2, 12, 8, 8), torch.ones(2, 12, 8, 8, dtype=torch.bool)
    with pytest.raises(MogeError, match="CUDA"):
        P.merge_panoramas(64, 32, dist, mask)
    with pytest.raises(MogeError, match="mask"):
        P.merge_panoramas(64, 32, dist, mask[:, :, :, :7])
    with pytest.raises(MogeError, match="mask"):
        P.merge_panoramas(64, 32, dist, mask[:1])
    with pytest.raises(MogeError, match="float32"):
        P.merge_panoramas(64, 32, dist.double(), mask)
    with pytest.raises(MogeError, match="float32"):
        P.merge_panoramas(64, 32, dist[0], mask[0])                   # a single panorama's rank
    with pytest.raises(MogeError, match="float32"):
        P.merge_panoramas(64, 32, torch.ones(2, 12, 8, 8, 2), mask)
    with pytest.raises(MogeError, match=r"outside \[1, 64\]"):
        P.merge_panoramas(64, 32, dist[:0], mask[:0])
    with pytest.raises(MogeError, match=r"outside \[1, 64\]"):
        P.merge_panoramas(64, 32, torch.ones(65, 12, 2, 2), torch.ones(65, 12, 2, 2, dtype=torch.bool))
    with pytest.raises(MogeError, match="outside"):
        P.merge_panoramas(1, 32, dist, mask)


def test_finish_and_infer_panoramas_checks():
    depth, mask = torch.ones(2, 16, 32), torch.ones(2, 16, 32, dtype=torch.bool)
    with pytest.raises(MogeError, match="CUDA"):
        P.finish_panoramas(depth, mask, 32, 64)
    with pytest.raises(MogeError, match="depth"):
        P.finish_panoramas(depth, mask[:1], 32, 64)
    with pytest.raises(MogeError, match=r"outside \[1, 64\]"):
        P.finish_panoramas(depth[:0], mask[:0], 32, 64)
    imgs = torch.zeros(2, 64, 128, 3, dtype=torch.uint8)
    with pytest.raises(MogeError, match="batch_size"):
        P.infer_panoramas(None, imgs, batch_size=0)
    with pytest.raises(MogeError, match="CUDA"):
        P.infer_panoramas(None, imgs)
    with pytest.raises(MogeError, match="uint8"):
        P.infer_panoramas(None, imgs.float())
    with pytest.raises(MogeError, match=r"\(P, H, W, 3\)"):
        P.infer_panoramas(None, imgs[0])
    with pytest.raises(MogeError, match=r"outside \[1, 64\]"):
        P.infer_panoramas(None, torch.zeros(65, 2, 2, 3, dtype=torch.uint8))

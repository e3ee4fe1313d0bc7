"""-m gpu: the engine's weight loading (weights.cu).  Every weight is checked against its full shape before a load-time launch reads
it, and finalize frees each fp32 staging weight that no kernel reads at run time while keeping every one a plan reads."""
import re

import pytest
import torch

from moge_b200 import capi
from moge_b200.configs import model_config, v1_model_config
from moge_b200.synthetic import make_state_dict, make_v1_state_dict, synthetic_images

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


def _v2(sd):
    from moge.model.v2 import MoGeModel
    m = MoGeModel(**model_config("vits", True))
    m.load_state_dict(sd)
    return m.to(DEV).eval()


def _v1(sd):
    from moge.model.v1 import MoGeModel
    m = MoGeModel(**v1_model_config("vits"))
    m.load_state_dict(sd)
    return m.to(DEV).half()


@pytest.fixture(scope="module")
def v2_weights():
    return make_state_dict(model_config("vits", True), 0, well_posed=True)


@pytest.fixture(scope="module")
def image():
    return synthetic_images(1, 70, 98, 3).to(DEV)


@pytest.mark.parametrize("name", ["mlp.fc2.weight", "attn.qkv.weight", "mlp.fc1.weight"])
def test_transposed_linear_is_rejected(name, v2_weights, image):
    """A transposed encoder linear has the right numel and correct biases, so only the shape check can catch it."""
    key = f"encoder.backbone.blocks.3.{name}"
    bad = dict(v2_weights)
    bad[key] = v2_weights[key].t().contiguous()
    m = _v2(bad)
    with pytest.raises(capi.MogeError, match=re.escape(f"weight '{key}' has shape")):
        m.forward(image, 100)
    m.load_state_dict(v2_weights)                 # the same model with the right weight loads and runs
    out = m.forward(image, 100)
    ref = _v2(v2_weights).forward(image, 100)
    torch.cuda.synchronize()
    for k, v in ref.items():
        assert torch.equal(out[k], v), k


@pytest.mark.parametrize("version", [2, 1])
def test_freed_staging_weights_are_not_read(version, v2_weights, image):
    """Fill newly allocated device memory, which may take the place of the staging weights finalize freed, with NaN: a forward that
    read a freed weight would change, so the output before and after the fill must be bitwise equal."""
    if version == 2:
        m = _v2(v2_weights)
    else:
        m = _v1(make_v1_state_dict(v1_model_config("vits"), 0, well_posed=True))
    m.forward(image, 100)                         # the first call runs eagerly, the later ones replay the plan's graph
    before = {k: v.clone() for k, v in m.forward(image, 100).items()}
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    fill = [torch.full((1 << 19,), float("nan"), device=DEV) for _ in range(512)]      # 512 x 2 MiB = 1 GiB
    torch.cuda.synchronize()
    after = m.forward(image, 100)
    torch.cuda.synchronize()
    del fill
    torch.cuda.empty_cache()
    for k, v in before.items():
        assert torch.isfinite(v).all(), k
        assert torch.equal(after[k], v), k

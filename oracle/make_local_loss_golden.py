"""Generate tests/golden/local_loss.pt from the UNMODIFIED reference `moge.train.losses.affine_invariant_local_loss` (CPU, fp32).

    MOGE_REFERENCE=<checkout of microsoft/MoGe> python oracle/make_local_loss_golden.py

utils3d resolves to the stand-in under oracle/utils3d_shim, with `masked_nearest_resize` from oracle/utils3d_metrics.py.  Inputs
come from moge_b200.synthetic.synthetic_loss_case plus a seeded focal; each case draws its random numbers from
`torch.manual_seed(draw_seed)` on the CPU.  The reference's `torch.randint` / `torch.multinomial` results and its alignment's
scale and shift are recorded by wrapping those calls.  The file stores each case's recipe, SHA-256 digests of its inputs and of
the two offset tensors (they are regenerated from the seed, being 1 KiB per pixel), the multinomial's selection, the kept
patches, the alignment's scale and shift, the loss and misc, and, for the reference's cases of at most 61×83 pixels, the
gradient of loss.sum() with respect to pred_points.  The other gradients are left out to keep the file small: the port
reproduces them bitwise here, so the GPU test checks those against the port running on the engine's alignment.

Every case is also run through oracle/local_loss_port.py given the recorded draws and the reference's solver, and the two must agree
bitwise.  The reference raises for a batch of more than one image (its (B,) focal and global_scale broadcast against the map's
width and the patch axis), so the batch cases are the port's, run with the reference's solver on draws it makes itself from the
same seed.
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle", "utils3d_shim"))
if not os.environ.get("MOGE_REFERENCE"):
    sys.exit("set MOGE_REFERENCE to a checkout of the reference (microsoft/MoGe)")
sys.path.insert(1, os.environ["MOGE_REFERENCE"])

import torch  # noqa: E402

from moge_b200.synthetic import array_digest, synthetic_loss_case  # noqa: E402
from oracle.utils3d_metrics import install  # noqa: E402

install()
from oracle import local_loss_port  # noqa: E402
from moge.train import losses as ref  # noqa: E402  (the real reference)
from moge.utils import alignment as ref_alignment  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "local_loss.pt")
V2 = {4: {"level": 4, "num_patches": 16, "align_resolution": 24}, 16: {"level": 16, "num_patches": 256, "align_resolution": 12},
      64: {"level": 64, "num_patches": 4096, "align_resolution": 6}}

# (name, level, batch shape, H, W, image 0 without valid GT, global scale ("none", "fit": the patches' median scale, "reject":
# a tenth of it, so that some patches fall outside (0.1, 10) times it), extra keyword arguments)
CASES = [
    ("local4_48x64", 4, (), 48, 64, False, "none", {}),
    ("local16_48x64_reject", 16, (), 48, 64, False, "reject", {}),
    ("local4_61x83_beta_sparsity_trunc", 4, (), 61, 83, False, "fit", {"beta": 0.01, "sparsity_aware": True, "trunc": 0.05}),
    ("local16_b2_61x83_empty_image", 16, (2,), 61, 83, True, "fit", {}),
    ("local4_b2_48x64", 4, (2,), 48, 64, False, "none", {"sparsity_aware": True}),
    ("local64_144x224", 64, (), 144, 224, False, "none", {}),
    ("local64_48x64_no_patch", 64, (), 48, 64, False, "none", {}),
]


def case_inputs(seed, batch_shape, H, W, empty):
    inputs = synthetic_loss_case(seed, batch_shape, H, W, empty_image=empty)
    g = torch.Generator().manual_seed(6000 + seed)
    # a focal below the scene's (0.55 to 0.95 of the width), so that a patch's 3D radius reaches its box's corners
    focal = 0.15 + 0.15 * torch.rand(batch_shape, generator=g)
    return inputs["pred_points"], inputs["gt_points"], focal


def input_digest(pred, gt, focal) -> str:
    return array_digest(pred.numpy(), gt.numpy(), focal.numpy())


RECORD = {}
_randint, _multinomial, _ref_align = torch.randint, torch.multinomial, ref.align_points_scale_xyz_shift


def _recording_randint(*args, **kwargs):
    out = _randint(*args, **kwargs)
    RECORD.setdefault("randint", []).append(out.clone())
    return out


def _recording_multinomial(*args, **kwargs):
    out = _multinomial(*args, **kwargs)
    RECORD["multinomial"] = out.clone()
    return out


def _recording_align(*args, **kwargs):
    scale, shift = _ref_align(*args, **kwargs)
    RECORD["scale"], RECORD["shift"] = scale.detach().clone(), shift.detach().clone()
    return scale, shift


def ref_solver(p, g, w, trunc):
    return ref_alignment.align_points_scale_xyz_shift(p, g, w, trunc=trunc)


def run_reference(pred, gt, focal, global_scale, kwargs, draw_seed):
    RECORD.clear()
    torch.randint, torch.multinomial, ref.align_points_scale_xyz_shift = _recording_randint, _recording_multinomial, _recording_align
    try:
        torch.manual_seed(draw_seed)
        p = pred.clone().requires_grad_(True)
        loss, misc = ref.affine_invariant_local_loss(p, gt, focal, global_scale, **kwargs)
    finally:
        torch.randint, torch.multinomial, ref.align_points_scale_xyz_shift = _randint, _multinomial, _ref_align
    grad = None
    if loss.requires_grad:
        loss.sum().backward()
        grad = p.grad.clone()
    draws = {"delta_i": RECORD["randint"][0], "delta_j": RECORD["randint"][1], "selection": RECORD["multinomial"]}
    return loss.detach(), misc, grad, draws, RECORD.get("scale"), RECORD.get("shift")


def run_port(pred, gt, focal, global_scale, kwargs, draws=None, draw_seed=None):
    record = {}
    if draw_seed is not None:
        torch.manual_seed(draw_seed)
    p = pred.clone().requires_grad_(True)
    loss, misc = local_loss_port.affine_invariant_local_loss(p, gt, focal, global_scale, align=ref_solver, draws=draws, record=record,
                                                         **kwargs)
    grad = None
    if loss.requires_grad:
        loss.sum().backward()
        grad = p.grad.clone()
    return loss.detach(), misc, grad, record


def global_scale_for(mode, pred, gt, focal, kwargs, draw_seed, batch_shape):
    if mode == "none":
        return None
    _, _, _, record = run_port(pred, gt, focal, None, kwargs, draw_seed=draw_seed)
    med = record["scale"].median()
    return torch.full(batch_shape, float(med) * (1.0 if mode == "fit" else 0.1))


def main():
    torch.use_deterministic_algorithms(True)     # the CPU index_put backward over overlapping patches accumulates in a fixed order
    gold = []
    for seed, (name, level, batch_shape, H, W, empty, gs_mode, extra) in enumerate(CASES):
        pred, gt, focal = case_inputs(seed, batch_shape, H, W, empty)
        kwargs = {**V2[level], **extra}
        draw_seed = 7000 + seed
        global_scale = global_scale_for(gs_mode, pred, gt, focal, kwargs, draw_seed, batch_shape)
        if batch_shape == ():
            loss, misc, grad, draws, scale, shift = run_reference(pred, gt, focal, global_scale, kwargs, draw_seed)
            p_loss, p_misc, p_grad, record = run_port(pred, gt, focal, global_scale, kwargs, draws=draws)
            assert torch.equal(loss, p_loss) and misc == p_misc, (name, loss, p_loss, misc, p_misc)
            assert (grad is None) == (p_grad is None) and (grad is None or torch.equal(grad, p_grad)), name
            assert (scale is None) == (record.get("scale") is None), name
            assert scale is None or (torch.equal(scale, record["scale"]) and torch.equal(shift, record["shift"])), name
            kept = record["kept"]
        else:
            try:
                run_reference(pred, gt, focal, global_scale, kwargs, draw_seed)
                raise AssertionError(f"{name}: the reference was expected to raise for a batch")
            except RuntimeError as e:
                print(f"{name}: the reference raises for a batch ({str(e).splitlines()[0]})")
            loss, misc, grad, record = run_port(pred, gt, focal, global_scale, kwargs, draw_seed=draw_seed)
            draws = {k: record[k] for k in ("delta_i", "delta_j", "selection")}
            scale, shift, kept = record.get("scale"), record.get("shift"), record["kept"]
        # the offsets regenerate from the seed
        torch.manual_seed(draw_seed)
        r = draws["delta_i"].abs().max().item()
        assert torch.equal(torch.randint(-r, r + 1, draws["delta_i"].shape), draws["delta_i"])
        assert torch.equal(torch.randint(-r, r + 1, draws["delta_j"].shape), draws["delta_j"])
        gold.append({"name": name, "seed": seed, "batch_shape": batch_shape, "H": H, "W": W, "empty_image": empty, "kwargs": kwargs,
                     "global_scale": global_scale, "draw_seed": draw_seed, "reference": batch_shape == (),
                     "inputs_sha256": input_digest(pred, gt, focal),
                     "draws_sha256": array_digest(draws["delta_i"].numpy(), draws["delta_j"].numpy()),
                     "selection": draws["selection"], "kept": kept, "scale": scale, "shift": shift,
                     "loss": loss, "misc": misc, "grad": grad if batch_shape == () and H * W <= 61 * 83 else None})
        print(f"{name:36s} kept {kept.numel():5d}  loss {loss.tolist()}  misc {misc}")
    torch.save(gold, OUT)
    print("wrote", OUT, os.path.getsize(OUT), "bytes")


if __name__ == "__main__":
    main()

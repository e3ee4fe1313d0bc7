"""Reading the reference goldens under tests/golden (oracle/make_golden.py): `<name>.pt` holds meta and the forward() outputs,
the infer() outputs are in the same file or, where the two together would pass 1 MB, in `<name>.infer.pt`."""
import os

import torch


def load_golden(golden_dir, name):
    gold = torch.load(os.path.join(golden_dir, name + ".pt"), weights_only=False)
    if "infer" not in gold:
        gold["infer"] = torch.load(os.path.join(golden_dir, name + ".infer.pt"), weights_only=False)
    return gold

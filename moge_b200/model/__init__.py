"""Mirror of /root/reference/moge/model/__init__.py:9-18."""
import importlib


def import_model_class_by_version(version: str):
    assert version in ["v1", "v2"], f'Unsupported model version: {version}'
    if version == "v1":
        raise NotImplementedError("import_model_class_by_version('v1') is not wired yet: use moge.model.v1.MoGeModel "
                                  "(moge_b200.model.v1.MoGeModel) for MoGe-1")
    module = importlib.import_module(".v2", __package__)
    return getattr(module, "MoGeModel")

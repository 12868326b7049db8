"""`{"TypeName": {kwargs}}` factories (reference: common/factories/base_factory.py:37-72,
detection_modules_factory.py:15-28, activations_type_factory.py)."""
from collections.abc import Mapping
from typing import Any, Dict, Union

from torch import nn

from .registry import ALL_DETECTION_MODULES, LOSSES, METRICS


class UnknownTypeException(Exception):
    def __init__(self, unknown_type, choices):
        super().__init__(f"Unknown object type: {unknown_type} in configuration. valid types are: {sorted(choices)}")


def _fuzzy(name) -> str:
    """Registry names are matched without sensitivity to case, underscores and punctuation when there is no exact hit
    (training/utils/utils.py:255-261): the shipped recipes write `yolo_nas_pose_loss` for the class registered as `YoloNASPoseLoss`."""
    import re

    return re.sub(r"[^\w|\/]", "", str(name)).replace("_", "").lower()


class BaseFactory:
    def __init__(self, type_dict: Dict[str, type]):
        self.type_dict = type_dict

    def _resolve(self, name):
        if name in self.type_dict:
            return self.type_dict[name]
        loose = {_fuzzy(k): v for k, v in self.type_dict.items()}
        if _fuzzy(name) in loose:
            return loose[_fuzzy(name)]
        raise UnknownTypeException(name, self.type_dict.keys())

    def get(self, conf: Union[str, dict]):
        if isinstance(conf, str):
            return self._resolve(conf)()
        if isinstance(conf, Mapping):
            if len(conf) != 1:
                raise RuntimeError(f"Malformed object definition: expected a type name or a single-entry dict {{type_name: {{params}}}}, received: {conf}")
            (_type, _params), = conf.items()
            return self._resolve(_type)(**_params)
        return conf


class DetectionModulesFactory(BaseFactory):
    def __init__(self):
        super().__init__(ALL_DETECTION_MODULES)

    @staticmethod
    def insert_module_param(conf, name: str, value: Any):
        if isinstance(conf, str):
            return {conf: {name: value}}
        cls_type = list(conf.keys())[0]
        conf[cls_type][name] = value
        return conf


class LossesFactory(BaseFactory):
    def __init__(self):
        super().__init__(LOSSES)


class MetricsFactory(BaseFactory):
    """`valid_metrics_list` entries (reference: common/factories/metrics_factory.py): a name, `{name: {kwargs}}` or an object."""

    def __init__(self):
        super().__init__(METRICS)


ACTIVATIONS = {"relu": nn.ReLU, "silu": nn.SiLU, "swish": nn.SiLU, "identity": nn.Identity, None: None}


def resolve_activation(act):
    """String (recipes) or nn.Module type -> nn.Module type, as ActivationsTypeFactory does."""
    if act is None or isinstance(act, type):
        return act
    if isinstance(act, str):
        if act.lower() not in ACTIVATIONS:
            raise UnknownTypeException(act, [k for k in ACTIVATIONS if k])
        return ACTIVATIONS[act.lower()]
    raise TypeError(f"unsupported activation spec {act!r}")


def activation_code(act_type) -> str:
    """nn.Module activation type -> epilogue code of the kernels.  Only the activations on the YOLO-NAS / ResNet /
    PP-YOLOE paths are implemented (SURVEY.md D1); anything else fails loudly instead of silently falling back."""
    if act_type is None or act_type is nn.Identity:
        return "none"
    if act_type is nn.ReLU:
        return "relu"
    if act_type is nn.SiLU:
        return "silu"
    raise NotImplementedError(f"activation {act_type} has no sm_90a epilogue in super_gradients_b200")

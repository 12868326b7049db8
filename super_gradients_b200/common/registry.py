"""Name -> class registries: the plug-in boundary of the reference (common/registry/registry.py:14-88).
Same decorator contract: re-registering a DIFFERENT class under an existing name raises."""
import inspect
from typing import Callable, Dict, Optional


def create_register_decorator(registry: Dict[str, Callable]) -> Callable:
    def register(name: Optional[str] = None, deprecated_name: Optional[str] = None) -> Callable:
        def decorator(cls: Callable) -> Callable:
            for key in filter(None, (name or cls.__name__, deprecated_name)):
                if key in registry and registry[key] is not cls:
                    prev = registry[key]
                    raise Exception(f"`{key}` is already registered and points to `{inspect.getmodule(prev).__name__}.{prev.__name__}`")
                registry[key] = cls
            return cls

        return decorator

    return register


ARCHITECTURES: Dict[str, Callable] = {}
register_model = create_register_decorator(ARCHITECTURES)
ALL_DETECTION_MODULES: Dict[str, Callable] = {}
register_detection_module = create_register_decorator(ALL_DETECTION_MODULES)
LOSSES: Dict[str, Callable] = {}
register_loss = create_register_decorator(LOSSES)
CALLBACKS: Dict[str, Callable] = {}
register_callback = create_register_decorator(CALLBACKS)
METRICS: Dict[str, Callable] = {}
register_metric = create_register_decorator(METRICS)
TRANSFORMS: Dict[str, Callable] = {}
register_transform = create_register_decorator(TRANSFORMS)
COLLATE_FUNCTIONS: Dict[str, Callable] = {}
register_collate_function = create_register_decorator(COLLATE_FUNCTIONS)

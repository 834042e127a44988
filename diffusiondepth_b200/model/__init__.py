"""Mirror of the reference's `src/model` plugin surface (reference src/model/__init__.py:17-23):
`get(args)` -> model class, looked up as `<args.model_name>Model` in module `<that name, lower-cased>`."""
from importlib import import_module


def get(args):
    model_name = args.model_name + 'Model'
    try:
        module = import_module(f"{__name__}.{model_name.lower()}")
    except ModuleNotFoundError as e:
        raise ModuleNotFoundError(
            f"{model_name}: only the DiffusionDepth model (Diffusion_DCbase_) is served by the H100 engine; "
            "NLSPN and the DCN extension are out of scope (DESIGN.md)") from e
    return getattr(module, model_name)


# importing the package registers the codec and head classes (HEADS / DEPTH_TRANSFORM lookups need them)
from .ops import depth_transform as _codec  # noqa: E402,F401
from . import head as _head  # noqa: E402,F401

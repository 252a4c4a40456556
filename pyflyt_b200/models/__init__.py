"""Vehicle descriptions (host side): link tables + coefficient tables → ``PfbModel``."""
from .tables import MAX_QUADX_MODELS, ModelSetError, PfbEnvConfig, PfbModel, PfbShape, build_mixed_model_set, build_model, build_model_set, load_vehicle  # noqa: F401

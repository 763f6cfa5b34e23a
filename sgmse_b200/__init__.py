"""sgmse_b200 — H100-native (sm_90a) reverse-SDE enhancement engine behind sp-uhh/sgmse's
``ScoreModel.enhance()`` / ``get_pc_sampler()``.  See DESIGN.md and include/sgmse_b200.h."""
from .engine import Engine, EngineConfig, rk45_host, rk45_host_groups  # noqa: F401
from .api import install, uninstall, refresh, engine_from_score_model, config_from_score_model  # noqa: F401
from .service import BatchedEnhancer, plan_batches  # noqa: F401
from .files import DirectoryEnhancer, list_audio_files  # noqa: F401

__all__ = ["Engine", "EngineConfig", "install", "uninstall", "refresh", "engine_from_score_model", "config_from_score_model",
           "BatchedEnhancer", "plan_batches", "DirectoryEnhancer", "list_audio_files", "rk45_host", "rk45_host_groups"]

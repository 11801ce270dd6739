"""Built-in game configurations (reference: python/magent/builtin/config/) and scripted opponents (rule_model)."""
from . import config
from . import rule_model

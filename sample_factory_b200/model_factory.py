"""The registry for custom model parts (the reference's model/model_factory.py:16-60, algo/utils/context.py).

The device engine runs the reference's BUILT-IN model families as hand-written sm_90a kernels (ModelSpec.from_cfg);
an arbitrary torch module cannot be lowered onto them and there is no eager-PyTorch fallback on this path.  The registry
therefore keeps the reference's API -- registration succeeds, so import-time `register_*` calls in user scripts work --
and the runner refuses to start with an explicit message if a custom factory is installed (`check_supported`)."""
from typing import Callable, Optional


class UnsupportedCustomModel(NotImplementedError):
    pass


class ModelFactory:
    def __init__(self):
        self.make_actor_critic_func: Optional[Callable] = None
        self.make_model_encoder_func: Optional[Callable] = None
        self.make_model_core_func: Optional[Callable] = None
        self.make_model_decoder_func: Optional[Callable] = None

    def register_actor_critic_factory(self, make_actor_critic_func: Callable):
        self.make_actor_critic_func = make_actor_critic_func

    def register_encoder_factory(self, make_model_encoder_func: Callable):
        self.make_model_encoder_func = make_model_encoder_func

    def register_model_core_factory(self, make_model_core_func: Callable):
        self.make_model_core_func = make_model_core_func

    def register_decoder_factory(self, make_model_decoder_func: Callable):
        self.make_model_decoder_func = make_model_decoder_func

    def custom_parts(self):
        parts = dict(actor_critic=self.make_actor_critic_func, encoder=self.make_model_encoder_func,
                     core=self.make_model_core_func, decoder=self.make_model_decoder_func)
        return {k: v for k, v in parts.items() if v is not None}

    def check_supported(self) -> None:
        custom = self.custom_parts()
        if custom:
            names = ", ".join(f"{k} ({getattr(v, '__name__', v)})" for k, v in custom.items())
            raise UnsupportedCustomModel(
                f"custom model parts are registered: {names}.  sample_factory_b200 runs the built-in model families "
                "(encoder_mlp_layers / encoder_conv_architecture / rnn_type / decoder_mlp_layers) as hand-written CUDA "
                "kernels and has no eager-PyTorch path for arbitrary torch modules; express the model through those flags "
                "or run this experiment on the reference implementation.")


_GLOBAL_MODEL_FACTORY = ModelFactory()


def global_model_factory() -> ModelFactory:
    return _GLOBAL_MODEL_FACTORY


def reset_global_model_factory() -> ModelFactory:
    global _GLOBAL_MODEL_FACTORY
    _GLOBAL_MODEL_FACTORY = ModelFactory()
    return _GLOBAL_MODEL_FACTORY

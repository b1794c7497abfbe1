"""CPU checks of the activation-checkpointing switch: HF's gradient_checkpointing_enable() / _disable() reach the training
engine's `checkpoint` flag on every training call, on the module and through get_peft_model's wrapper, with no rebuild
(the engine and the autograd bridge are stubbed: the CUDA side is tests/test_checkpointing_gpu.py)."""
import torch

from test_lora_gpu import _tiny_model, reference_linear_names


class _Engine:
    checkpoint = False


def _wire(monkeypatch, model):
    from u2tokenizer_b200 import modeling
    eng = _Engine()
    seen = []
    model.__dict__["train_engine"] = lambda **kw: eng

    def apply(te, batch, names, *params):
        seen.append(te.checkpoint)
        return torch.zeros((), requires_grad=True)
    monkeypatch.setattr(modeling._U2TrainLoss, "apply", apply)
    return eng, seen


def _step(model):
    ids = torch.randint(1, 500, (2, 12))
    model(input_ids=ids, labels=ids.clone(), images=None)


def test_enable_disable_reach_the_engine(monkeypatch):
    model = _tiny_model()
    model.train()
    eng, seen = _wire(monkeypatch, model)
    _step(model)
    model.gradient_checkpointing_enable()
    _step(model)
    model.gradient_checkpointing_disable()
    _step(model)
    model.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    _step(model)
    assert seen == [False, True, False, True]
    assert eng.checkpoint


def test_enable_through_peft_wrapper(monkeypatch):
    from u2tokenizer_b200.lora import LoraConfig, get_peft_model
    model = _tiny_model()
    peft = get_peft_model(model, LoraConfig(r=16, lora_alpha=32, target_modules=reference_linear_names(model),
                                            lora_dropout=0.05))
    peft.train()
    eng, seen = _wire(monkeypatch, model)
    _step(peft)
    peft.gradient_checkpointing_enable(gradient_checkpointing_kwargs={"use_reentrant": False})
    peft.enable_input_require_grads()   # HF Trainer's call for PEFT with checkpointing: harmless here
    _step(peft)
    peft.gradient_checkpointing_disable()
    _step(peft)
    assert seen == [False, True, False]

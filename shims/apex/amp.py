"""apex.amp stand-in for the reference's --fp16 path (train_generator.py:161-169,317-321,355-359).

The kernels already compute in a 16-bit storage type with fp32 accumulation, so there is nothing to cast.  What apex O1 adds is
dynamic loss scaling, and that depends on the storage type (hrviton_b200.ops.set_precision, or HRV_PRECISION for the scripts):
  * fp16 storage: initialize(..., num_losses=n) creates n hrviton_b200.loss_scale.DynamicLossScaler (apex's defaults: S = 2^16,
    x2 after 2000 clean steps, x0.5 on overflow).  scale_loss(loss, optimizer, loss_id) yields loss * S; on exit it divides the
    optimiser's gradients by S (one kernel, which also flags inf / NaN), updates scaler loss_id, and makes that optimiser's next
    step() a no-op when a gradient was not finite.  That decision syncs once per step, as apex does: the reference's plain
    torch.optim.Adam cannot take a device-side skip flag.
  * bf16 storage (the default; 8 exponent bits, no underflow to fix) and fp32: initialize returns its arguments, scale_loss yields
    the loss unchanged.
amp.state_dict / load_state_dict are not provided: the reference never calls them."""
import contextlib

_SCALERS = []


def _fp16_storage():
    import hrviton_b200.ops as ops  # bound by the drop-in networks / network_generator modules before the scripts run
    return ops.get_precision() == "fp16"


def _wrap_step(optimizer):
    """optimizer.step() skips the update (once) after scale_loss found a non-finite gradient."""
    if getattr(optimizer, "_amp_skip_next", None) is not None:
        return
    optimizer._amp_skip_next = False
    step = optimizer.step

    def guarded_step(*args, **kwargs):
        if optimizer._amp_skip_next:
            optimizer._amp_skip_next = False
            return None
        return step(*args, **kwargs)

    optimizer.step = guarded_step


def initialize(models, optimizers=None, opt_level="O1", num_losses=1, **kwargs):
    if _fp16_storage():
        from hrviton_b200.loss_scale import DynamicLossScaler
        opts = [] if optimizers is None else (optimizers if isinstance(optimizers, (list, tuple)) else [optimizers])
        device = opts[0].param_groups[0]["params"][0].device if opts else "cuda"
        _SCALERS[:] = [DynamicLossScaler(device) for _ in range(num_losses)]
        for o in opts:
            _wrap_step(o)
    return (models, optimizers) if optimizers is not None else models


@contextlib.contextmanager
def scale_loss(loss, optimizer, loss_id=0, **kwargs):
    if not _SCALERS or not _fp16_storage():
        yield loss
        return
    scaler = _SCALERS[loss_id]
    yield scaler.scale_loss(loss)
    scaler.unscale_and_check(optimizer)
    optimizer._amp_skip_next = bool(scaler.found_inf)
    scaler.update()

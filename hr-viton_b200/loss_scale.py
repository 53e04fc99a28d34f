"""Dynamic loss scaling for fp16-storage training: the policy of apex O1 (train_generator.py:161-169,317-321,355-359), with every
decision on the device so that a whole training step, scaler included, can be captured into one CUDA graph.

fp16's smallest subnormal is 2^-24: the per-element seeds of the loss gradients (VGGLoss writes 10 * w_i / numel into every element
of its slice, DESIGN.md §4) fall below it at the training resolutions, so without a scale the generator receives no gradient from
the shallow VGG slices.  The loss is multiplied by S before backward(); the fp32 parameter gradients are divided by S again
(hrv_grad_unscale_check, which also flags inf / NaN); a step with a non-finite gradient is skipped and halves S; 2000 clean steps
in a row double S.  In bf16 storage (8 exponent bits, the range of fp32) scaling is allowed but has nothing to fix."""
import torch

from . import ops


class DynamicLossScaler:
    """Device state: `scale` (fp32), `growth_tracker` (int32, clean steps since the last change) and `found_inf` (fp32, 1.0 when the
    last unscale_and_check saw a non-finite gradient).  Use per step, for one loss and the optimiser of its parameters:

        scaler.scale_loss(loss).backward();  scaler.unscale_and_check(opt);  opt.step();  scaler.update()

    For the package's fused Adam set `opt.found_inf = scaler.found_inf` once: torch's fused Adam then leaves parameters, moments and
    step count untouched on a flagged step, without a host synchronisation."""

    def __init__(self, device="cuda", init_scale=2.0 ** 16, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000):
        self.scale = torch.full((), float(init_scale), dtype=torch.float32, device=device)
        self.growth_tracker = torch.zeros((), dtype=torch.int32, device=device)
        self.found_inf = torch.zeros((), dtype=torch.float32, device=device)
        self._inv_scale = torch.empty((), dtype=torch.float32, device=device)
        self.growth_factor, self.backoff_factor, self.growth_interval = float(growth_factor), float(backoff_factor), int(growth_interval)
        self._tables = {}  # id(optimizer) -> device segment table of its gradients (ops.grad_unscale_check)

    def scale_loss(self, loss):
        return loss * self.scale

    @staticmethod
    def gradients(optimizer, reducer=None):
        """The fp32 tensors that hold the gradients of `optimizer`'s parameters: the flat buckets of a ddp.GradBucketReducer once it has
        built them (every bucketed p.grad is a view into one), plus the .grad of any parameter outside the buckets."""
        buckets = reducer._buckets if reducer is not None and reducer._buckets is not None else []
        out = [b["flat"] for b in buckets]
        covered = {id(p) for b in buckets for p in b["params"]}
        for group in optimizer.param_groups:
            out += [p.grad for p in group["params"] if p.grad is not None and id(p) not in covered]
        return out

    def unscale_and_check(self, optimizer, reducer=None):
        """g /= S for every gradient of `optimizer`, in place; found_inf = 1 if any was inf / NaN.  Under data parallelism call it after
        the bucket all-reduces have been joined: a non-finite value on any rank reaches every rank through the sum, so all ranks skip
        the same steps without another collective."""
        self.found_inf.zero_()
        torch.reciprocal(self.scale, out=self._inv_scale)
        key = id(optimizer)
        self._tables[key] = ops.grad_unscale_check(self.gradients(optimizer, reducer), self._inv_scale, self.found_inf, self._tables.get(key))

    def update(self):
        """Backoff on a flagged step, growth after growth_interval clean ones (torch._amp_update_scale_: on the device, capturable)."""
        torch._amp_update_scale_(self.scale, self.growth_tracker, self.found_inf, self.growth_factor, self.backoff_factor, self.growth_interval)

    def state_dict(self):
        return {"scale": float(self.scale), "growth_tracker": int(self.growth_tracker), "growth_factor": self.growth_factor,
                "backoff_factor": self.backoff_factor, "growth_interval": self.growth_interval}

    def load_state_dict(self, sd):
        """In place, so that a captured graph keeps reading the same tensors."""
        self.scale.fill_(float(sd["scale"]))
        self.growth_tracker.fill_(int(sd["growth_tracker"]))
        self.growth_factor, self.backoff_factor, self.growth_interval = float(sd["growth_factor"]), float(sd["backoff_factor"]), int(sd["growth_interval"])


def make_scalers(loss_scale, names, device):
    """{} for loss_scale None, one DynamicLossScaler per name for "dynamic" (one per loss, as apex's num_losses)."""
    if loss_scale is None:
        return {}
    if loss_scale != "dynamic":
        raise ValueError("loss_scale must be None or 'dynamic', got %r" % (loss_scale,))
    ops.require_trainable_storage("loss_scale='dynamic'")
    return {n: DynamicLossScaler(device) for n in names}

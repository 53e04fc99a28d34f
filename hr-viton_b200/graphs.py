"""CUDA-graph capture shared by the training steps (train_step._GraphMixin) and the inference runners (pipeline.TryOnGraph,
pipeline.GeneratorGraph): eager warm-up on a side stream, capture, replay, release."""
import gc

import torch

from . import ops


class CapturedCall:
    """fn() captured into one CUDA graph; `out` is what the captured call returned (tensors that every replay rewrites).

    warm: eager calls of fn() on a side stream before the capture, so that lazy initialisation (packed-weight caches, workspaces,
    optimiser state) happens outside it.  keep_rng=True puts torch's CUDA generator back where it was before the warm-up, so the
    first replay draws what one eager call from that state would have drawn.  The graph keeps the ops workspaces it was captured
    with alive: ops._workspace replaces a workspace that is too small for a later call, and the replayed kernels keep writing to
    the one they were captured with."""

    def __init__(self, fn, warm=2, capture_error_mode="global", keep_rng=False):
        rng = torch.cuda.get_rng_state() if keep_rng else None
        try:
            cur = torch.cuda.current_stream()
            side = torch.cuda.Stream()
            side.wait_stream(cur)
            with torch.cuda.stream(side):
                for _ in range(warm):
                    fn()
            cur.wait_stream(side)
            torch.cuda.synchronize()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, capture_error_mode=capture_error_mode):
                self.out = fn()
            self.workspaces = list(ops._ws.values())
        finally:
            if rng is not None:
                torch.cuda.set_rng_state(rng)

    def replay(self):
        self.graph.replay()
        return self.out

    def release(self):
        """Destroy the graph and drop its outputs (graph nodes can hold references on an NCCL communicator: ncclCommDestroy at
        process-group tear-down waits for them — two-GPU training runs printed their result and then hung in
        destroy_process_group)."""
        torch.cuda.synchronize()
        self.graph = None
        self.out = None
        self.workspaces = None
        gc.collect()
        torch.cuda.synchronize()

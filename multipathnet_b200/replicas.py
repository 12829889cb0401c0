"""Several replicas of one model on ONE GPU.

The reference's inference runner keeps one model replica per donkey thread, each pinned to a GPU (test_runner.lua:55-66), and
deals the images round-robin (:91-104). Nothing ties the number of threads to the number of GPUs: with K threads per GPU —
here K `mpn_ctx` contexts, each on a stream of its own (`mpn_ctx_create_stream`), each with its own `mpn_model` (weights
duplicated: 0.55 GB for VGG-16 Fast R-CNN on an 80 GB part) — the kernels of one replica fill the layer-boundary and
NMS-chain bubbles of the others (measured on one H100 80GB HBM3 capped at 400 W, BASELINE configs[1], 200 steps, each count run twice: 2.50-2.60e5
proposals/s with one replica, 2.57-2.58e5 with two, 2.64-2.65e5 with three — a few percent, the card ran at its power cap).
Per-image latency does not improve (it grows with K); this is a throughput arrangement.

`ModelReplicas` owns the K (ctx, model) pairs and deals work round-robin; results are those of a single model, bit for bit
(every replica runs the same deterministic kernels). `join()` makes replica 0's stream wait for the others — the point at
which the end-of-run gather of the detection records (SURVEY 8e) is issued on replica 0's context.
"""
from __future__ import annotations

from typing import List, Optional

from ._lib import Context, Model


class ModelReplicas:
    def __init__(self, device: int, spec, n_replicas: int = 2, max_rois: int = 2048, max_h: int = 1024, max_w: int = 1344,
                 first_ctx: Optional[Context] = None):
        """first_ctx: use this context (e.g. one bound to the caller's stream) for replica 0; the others get streams of their own"""
        if n_replicas < 1:
            raise ValueError("n_replicas must be >= 1")
        self.ctxs: List[Context] = []
        self.models: List[Model] = []
        self._owned: List[Context] = []
        for k in range(n_replicas):
            if k == 0 and first_ctx is not None:
                ctx = first_ctx
            else:
                ctx = Context(device, own_stream=True)
                self._owned.append(ctx)
            self.ctxs.append(ctx)
            self.models.append(Model(ctx, spec, max_rois=max_rois, max_h=max_h, max_w=max_w))

    def __len__(self):
        return len(self.models)

    def model(self, i: int) -> Model:
        """the replica image i goes to (round-robin, test_runner.lua:91-104)"""
        return self.models[i % len(self.models)]

    def join(self):
        """replica 0's stream waits for everything the other replicas have enqueued"""
        for c in self.ctxs[1:]:
            self.ctxs[0].wait_ctx(c)

    def synchronize(self):
        for c in self.ctxs:
            c.synchronize()

    @property
    def launch_count(self) -> int:
        return sum(c.launch_count for c in self.ctxs)

    def close(self):
        for m in self.models:
            m.close()
        self.models = []
        for c in self._owned:
            c.close()
        self._owned = []
        self.ctxs = []

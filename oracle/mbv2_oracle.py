"""StepOracle for graphs with Dropout ops (MobileNet-v2's head, slim.dropout).

TEST INFRASTRUCTURE ONLY.  The device draws its dropout masks from its own Philox stream; a test reads that mask
back and hands it in here (`masks`: op name -> 0/1 array of the op's shape), and the oracle applies TF 1.x's op chain
y = (x / keep_prob) * mask in fp32, whose autograd backward is dx = (dy * mask) / keep_prob.  A Dropout op in
inference mode (or an inference-mode pass) is the identity.  Every other op is StepOracle's: the graph is cut at each
Dropout and the pieces run through StepOracle.forward unchanged.
"""
import copy

import numpy as np
import torch

from .step_oracle import StepOracle


class DropoutStepOracle(StepOracle):
    def __init__(self, *args, masks=None, **kw):
        super().__init__(*args, **kw)
        self.masks = dict(masks or {})

    def forward(self, params, images, training=True, stats_out=None, force=None, local_out=None):
        val = {}
        cur_in, cur_val, seg = self.images_t, images, []
        for op in self.ops + [None]:
            if op is not None and op.type != 'Dropout':
                seg.append(op)
                continue
            part = copy.copy(self)
            part.ops, part.images_t = seg, cur_in
            val.update(StepOracle.forward(part, params, cur_val, training, stats_out, force, local_out))
            if op is None:
                break
            x = val[op.inputs[0].name]
            if op.attrs['training'] and training:
                keep = torch.tensor(op.attrs['keep_prob'], dtype=torch.float32)
                m = torch.from_numpy(np.asarray(self.masks[op.name], np.float32).reshape(x.shape))
                y = (x / keep) * m
            else:
                y = x
            if local_out is not None:
                local_out[op.output.name] = y
            if force is not None and op.output.name in force:
                y = force[op.output.name]
            val[op.output.name] = y
            cur_in, cur_val, seg = op.output, y, []
        return val

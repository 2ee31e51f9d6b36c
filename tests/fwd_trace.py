"""Diagnostic (not a collected test; lives under tests/ because only tests may use the oracle): per-op forward
differences between the CUDA step and the CPU oracle for a bench.py workload at a small batch.
usage: python tests/fwd_trace.py <workload> <batch> [a_bits]   (PF_TC_LEVELS / PF_TC_FEED / PF_CONV_PATH select the path)"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from support import gpu_activation, oracles  # noqa: E402

F32 = np.float32


def main():
    workload, batch = sys.argv[1], int(sys.argv[2])
    lrn = bench.build_learner(workload, 1, batch)
    if len(sys.argv) > 3:
        from pocketflow_b200.flags import FLAGS
        import importlib
        FLAGS.uql_activation_bits = int(sys.argv[3])
        from pocketflow_b200.learners.learner_utils import create_learner
        mod = importlib.import_module(lrn.model_helper.__module__) if hasattr(lrn, 'model_helper') else None
        from pocketflow_b200.nets import resnet_at_ilsvrc12 as R
        lrn = create_learner(None, (mod or R).ModelHelper())
    ex = lrn.sess_train
    orc = oracles(lrn)
    state = ex.store.state_dict()
    tstate = ex.teacher.store.state_dict() if ex.teacher is not None else None
    images, labels = lrn.iterator_train.next_batch()
    ex.buf[lrn.images].copy_(images)
    ex.buf[lrn.labels].copy_(labels)
    ex.run_step(lrn.lrn_rate(0))
    got = ex.fetch_losses()
    kind = 'adam' if ex.S2 is not None else 'momentum'
    ref, _, _ = orc.step(state, images.numpy(), labels.numpy(), dict(kind=kind, slots={}, momentum=0.9), lrn.lrn_rate(0),
                         teacher_state=tstate)
    print('levels: act %d  weights %d | loss gpu %.7f ref %.7f | ce %.7f / %.7f' % (
        len(ex.act_lv), len(ex.w_lv), got['loss'], ref['loss'], got['ce'], ref['ce']))
    params = {k: torch.from_numpy(np.array(v, dtype=F32, copy=True)) for k, v in state.items()}
    with torch.no_grad():
        val = orc.forward(params, images, True)
    shown = 0
    for op in ex.ops:
        if op.type in ('Placeholder', 'Reshape', 'Identity') or op in ex.fused_act:
            continue
        try:
            if op.type in ('Relu', 'Relu6'):
                a = gpu_activation(ex, op)
            elif op.type == 'FusedBatchNorm':
                pl = ex.xplanes.get(op)
                if pl is not None and not ex.bn_need_f32.get(op, True):
                    continue
                a = ex.T(op.output).cpu().numpy()
            else:
                a = ex.T(op.output).cpu().numpy()
        except Exception as e:  # noqa: BLE001
            print('  %-60s unavailable (%s)' % (op.name[-60:], e))
            continue
        b = val[op.output.name].numpy()
        err = float(np.abs(a - b).max() / (np.abs(b).max() + 1e-12))
        mark = ' <<<' if err > 1e-4 else ''
        if err > 1e-4 and op.type == 'Conv2D' and op in ex.tc and op not in ex.fused_add and not getattr(main, 'diag', False):
            main.diag = True
            from pocketflow_b200 import ops
            d, tw = ex.desc[op], ex.tc[op]
            xin_ref = val[op.inputs[0].name]
            wq_gpu = ex.kernel_of(op).cpu().numpy()
            print('    --- first diverging tensor-core conv: %s ksize %s strides %s pad %s' % (
                op.name, op.attrs['ksize'], op.attrs['strides'], op.attrs['pad']))
            # (1) the weights the engine hands to the preparation vs the oracle's quantized weights
            import torch.nn.functional as F_
            from oracle.step_oracle import weight_fake_quant
            w_or = params[op.vars['kernel'].name]
            if op.name in orc.wq_bits:
                w_or = weight_fake_quant(w_or, orc.wq_bits[op.name], orc.wq.get('use_buckets', False),
                                         orc.wq.get('bucket_type', 'channel'), orc.wq.get('bucket_size', 256))
            print('    quantized weights engine vs oracle: max |d| %.3e' % float(np.abs(wq_gpu - w_or.numpy()).max()))
            # (2) prepared K-major copy vs the weights
            kk = wq_gpu.shape[-1]
            wmat = wq_gpu.reshape(-1, kk).T                     # [cout][(r,s,c)]
            prep = (tw.f_hi.float() + tw.f_lo.float()).cpu().numpy().reshape(kk, -1)[:, :wmat.shape[1]]
            print('    prepared fwd copy vs weights: max |d| %.3e (of %.3e)' % (float(np.abs(prep - wmat).max()),
                                                                               float(np.abs(wmat).max())))
            # (3) the conv recomputed now from the engine's own operand planes, both feeds, into a fresh buffer
            xp = ex.planes_of(op.inputs[0])
            for feed in (1, 0):
                ops.conv2d_tc_set_feed(feed)
                y2 = torch.full(tuple(op.output.shape), float('nan'), device=ex.device)
                ops.conv2d_tc_fwd_planes(d, xp, tw, None, False, y2)
                torch.cuda.synchronize()
                e2 = float(np.abs(y2.cpu().numpy() - b).max() / (np.abs(b).max() + 1e-12))
                e3 = float(np.abs(y2.cpu().numpy() - a).max() / (np.abs(b).max() + 1e-12))
                print('    recomputed (feed %d): vs oracle %.3e, vs the step\'s buffer %.3e' % (feed, e2, e3))
            ops.conv2d_tc_set_feed(-1)
            # (4) exact fp32 kernel on the reconstructed input
            xin = gpu_activation(ex, op.inputs[0].op) if op.inputs[0].op.type in ('Relu', 'Relu6') else ex.T(op.inputs[0]).cpu().numpy()
            y3 = torch.empty(tuple(op.output.shape), device=ex.device)
            ops.conv2d_fwd(d, torch.from_numpy(np.ascontiguousarray(xin)).to(ex.device), ex.kernel_of(op).contiguous(), None, False, y3)
            torch.cuda.synchronize()
            print('    exact-fp32 kernel on the same input / weights: vs oracle %.3e' % float(
                np.abs(y3.cpu().numpy() - b).max() / (np.abs(b).max() + 1e-12)))
            print('    input vs oracle input: %.3e' % float(np.abs(xin - xin_ref.numpy()).max() / (np.abs(xin_ref.numpy()).max() + 1e-12)))
        if shown < 400:
            print('  %-58s %-16s %s err %.2e%s' % (op.name[-58:], op.type, tuple(op.output.shape), err, mark))
            shown += 1


if __name__ == '__main__':
    main()

"""Storage format of tests/golden/learner_minibatch.pt (written by make_golden_minibatch.py), kept small:

* the weights before the update were rounded to values float16 holds exactly before the reference ran, and are stored
  as float16;
* the weights after the update are stored, for the trained tensors only, as int16 steps of 2^-23 from the weights
  before (six Adam steps of lr 5e-4 move a weight by less than 32767 steps).  The step is the float32 spacing of
  weights around 1, so decoding in float64 is within 6e-8 of the reference's float32 result; the writer asserts that.

``load`` returns the fixture with both decoded: ``*_before`` float32, ``*_after`` float64."""
import torch

STEP = 2.0 ** -23


def encode_after(after, before, keys):
    out = {}
    for k in keys:
        q = torch.round((after[k].double() - before[k].double()) / STEP)
        assert float(q.abs().max()) <= 32767 and float(q.abs().max()) > 0, k
        assert float((before[k].double() + q * STEP - after[k].double()).abs().max()) <= 0.5 * STEP, k
        out[k] = q.to(torch.int16)
    return out


def load(path):
    g = torch.load(path, weights_only=False)
    for kind in ("actors", "critics"):
        g[kind + "_before"] = [{k: v.float() if v.is_floating_point() else v for k, v in sd.items()} for sd in g[kind + "_before"]]
        g[kind + "_after"] = [{k: b[k].double() + q.double() * STEP for k, q in sd.items()}
                              for sd, b in zip(g[kind + "_after"], g[kind + "_before"])]
    return g

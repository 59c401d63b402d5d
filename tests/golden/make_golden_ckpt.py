"""Shrunk copies of the reference's shipped Lightning checkpoints, for the checkpoint-reader tests:
    python tests/golden/make_golden_ckpt.py
reads pretrained/{colab-lego-nerf-high-res,buff-synthetic-lego}/default/version_0/checkpoints/model_last.ckpt of the reference
and writes tests/golden/ckpt_lego_nerf.ckpt and ckpt_lego_buff.ckpt in the same legacy torch serialisation, with the same
pickled classes (pytorch_lightning.utilities.parsing.AttributeDict, nerf.cfgnode.CfgNode, nerf.tree.Node): every entry is kept
as it is (hyper-parameters, the BuFF tree with its node graph, voxels, weights and counter), except that the optimiser and
scheduler states are emptied and the state dict keeps only its tensors of at most 4096 elements (biases, encodings, heads,
tables), to stay far below 1 MB.
"""
import os
import pickle
import sys
import types

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/pretrained/{}/default/version_0/checkpoints/model_last.ckpt"

# stand-ins for the foreign classes: registered under their original module paths so that pickling them again writes the
# same GLOBAL records the reference's files hold
_STUBS = {("pytorch_lightning.utilities.parsing", "AttributeDict"): dict, ("nerf.cfgnode", "CfgNode"): dict, ("nerf.tree", "Node"): object}
for (mod, name), base in _STUBS.items():
    parts = mod.split(".")
    for i in range(1, len(parts) + 1):
        sys.modules.setdefault(".".join(parts[:i]), types.ModuleType(".".join(parts[:i])))
    cls = type(name, (base,), {"__module__": mod, "__qualname__": name})
    setattr(sys.modules[mod], name, cls)


class _Unpickler(pickle.Unpickler):
    def find_class(self, module, name):
        if (module, name) in _STUBS:
            return getattr(sys.modules[module], name)
        return super().find_class(module, name)


class _PickleModule:
    Unpickler = _Unpickler
    load = staticmethod(lambda f, **kw: _Unpickler(f, **kw).load())
    dump, dumps, Pickler = pickle.dump, pickle.dumps, pickle.Pickler


def shrink(src, dst):
    ck = torch.load(src, map_location="cpu", weights_only=False, pickle_module=_PickleModule)
    ck["optimizer_states"], ck["lr_schedulers"] = [], []
    sd = ck["state_dict"]
    for k in list(sd):
        if sd[k].numel() > 4096:
            del sd[k]
    torch.save(ck, dst, _use_new_zipfile_serialization=False)
    print(dst, os.path.getsize(dst))


if __name__ == "__main__":
    shrink(REF.format("colab-lego-nerf-high-res"), os.path.join(HERE, "ckpt_lego_nerf.ckpt"))
    shrink(REF.format("buff-synthetic-lego"), os.path.join(HERE, "ckpt_lego_buff.ckpt"))

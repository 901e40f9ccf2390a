"""Drop-in for the reference's ``reid_models/load_model_tools.py``: ``load_pretrained_weights(model, weight_path)``, what
``StrongSORT.__init__`` calls (reference strongsort.py:29).  Reads a checkpoint (a state dict, or a dict holding one under
'state_dict'), drops a DataParallel ``module.`` prefix, and loads every tensor whose name and shape the model has; the rest (the
checkpoint's classifier for another number of identities) is skipped and reported."""
import torch


def load_pretrained_weights(model, weight_path):
    ckpt = torch.load(weight_path, map_location='cpu', weights_only=False)
    sd = ckpt['state_dict'] if isinstance(ckpt, dict) and 'state_dict' in ckpt else ckpt
    own = model.state_dict()
    keep, skipped = {}, []
    for k, v in sd.items():
        k = k[7:] if k.startswith('module.') else k
        if k in own and own[k].size() == v.size():
            keep[k] = v
        else:
            skipped.append(k)
    if not keep:
        raise RuntimeError('load_pretrained_weights: no tensor of %s matches the model (check the checkpoint)' % weight_path)
    own.update(keep)
    model.load_state_dict(own)
    print('Successfully loaded pretrained weights from "%s"' % weight_path)
    if skipped:
        print('** The following layers are discarded due to unmatched keys or layer size: %s' % skipped)

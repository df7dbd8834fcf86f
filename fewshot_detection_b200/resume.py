"""The training-state file written beside each checkpoint's weight file, and the checks a resumed run makes on it.

The weight file (`%06d.weights`, the reference's format) holds the parameters and `seen` only.  A run continued from it
alone, as train_meta.py:93-99 does, restarts momentum from the gradient, recomputes its schedule position from `seen`
(which counts whole epochs of samples, not batches), resets region_loss.seen and reseeds its random streams.  The state
file `%06d.state` keeps what that loses, so `tools/train_meta_b200.py --resume` continues bit for bit as the run would
have gone on:

    format        FORMAT
    weights       {'name', 'bytes', 'sha256'} of the paired weight file
    fingerprint   what the run depends on (see fingerprint()): block lists, .data options, world, batches, training list
    seed          the seed the training list was built from
    trainer       MetaTrainer.state_dict() of rank 0 without its random generators: next epoch, processed_batches,
                  both `seen` counters, the optimizer's hyper-parameters and fp32 momentum (host copies, bits unchanged)
    ranks         per rank: {'model_seen', 'rng'} - the random generators (Python, numpy, torch CPU) of every rank,
                  which diverge after the first step (each rank's neg_filter draws once per empty row of its shard), and
                  model.seen, which only the saving rank updates

The file is `MAGIC`, the byte length of a JSON header, the header, then the raw bytes of every tensor in order.  The
header is the state with each tensor replaced by its dtype, shape and index, and tuples and dicts tagged so that they
read back as they were; it also records the data section's length, so a truncated file is recognised.  Nothing in it
depends on the time or the path of the write, so the same state always gives the same bytes.  It is written to a
temporary name and renamed, so a run killed mid-write leaves the previous file intact.
"""
import hashlib
import json
import os

import numpy as np
import torch

from .trainer import rng_state

FORMAT = 1
MAGIC = b'FSDET-TRAINING-STATE\n'
_DTYPES = ('float32', 'float64', 'int64', 'int32', 'uint8')


class StateFileError(ValueError):
    """A state file that cannot be used to resume this run; the message names the file and both values."""


def file_digest(path, chunk=1 << 24):
    """{'name', 'bytes', 'sha256'} of a file."""
    h = hashlib.sha256()
    n = 0
    with open(path, 'rb') as f:
        while True:
            b = f.read(chunk)
            if not b:
                break
            h.update(b)
            n += len(b)
    return dict(name=os.path.basename(path), bytes=n, sha256=h.hexdigest())


def _sha(obj):
    return hashlib.sha256(json.dumps(obj, sort_keys=True).encode()).hexdigest()


def fingerprint(darknet_blocks, learnet_blocks, data_options, world, batch_size, per_rank, trainlist=None, replicas=None):
    """What a resumed run must share with the run that wrote the state: the parsed darknet and learnet block lists, the
    `.data` options, the world size, the replicas per step (nn.DataParallel replicas, default one per rank), the global
    and per-rank batch and the built training list (length and hash; left out while trainlist is None, so the other
    values can be checked before the list is built)."""
    fp = dict(cfg=_sha([[dict(b) for b in darknet_blocks], [dict(b) for b in learnet_blocks]]),
              data=dict(data_options), world=int(world), batch=int(batch_size), per_rank=int(per_rank),
              replicas=int(world if replicas is None else replicas))
    if trainlist is not None:
        fp['trainlist'] = dict(n=len(trainlist), sha256=_sha([str(l) for l in trainlist]))
    return fp


def _encode(obj, tensors):
    if torch.is_tensor(obj):
        t = obj.detach().to('cpu').contiguous()
        name = str(t.dtype).replace('torch.', '')
        if name not in _DTYPES:
            raise TypeError('state file: tensors of dtype %s are not stored' % name)
        tensors.append(t)
        return {'t': [len(tensors) - 1, name, list(t.shape)]}
    if isinstance(obj, dict):
        return {'d': [[_encode(k, tensors), _encode(v, tensors)] for k, v in obj.items()]}
    if isinstance(obj, tuple):
        return {'u': [_encode(v, tensors) for v in obj]}
    if isinstance(obj, list):
        return [_encode(v, tensors) for v in obj]
    if obj is None or isinstance(obj, (bool, int, float, str)):
        return obj
    raise TypeError('state file: cannot store a %s' % type(obj).__name__)


def _decode(obj, tensors):
    if isinstance(obj, list):
        return [_decode(v, tensors) for v in obj]
    if isinstance(obj, dict):
        (tag, v), = obj.items()
        if tag == 't':
            return tensors[v[0]]
        if tag == 'd':
            return {_decode(k, tensors): _decode(x, tensors) for k, x in v}
        return tuple(_decode(x, tensors) for x in v)
    return obj


def write_state(path, state):
    """Write `state` (dicts, lists, tuples, numbers, strings and tensors) to `path` atomically: a temporary file in the
    same directory, flushed to disk, then renamed over `path`.  On any failure the temporary file is removed and an
    existing `path` is left as it was."""
    tensors = []
    body = _encode(state, tensors)
    sizes = [t.numel() * t.element_size() for t in tensors]
    header = json.dumps(dict(body=body, tensors=[[str(t.dtype).replace('torch.', ''), list(t.shape)] for t in tensors],
                             data_bytes=sum(sizes)), sort_keys=True).encode()
    tmp = path + '.tmp'
    try:
        with open(tmp, 'wb') as f:
            f.write(MAGIC + len(header).to_bytes(8, 'little') + header)
            for t in tensors:
                f.write(t.numpy().tobytes() if t.dim() == 0 else memoryview(t.numpy()).cast('B'))
            f.flush()
            os.fsync(f.fileno())
        os.replace(tmp, path)
    except BaseException:
        if os.path.exists(tmp):
            os.remove(tmp)
        raise


def read_state(path):
    """Load a state file; refuses a missing, truncated or foreign file and an unknown format version."""
    if not os.path.isfile(path):
        raise StateFileError('state file %s: no such file' % path)
    size = os.path.getsize(path)
    with open(path, 'rb') as f:
        blob = f.read()
    n0 = len(MAGIC) + 8
    if blob[:len(MAGIC)] != MAGIC:
        raise StateFileError('state file %s (%d bytes): not a training-state file' % (path, size))
    try:
        hlen = int.from_bytes(blob[len(MAGIC):n0], 'little')
        header = json.loads(blob[n0:n0 + hlen].decode())
        want = n0 + hlen + int(header['data_bytes'])
    except Exception as e:
        raise StateFileError('state file %s (%d bytes) is truncated or damaged: %s' % (path, size, e))
    if size != want:
        raise StateFileError('state file %s is %d bytes, its header says %d: truncated or damaged' % (path, size, want))
    tensors, off = [], n0 + hlen
    for name, shape in header['tensors']:
        n = int(np.prod(shape, dtype=np.int64)) * np.dtype(name).itemsize
        tensors.append(torch.from_numpy(np.frombuffer(blob, dtype=name, count=n // np.dtype(name).itemsize,
                                                      offset=off).reshape(shape).copy()))
        off += n
    state = _decode(header['body'], tensors)
    if not isinstance(state, dict) or 'format' not in state:
        raise StateFileError('state file %s: not a training-state file' % path)
    if state['format'] != FORMAT:
        raise StateFileError('state file %s has format version %r, this version reads %r' % (path, state['format'], FORMAT))
    return state


def check_weights(state, path, weightfile):
    """The positional weight file must be the one the state was written with (same size and sha256)."""
    if not os.path.isfile(weightfile):
        raise StateFileError('state file %s pairs with %s (%d bytes), but weight file %s does not exist'
                             % (path, state['weights']['name'], state['weights']['bytes'], weightfile))
    got = file_digest(weightfile)
    want = state['weights']
    if (got['bytes'], got['sha256']) != (want['bytes'], want['sha256']):
        raise StateFileError('state file %s pairs with %s (%d bytes, sha256 %s), weight file %s is %d bytes, sha256 %s'
                             % (path, want['name'], want['bytes'], want['sha256'], weightfile, got['bytes'], got['sha256']))


def check_fingerprint(state, path, current):
    """Compare `current` (fingerprint() of this run) with the stored one, key by key in the order world, batches, cfg,
    .data, training list; the first difference is refused with both values."""
    stored = dict(state['fingerprint'])
    stored.setdefault('replicas', stored.get('world'))     # written before replicas were recorded: one per rank
    names = dict(world='world size', replicas='replicas per step', batch='global batch', per_rank='per-rank batch',
                 cfg='cfg block lists (sha256)', data='.data options', trainlist='training list')
    for k in [k for k in names if k in current]:
        if stored[k] != current[k]:
            if k == 'data':
                diff = sorted(n for n in set(stored[k]) | set(current[k]) if stored[k].get(n) != current[k].get(n))
                raise StateFileError('state file %s was written with .data options %s, this run has %s'
                                     % (path, {n: stored[k].get(n) for n in diff}, {n: current[k].get(n) for n in diff}))
            raise StateFileError('state file %s was written with %s %s, this run has %s' % (path, names[k], stored[k], current[k]))


def state_path(weightfile_path):
    """`backup/000004.weights` -> `backup/000004.state`."""
    stem, ext = os.path.splitext(weightfile_path)
    return stem + '.state'


def state_saver(fp, seed, world=1, rank=0, log=print):
    """save_state(trainer, epoch) for MetaTrainer: on every rank, gathers each rank's random generators and model.seen
    to rank 0, which writes `<backupdir>/%06d.state` beside the epoch's weight file and then deletes the state file it
    wrote at the previous checkpoint (and no other file)."""
    last = []

    def save_state(trainer, epoch):
        import time
        t0 = time.time()
        sd = trainer.state_dict() if rank == 0 else None
        mine = dict(model_seen=int(trainer.model.seen), rng=rng_state())
        if world > 1:
            import torch.distributed as dist
            ranks = [None] * world
            dist.all_gather_object(ranks, mine)
        else:
            ranks = [mine]
        if rank != 0 or trainer.backupdir is None:
            return
        rng_free = {k: v for k, v in sd.items() if k not in ('rng', 'model_seen')}
        weights = '%s/%06d.weights' % (trainer.backupdir, epoch)
        path = state_path(weights)
        write_state(path, dict(format=FORMAT, weights=file_digest(weights), fingerprint=fp, seed=int(seed),
                               trainer=rng_free, ranks=ranks))
        for old in last:
            if old != path and os.path.exists(old):
                os.remove(old)
        last[:] = [path]
        log('save training state to %s (%.2f s)' % (path, time.time() - t0))
    return save_state


def restore(trainer, state, rank=0):
    """Load rank `rank`'s view of `state` into a MetaTrainer (MetaTrainer.load_state_dict): the shared schedule and
    optimizer state, this rank's model.seen and random generators.  Call it last before fit(): it sets the generators."""
    if rank >= len(state['ranks']):
        raise StateFileError('state file holds %d ranks, this is rank %d' % (len(state['ranks']), rank))
    sd = dict(state['trainer'])
    sd.update(state['ranks'][rank])
    trainer.load_state_dict(sd)

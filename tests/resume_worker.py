"""Subprocess side of tests/test_gpu_resume.py: the training driver (tools/train_meta_b200.py) on the synthetic VOC set of
tools/e2e_train_synth.py, with what the test compares written under an output directory.

    python tests/resume_worker.py setup ROOT base|tune        data set, cfgs, .data file, starting weights (seen 256000)
    python tests/resume_worker.py run ROOT base|tune OUT STOP [driver flags...]
    torchrun --nproc-per-node 2 tests/resume_worker.py run ...

`run` trains with save_interval 1 and stops after epoch STOP (0: runs to the end).  After every epoch rank 0 copies
each weight and state file of the backup directory to OUT/files/ and appends the epoch's steps to OUT/steps.txt, one
line per step: epoch, input size, loss (float.hex)."""
import os
import shutil
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
N_IMAGES = 256
SEEN = 256000          # past 4000 batches of 64: the multi-scale schedule draws a size every 64 samples


def load(path, name):
    import importlib.util
    spec = importlib.util.spec_from_file_location(name, path)
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def data_file(root, mode):
    return os.path.join(root, mode + '.data')


def setup(root, mode):
    import torch
    from fewshot_detection_b200 import netcfg
    from fewshot_detection_b200.cfg import cfg
    from fewshot_detection_b200.darknet_meta import Darknet
    from fewshot_detection_b200.utils import read_data_cfg
    from fewshot_detection_b200 import lists as LS
    synth = load(os.path.join(ROOT, 'tools', 'e2e_train_synth.py'), 'e2e_train_synth')
    if not os.path.exists(os.path.join(root, 'novels.txt')):
        synth.make_dataset(root, N_IMAGES)
    lists = os.path.join(root, 'lists')
    shutil.copy(os.path.join(lists, 'dict_full.txt'), os.path.join(lists, 'dict_3shot.txt'))   # cfg.shot from the name
    common = 'metayolo=1\nmetain_type=2\ndata=voc\nrand = 0\nnovel = %s\nnovelid = 0\ntrain = %s\nbackup = %s\n' % (
        os.path.join(root, 'novels.txt'), os.path.join(lists, 'train.txt'), os.path.join(root, 'backup'))
    with open(data_file(root, mode), 'w') as f:
        if mode == 'base':
            f.write(common + 'neg = 1\nmeta = %s\n' % os.path.join(lists, 'dict_full.txt'))
        else:
            f.write(common + 'neg = 0\ntuning = 1\nmax_epoch = 4\nrepeat = 1\nmeta = %s\n' % os.path.join(lists, 'dict_3shot.txt'))
    det = netcfg.darknet_dynamic_blocks()
    det[0]['batch'] = '64'
    if mode == 'base':                 # four epochs after the starting weights' seen: max_epochs = init_epoch + 4
        cfg.config_data(read_data_cfg(data_file(root, mode)))
        nsamples = len(LS.build_dataset(read_data_cfg(data_file(root, mode))))
        det[0]['max_batches'] = str(((SEEN // nsamples + 3) * nsamples + 63) // 64)
    netcfg.write_cfg(det, os.path.join(root, mode + '_dyn.cfg'))
    netcfg.write_cfg(netcfg.reweighting_net_blocks(), os.path.join(root, 'rw.cfg'))
    wfile = os.path.join(root, 'init.weights')
    if not os.path.exists(wfile):
        torch.manual_seed(0)
        m0 = Darknet(det, netcfg.reweighting_net_blocks())
        head = [mod for mod in m0.models if isinstance(mod, torch.nn.Sequential)][-1][0]
        with torch.no_grad():
            head.weight.mul_(0.02)
            head.bias.zero_()
        m0.seen = SEEN
        m0.save_weights(wfile)
    return 0


def run(root, mode, out, stop, flags):
    import torch
    from fewshot_detection_b200 import trainer as T
    from fewshot_detection_b200.cfg import cfg
    cli = load(os.path.join(ROOT, 'tools', 'train_meta_b200.py'), 'train_meta_b200')
    rank = int(os.environ.get('RANK', '0'))
    files = os.path.join(out, 'files')
    os.makedirs(files, exist_ok=True)
    steps = []

    class Stop(Exception):
        pass

    orig_step, orig_epoch = T.MetaTrainer.train_step, T.MetaTrainer.train_epoch

    def train_step(self, data, metax, mask, target):
        loss = orig_step(self, data, metax, mask, target)
        steps.append((int(data.size(-1)), loss.detach().clone()))
        return loss

    def train_epoch(self, epoch, max_epochs=None):
        nb = orig_epoch(self, epoch, max_epochs)
        if rank == 0:
            with open(os.path.join(out, 'steps.txt'), 'a') as f:
                f.write(''.join('%d %d %s\n' % (epoch, s, float(l).hex()) for s, l in steps))
            for name in os.listdir(self.backupdir):
                if name.endswith('.weights') or name.endswith('.state'):
                    shutil.copy(os.path.join(self.backupdir, name), os.path.join(files, name))
        del steps[:]
        if stop and epoch + 1 - self.first_epoch >= stop:
            raise Stop()
        return nb

    orig_fit = T.MetaTrainer.fit

    def fit(self, init_epoch, max_epochs):
        self.first_epoch = self.resume_epoch if self.resume_epoch is not None else int(init_epoch)
        return orig_fit(self, init_epoch, max_epochs)
    T.MetaTrainer.train_step, T.MetaTrainer.train_epoch, T.MetaTrainer.fit = train_step, train_epoch, fit
    if mode == 'base':
        cfg.save_interval = 1          # fine-tuning with max_epoch 4, repeat 1 saves every epoch by itself
    sys.argv = ['train_meta_b200.py', data_file(root, mode), os.path.join(root, mode + '_dyn.cfg'),
                os.path.join(root, 'rw.cfg')] + flags
    try:
        rc = cli.main()
    except Stop:
        rc = 0
        torch.cuda.synchronize()
    return rc


if __name__ == '__main__':
    if sys.argv[1] == 'setup':
        sys.exit(setup(sys.argv[2], sys.argv[3]))
    sys.exit(run(sys.argv[2], sys.argv[3], sys.argv[4], int(sys.argv[5]), sys.argv[6:]))

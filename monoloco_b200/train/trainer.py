"""`Trainer`: the reference's training entry point (monoloco/train/trainer.py:36-389, driven by run.py train and
hyp_tuning.py) on the fused kernels, with the same constructor, attributes, methods and results.

Per train batch: `train_step` (forward + multi-task loss + backward, one launch), `FusedClipAdam` (clip + Adam, two
launches), `StepLR`, and one `mlb_task_stats` launch that adds the batch's loss statistics into an fp64 epoch
accumulator on the device -- four library launches and no host synchronisation. Per val batch: one eval forward and one
statistics launch. The accumulators cross to the host once per epoch. `evaluate()` runs one eval forward over the val
split and its distance clusters, one statistics launch over the five segments and one copy back.

Differences from the reference, on purpose: CUDA only; `debug=True` (interactive histograms) is refused; the statistics
are summed in fp64 where the reference sums fp32 means. Quirks kept as they are: see INTEGRATION.md."""
import copy
import datetime
import logging
import os
import time
from collections import defaultdict
from itertools import chain

import numpy as np
import torch
from torch.optim import lr_scheduler

try:
    import matplotlib.pyplot as plt
except ImportError:
    plt = None

from .. import _lib as L_
from ..network.architectures import LocoModel
from ..utils.logs import set_logger
from .datasets import DeviceLoader, KeypointsDataset
from .fused import train_step
from .losses import AutoTuneMultiTaskLoss, CompositeLoss, MultiTaskLoss
from .optim import FusedClipAdam
from .stats import err_std, task_stats, val_values


class Trainer:
    VAL_BS = 10000

    tasks = ('d', 'x', 'y', 'h', 'w', 'l', 'ori', 'aux')
    val_task = 'd'
    lambdas = (1, 1, 1, 1, 1, 1, 1, 1)
    clusters = ['10', '20', '30', '40']
    input_size = dict(mono=34, stereo=68)
    output_size = dict(mono=9, stereo=10)
    dir_figures = os.path.join('figures', 'losses')

    def __init__(self, args):
        assert os.path.exists(args.joints), "Input file not found"
        self.mode = args.mode
        self.joints = args.joints
        self.num_epochs = args.epochs
        self.no_save = args.no_save
        self.print_loss = args.print_loss
        self.lr = args.lr
        self.sched_step = args.sched_step
        self.sched_gamma = args.sched_gamma
        self.hidden_size = args.hidden_size
        self.n_stage = args.n_stage
        self.r_seed = args.r_seed
        self.auto_tune_mtl = args.auto_tune_mtl

        if args.out:
            self.path_out = args.out
            dir_out = os.path.split(self.path_out)[0]
        else:
            dir_out = os.path.join('data', 'outputs')
            stamp = datetime.datetime.now().strftime("%Y%m%d-%H%M")[2:]
            self.path_out = os.path.join(dir_out, '%s-%s.pkl' % ('monoloco_pp' if self.mode == 'mono' else 'monstereo',
                                                                 stamp))
        assert os.path.exists(dir_out), "Directory to save the model not found"
        print(self.path_out)
        if not torch.cuda.is_available():
            raise RuntimeError("monoloco_b200 Trainer runs on CUDA only (no CPU fallback)")
        self.device = torch.device('cuda')
        print('Device: ', self.device)
        torch.manual_seed(self.r_seed)
        torch.cuda.manual_seed(self.r_seed)

        if self.mode == 'mono' and self.tasks[-1] == 'aux':
            self.tasks, self.lambdas = self.tasks[:-1], self.lambdas[:-1]
        losses_tr, losses_val = CompositeLoss(self.tasks)()
        loss_cls = AutoTuneMultiTaskLoss if self.auto_tune_mtl else MultiTaskLoss
        self.mt_loss = loss_cls(losses_tr, losses_val, self.lambdas, self.tasks)
        self.mt_loss.to(self.device)

        # device-resident splits; with shuffle=True both draw their permutations from the global generator exactly as
        # the reference's DataLoaders do, so the batches and their order are the reference's
        self.datasets = {phase: KeypointsDataset(self.joints, phase=phase) for phase in ('train', 'val')}
        self.dataloaders = {phase: DeviceLoader(ds, batch_size=args.bs, shuffle=True, device=self.device)
                            for phase, ds in self.datasets.items()}
        self.dataset_sizes = {phase: len(ds) for phase, ds in self.datasets.items()}
        self.dataset_version = self.datasets['train'].get_version()

        self._set_logger(args)
        self.logger.info('Sizes of the dataset: {}'.format(self.dataset_sizes))
        print(">>> creating model")
        # built on the CPU, then moved: the initial weights draw from the CPU generator as the reference's do
        self.model = LocoModel(input_size=self.input_size[self.mode], output_size=self.output_size[self.mode],
                               linear_size=args.hidden_size, p_dropout=args.dropout, num_stage=self.n_stage,
                               device=self.device)
        self.model.to(self.device)
        print(">>> model params: {:.3f}M".format(sum(p.numel() for p in self.model.parameters()) / 1000000.0))
        print(">>> loss params: {}".format(sum(p.numel() for p in self.mt_loss.parameters())))

        self.optimizer = FusedClipAdam(chain(self.model.parameters(), self.mt_loss.parameters()), lr=args.lr,
                                       max_norm=3, clip_params=list(self.model.parameters()))
        self.scheduler = lr_scheduler.StepLR(self.optimizer, step_size=self.sched_step, gamma=self.sched_gamma)
        self._log_sigmas = self.mt_loss.log_sigmas if self.auto_tune_mtl else None

    # ------------------------------------------------------------------------------------------------ training
    def _run_phase(self, phase, acc):
        """One pass over a split; adds every batch's statistics into `acc` ([1, STATS_NACC] fp64, device)."""
        for inputs, labels, _, _ in self.dataloaders[phase]:
            if phase == 'train':
                self.optimizer.zero_grad()
                _, _, outputs = train_step(self.model, inputs, labels, self.tasks, self.lambdas, self._log_sigmas)
                self.optimizer.step()
                self.scheduler.step()
            else:
                with torch.no_grad():
                    outputs = self.model(inputs)
            # after optimizer.step(): the train-form total sees the updated log_sigmas, as trainer.py:166 does
            task_stats(outputs, labels, (0, inputs.shape[0]), self.tasks, self.lambdas, self._log_sigmas, acc=acc)

    def train(self):
        since = time.time()
        best_model_wts = copy.deepcopy(self.model.state_dict())
        best_acc, best_training_acc, best_epoch = 1e6, 1e6, 0
        epoch_losses = defaultdict(lambda: defaultdict(list))
        acc = torch.empty((2, L_.STATS_NACC), dtype=torch.float64, device=self.device)
        for epoch in range(self.num_epochs):
            acc.zero_()
            for i, phase in enumerate(('train', 'val')):
                self.model.train(phase == 'train')
                self._run_phase(phase, acc[i:i + 1])
            host = acc.cpu().numpy()   # the epoch's one device-to-host copy
            running_loss = defaultdict(lambda: defaultdict(int))
            for i, phase in enumerate(('train', 'val')):
                running_loss[phase]['all'] = float(host[i, L_.STAT_TOTAL])
                # sum over batches of (batch mean * batch rows) = sum over rows
                for task, v in zip(self.tasks, val_values(host[i], self.tasks)):
                    running_loss[phase][task] = float(v * host[i, L_.STAT_N])
            self.cout_values(epoch, epoch_losses, running_loss)
            if epoch_losses['val'][self.val_task][-1] < best_acc:
                best_acc = epoch_losses['val'][self.val_task][-1]
                best_training_acc = epoch_losses['train']['all'][-1]
                best_epoch = epoch
                best_model_wts = copy.deepcopy(self.model.state_dict())

        elapsed = time.time() - since
        print('\n\n' + '-' * 120)
        self.logger.info('Training:\nTraining complete in {:.0f}m {:.0f}s'.format(elapsed // 60, elapsed % 60))
        self.logger.info('Best training Accuracy: {:.3f}'.format(best_training_acc))
        self.logger.info('Best validation Accuracy for {}: {:.3f}'.format(self.val_task, best_acc))
        self.logger.info('Saved weights of the model at epoch: {}'.format(best_epoch))
        self._print_losses(epoch_losses)
        self.model.load_state_dict(best_model_wts)
        return best_epoch

    def epoch_logs(self, phase, loss, loss_values, inputs, running_loss):
        """trainer.py:193-197 for a caller that holds per-batch losses (the loop above sums on the device instead)."""
        rows = inputs.size(0)
        running_loss[phase]['all'] += float(loss) * rows
        for task, value in zip(self.tasks, loss_values):
            running_loss[phase][task] += float(value) * rows

    # ------------------------------------------------------------------------------------------------ evaluation
    def evaluate(self, load=False, model=None, debug=False):
        if debug:
            raise NotImplementedError("evaluate(debug=True) shows interactive input histograms and exits; not supported")
        if load:
            self.model.load_state_dict(torch.load(model, map_location=lambda storage, loc: storage))
        self.model.eval()
        dic_err = defaultdict(lambda: defaultdict(lambda: defaultdict(lambda: 0)))
        dic_err['val']['sigmas'] = [0.] * len(self.tasks)
        dataset = KeypointsDataset(self.joints, phase='val')
        size_eval = len(dataset)
        # the reference evaluates in chunks of VAL_BS rows and asserts on the first one when there is more than one
        assert size_eval <= self.VAL_BS, "Variance of errors not supported with partial evaluation"
        xs, ys, sizes = [dataset.inputs_all], [dataset.outputs_all], [size_eval]
        for clst in self.clusters:
            x, y, n = dataset.get_cluster_annotations(clst)
            xs.append(x)
            ys.append(y)
            sizes.append(n)
        off = np.concatenate(([0], np.cumsum(sizes))).tolist()
        with torch.no_grad():
            x = torch.cat(xs).to(self.device)
            y = torch.cat(ys).to(self.device)
            outputs = self.model(x)
            acc = task_stats(outputs, y, off, self.tasks, self.lambdas, self._log_sigmas)
        host, sigma_exp = self._to_host(acc)
        for s, clst in enumerate(['all'] + list(self.clusters)):
            if sizes[s] > 0 or clst != 'all':
                self._stats_into(host[s], sigma_exp, dic_err['val'], sizes[s], clst)
            self.cout_stats(dic_err['val'], sizes[s], clst=clst)

        if not (self.no_save or load):
            torch.save(self.model.state_dict(), self.path_model)
            print('-' * 120)
            self.logger.info("\nmodel saved: {} \n".format(self.path_model))
        else:
            self.logger.info("\nmodel not saved\n")
        return dic_err, self.model

    def _to_host(self, acc):
        """Accumulators (and exp(log_sigmas) for AutoTune) in one device-to-host copy."""
        flat = acc.flatten()
        if self._log_sigmas is not None:
            flat = torch.cat((flat, self._log_sigmas.detach().double().exp()))
        flat = flat.cpu().numpy()
        n = acc.numel()
        return flat[:n].reshape(acc.shape), (flat[n:].tolist() if self._log_sigmas is not None else None)

    def compute_stats(self, outputs, labels, dic_err, size_eval, clst):
        """trainer.py:250-284 on one (outputs, labels) pair: one statistics launch and one copy back."""
        with torch.no_grad():
            acc = task_stats(outputs, labels, (0, outputs.size(0)), self.tasks, self.lambdas, self._log_sigmas)
        host, sigma_exp = self._to_host(acc)
        self._stats_into(host[0], sigma_exp, dic_err, size_eval, clst)

    def _stats_into(self, row, sigma_exp, dic_err, size_eval, clst):
        n = int(row[L_.STAT_N])
        rel_frac = n / size_eval
        # what mt_loss(..., phase='val') returns: val-form means, then exp(log_sigma) per task for AutoTune
        loss_values = val_values(row, self.tasks) + (list(sigma_exp) if sigma_exp is not None else [])
        tasks = self.tasks[:-1] if self.tasks[-1] == 'aux' else self.tasks
        for idx, task in enumerate(tasks):
            dic_err[clst][task] += float(loss_values[idx]) * rel_frac
        assert rel_frac > 0.99, "Variance of errors not supported with partial evaluation"
        dic_err[clst]['bi'] += float(row[L_.STAT_BI] / n) * rel_frac
        dic_err[clst]['bi%'] += float(row[L_.STAT_BI_HIT]) / n * rel_frac
        dic_err[clst]['std'] = torch.tensor(err_std(row), dtype=torch.float32)   # assigned, not accumulated
        if self.mode == 'mono':
            dic_err[clst]['aux'] = 0
            dic_err['sigmas'].append(0)
        else:
            dic_err[clst]['aux'] += (1. - float(row[L_.STAT_AUX_MISS]) / n) * rel_frac
        if self.auto_tune_mtl:
            assert len(loss_values) == 2 * len(self.tasks)
            # trainer.py:284 indexes from len(tasks without aux) + 1: right for stereo, past the end for mono
            for i in range(len(self.tasks)):
                dic_err['sigmas'][i] += float(loss_values[len(tasks) + i + 1]) * rel_frac

    # ------------------------------------------------------------------------------------------------ printing
    def cout_stats(self, dic_err, size_eval, clst):
        e = dic_err[clst]
        if clst == 'all':
            print('-' * 120)
            self.logger.info(
                "Evaluation, val set: \nAv. dist D: {:.2f} m with bi {:.2f} ({:.1f}%), \nX: {:.1f} cm,  Y: {:.1f} cm "
                "\nOri: {:.1f}  \n H: {:.1f} cm, W: {:.1f} cm, L: {:.1f} cm\nAuxiliary Task: {:.1f} %, ".format(
                    e['d'], e['bi'], e['bi%'] * 100, e['x'] * 100, e['y'] * 100, e['ori'], e['h'] * 100,
                    e['w'] * 100, e['l'] * 100, e['aux'] * 100))
            if self.auto_tune_mtl:
                self.logger.info("Sigmas: Z: {:.2f}, X: {:.2f}, Y:{:.2f}, H: {:.2f}, W: {:.2f}, L: {:.2f}, ORI: {:.2f}"
                                 " AUX:{:.2f}\n".format(*dic_err['sigmas']))
            return
        self.logger.info(
            "Val err clust {} --> D:{:.2f}m,  bi:{:.2f} ({:.1f}%), STD:{:.1f}m   X:{:.1f} Y:{:.1f}  Ori:{:.1f}d,   "
            "H: {:.0f} W: {:.0f} L:{:.0f}  for {} pp. ".format(
                clst, e['d'], e['bi'], e['bi%'] * 100, e['std'], e['x'] * 100, e['y'] * 100, e['ori'], e['h'] * 100,
                e['w'] * 100, e['l'] * 100, size_eval))

    def cout_values(self, epoch, epoch_losses, running_loss):
        """Appends every phase's per-row means to epoch_losses; prints them every 10 epochs."""
        parts, values = ['\r{:.0f} '], [epoch]
        for phase in running_loss:
            parts.append(phase[:1].upper() + ':')
            for el in running_loss['train']:
                loss = running_loss[phase][el] / self.dataset_sizes[phase]
                epoch_losses[phase][el].append(loss)
                if el == 'all':
                    parts.append(':{:.1f}  ')
                elif el in ('ori', 'aux'):
                    parts.append(el + ':{:.1f}  ')
                else:
                    parts.append(el + ':{:.0f}  ')
                    loss = loss * 100
                values.append(loss)
        if epoch % 10 == 0:
            print(''.join(parts).format(*values))

    def _print_losses(self, epoch_losses):
        if not self.print_loss:
            return
        os.makedirs(self.dir_figures, exist_ok=True)
        if plt is None:
            raise Exception('please install matplotlib')
        for i, phase in enumerate(epoch_losses):
            for j, el in enumerate(epoch_losses['train']):
                plt.figure(i + j)
                plt.title(phase + '_' + el)
                plt.xlabel('epochs')
                plt.plot(epoch_losses[phase][el][10:], label='{} Loss: {}'.format(phase, el))
                plt.savefig(os.path.join(self.dir_figures, '{}_loss_{}.png'.format(phase, el)))
                plt.close()

    def _set_logger(self, args):
        if self.no_save:
            logging.basicConfig(level=logging.INFO)
            self.logger = logging.getLogger(__name__)
            return
        self.path_model = self.path_out
        print(self.path_model)
        self.logger = set_logger(os.path.splitext(self.path_out)[0])
        self.logger.info(
            '\nVERSION: monoloco_b200\n\nINPUT_FILE: {}\nInput file version: {}\nTorch version: {}\n\nTraining arguments:'
            '\nmode: {} \nlearning rate: {} \nbatch_size: {}\nepochs: {} \ndropout: {} \nscheduler step: {} '
            '\nscheduler gamma: {} \ninput_size: {} \noutput_size: {} \nhidden_size: {} \nn_stages: {} \n r_seed: {} '
            '\nlambdas: {}'.format(args.joints, self.dataset_version, torch.__version__, self.mode, args.lr, args.bs,
                                   args.epochs, args.dropout, args.sched_step, args.sched_gamma,
                                   self.input_size[self.mode], self.output_size[self.mode], args.hidden_size,
                                   args.n_stage, args.r_seed, self.lambdas))

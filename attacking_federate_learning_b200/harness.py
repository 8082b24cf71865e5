"""`main.py`-equivalent experiment loop with the stacked client gradients resident on the GPU (SURVEY 8f rank 4).

Reference behaviour mirrored (file:line in /root/reference):
    main(...)                      main.py:12-100   build users + server, epoch loop, test every 5 epochs, CSV, checkpoint
    corrupted_count, is_malicious  main.py:21,28    malicious ids are 0..int(mal_prop*N)-1
    epoch body                     main.py:64-71    dispatch_weights -> attacker.attack(mal_users) -> collect -> defend
    attacker                       main.py:44-54    -b pattern|1|2|3: BackdoorAttack (alpha 4, 5 malicious epochs,
                                                    main.py:139-142) with backdoor.py:13-159's training restated on
                                                    the synthetic data (BackdoorTrainer); otherwise DriftAttack (ALIE)
    backdoor check                 main.py:91-95    the global model tested on the backdoor data ('POST') at every test
    learning-rate fading           server.py:50-52  lr_t = lr * fading / (epoch + fading) for the CLIENT optimiser only;
                                                    the server step uses the base rate (server.py:89, reproduced)
    test                           server.py:92-112 sum of per-batch NLL / dataset size, argmax accuracy
    outputs                        main.py:85-89    torch.save({'epoch','state_dict','acc'}) to runs/<dataset>/checkpoint.pth.tar
                                   main.py:100      np.savetxt('logs/<...>.csv', accuracies, delimiter=',')

What differs, on purpose: (i) the reference downloads its datasets (data_sets.py:30, 60), which is impossible offline,
so without data_dir the clients train on a seeded synthetic 10-class 28x28 problem with the reference's MnistNet
architecture (data_sets.py:13-24, D = 79,510), or with -s CIFAR10 on a seeded synthetic [3, 32, 32] problem with
Cifar10Net (data_sets.py:33-52, D = 117,706), each user holding rows u, u + n, ... of it.  With data_dir (--data-dir:
the directory that holds torchvision's files, e.g. the reference's ./mnist_data or ./cifar10_data) they train on the
real MNIST or CIFAR10 through the reference's transforms (data.load), each user holding its DistributedSampler shard
(user.py:49-54, data.sampler_order) and the attacker its backdoor.py loader's rows (data.backdoor_indices), under the
reference's log and checkpoint names; (ii) clients are evaluated on the GPU and write their flat gradients straight
into their row of the device-resident N x D matrix (ingest.ParamLayout: user.py:17-28 order), so attack, defence and the server step never
leave the device.  The training simulation itself is not part of the accelerated path (SURVEY 2).

    python -m attacking_federate_learning_b200.harness -d Krum -e 30 --users-count 10
    python -m attacking_federate_learning_b200.harness -d Krum -e 30 -z 1.0 -b pattern

A grid of these experiments (defence x z x malicious share x users x seed) runs as one batch in `sweep.run` / `python -m
attacking_federate_learning_b200.sweep`: each experiment starts from `experiment_setup`'s data and weights, as here,
and the client gradients of every experiment come from one CUDA kernel instead of this file's per-client autograd (and,
with -b, the attacker's training of every backdoor experiment from another, on `backdoor_set`'s data).
"""
from __future__ import annotations

import argparse
import datetime
import os

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import batched
from . import data as _data
from . import defences
from . import malicious
from . import metrics
from .ingest import ParamLayout
from .server import AggregationServer

SYNTH = 'SYNTH-MNIST'
SYNTH_CIFAR10 = 'SYNTH-CIFAR10'
DATASETS = ('MNIST', 'CIFAR10')                  # main.py -s


class MnistNet(nn.Module):                       # data_sets.py:13-24
    def __init__(self):
        super().__init__()
        self.fc1 = nn.Linear(28 * 28, 100)
        torch.nn.init.xavier_uniform_(self.fc1.weight)
        self.fc2 = nn.Linear(100, 10)

    def forward(self, x):
        return F.log_softmax(self.fc2(F.relu(self.fc1(x))), dim=1)


class Cifar10Net(nn.Module):                     # data_sets.py:33-52
    def __init__(self):
        super().__init__()
        self.conv1 = nn.Conv2d(3, 16, 3)
        torch.nn.init.xavier_uniform_(self.conv1.weight)
        self.pool1 = nn.MaxPool2d(3)
        self.conv2 = nn.Conv2d(16, 64, 4)
        self.pool2 = nn.MaxPool2d(4)
        self.fc1 = nn.Linear(64, 384)
        self.fc2 = nn.Linear(384, 192)
        self.fc3 = nn.Linear(192, 10)

    def forward(self, x):
        x = self.pool1(F.relu(self.conv1(x)))
        x = self.pool2(F.relu(self.conv2(x)))
        x = F.relu(self.fc1(x.view(x.size(0), -1)))
        x = F.relu(self.fc2(x))
        return F.log_softmax(self.fc3(x), dim=1)


def synthetic_problem(n_train, n_test, device, seed=0):
    """10 Gaussian class prototypes in 784 dimensions + noise: learnable to > 90 % by the MLP in a few dozen rounds."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    protos = torch.randn(10, 28 * 28, generator=g)

    def draw(n):
        y = torch.randint(0, 10, (n,), generator=g)
        x = protos[y] + 2.5 * torch.randn(n, 28 * 28, generator=g)
        return x.to(device), y.to(device)
    return draw(n_train), draw(n_test)


def synthetic_cifar_problem(n_train, n_test, device, seed=0):
    """The CIFAR10 stand-in for Cifar10Net: [n, 3, 32, 32] images of 10 classes, x = 0.5 * proto[y] + 0.5 * noise.
    Each prototype is a random [3, 2, 2] grid upsampled bilinearly to 32x32 and scaled to unit standard deviation: a
    smooth colour gradient, so the class shows in every 3x3 patch of the 23x23 corner the net's pools read.

    main.py's rates (lr 0.1, momentum 0.9) train Cifar10Net unstably on every construction tried (per-pixel and smooth
    prototypes, 2x2 to 8x8 grids, scales 0.25 to 1, noise 0.25 to 2.5): accuracy climbs, collapses and recovers.  This
    one learned best: a CPU run of harness.main (NoDefense, no attacker, 10 users, m = 83, 20,000 training and 4,000
    test rows, tested every 10 epochs) reached 100.0 % (seed 0) and 79.8 % (seed 1) at best and ended at 100.0 % and
    56.9 % at epoch 99.  The learnability bar is therefore a best test accuracy of at least 40 % within 100 epochs."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    protos = F.interpolate(torch.randn(10, 3, 2, 2, generator=g), size=(32, 32), mode='bilinear', align_corners=False)
    protos = 0.5 * protos / protos.std(dim=(1, 2, 3), keepdim=True)

    def draw(n):
        y = torch.randint(0, 10, (n,), generator=g)
        x = protos[y] + 0.5 * torch.randn(n, 3, 32, 32, generator=g)
        return x.to(device), y.to(device)
    return draw(n_train), draw(n_test)


def check_dataset(dataset):
    if dataset not in DATASETS:
        raise ValueError(f"unknown dataset {dataset!r} (expected one of {', '.join(DATASETS)})")
    return dataset


def model(dataset='MNIST'):
    """The network main.py -s selects for the users, the server and the attacker (main.py:144-145, user.py:41-44,
    server.py:24-29, backdoor.py:23-26)."""
    return Cifar10Net() if check_dataset(dataset) == 'CIFAR10' else MnistNet()


def synth_name(dataset='MNIST'):
    return SYNTH_CIFAR10 if check_dataset(dataset) == 'CIFAR10' else SYNTH


def dataset_name(dataset='MNIST', data_dir=None):
    """The dataset's name in logs, checkpoint paths and prints: main.py's ('MNIST', 'CIFAR10') when the data come from
    data_dir, SYNTH-MNIST / SYNTH-CIFAR10 for the synthetic stand-ins."""
    return check_dataset(dataset) if data_dir is not None else synth_name(dataset)


def real_sizes(dataset, data_dir, train_size=None, test_size=None):
    """data.load(dataset, data_dir) and its (train, test) row counts; an explicit size that differs raises ValueError."""
    (xtr, ytr), (xte, yte) = loaded = _data.load(check_dataset(dataset), data_dir)
    for what, want, got in (('train_size', train_size, len(xtr)), ('test_size', test_size, len(xte))):
        if want is not None and want != got:
            raise ValueError(f"{what}={want}, but the {dataset} files under {data_dir} hold {got} rows")
    return loaded


def experiment_setup(seed, train_size, test_size, device, dataset='MNIST', data_dir=None):
    """The seeded start of an experiment: torch.manual_seed(seed), the synthetic train and test sets and the test
    network, whose parameters are the initial global weights.  ((xtr, ytr), (xte, yte), test_net).  dataset='CIFAR10':
    synthetic_cifar_problem's [n, 3, 32, 32] images and a Cifar10Net.  With data_dir the sets are data.load's, in
    file order (train_size and test_size: None, or the files' row counts), and the test net is the same seed's."""
    if data_dir is not None:
        (xtr, ytr), (xte, yte) = real_sizes(dataset, data_dir, train_size, test_size)
        torch.manual_seed(seed)
        return (xtr.to(device), ytr.to(device)), (xte.to(device), yte.to(device)), model(dataset).to(device)
    problem = synthetic_cifar_problem if check_dataset(dataset) == 'CIFAR10' else synthetic_problem
    torch.manual_seed(seed)
    train, test = problem(20000 if train_size is None else train_size, 4000 if test_size is None else test_size,
                          device, seed)
    return train, test, model(dataset).to(device)


def csv_name(num_std, defense, backdoor, mal_prop, users_count, alpha, learning_rate, dataset='MNIST', data_dir=None):
    """main.py:100's accuracy log name (without the logs/ directory)."""
    return '{}_stdev_{}_{}_backdoor-{}_mal_prop_{}_users_{}_alpha_{}_lr_{}.csv'.format(
        dataset_name(dataset, data_dir), num_std, defense, backdoor, mal_prop, users_count, alpha if backdoor else None,
        learning_rate)


class Client:
    """user.py:33-92 without the data loader machinery: one minibatch forward/backward per round, flat gradient out."""

    def __init__(self, user_id, is_malicious, x, y, batch_size, layout, device, dataset='MNIST'):
        self.user_id, self.is_malicious = user_id, is_malicious
        self.x, self.y, self.batch_size, self.pos = x, y, batch_size, 0
        self.net = model(dataset).to(device)
        self.layout = layout
        self.criterion = nn.NLLLoss()
        self.grads = None
        self.original_params = None
        self.learning_rate = None

    def step(self, current_params, learning_rate, out_row):
        if self.user_id == 0 and self.is_malicious:                       # user.py:84-86
            self.original_params = current_params.clone()
            self.learning_rate = learning_rate
        params = list(self.net.parameters())
        self.layout.row_into_parameters(current_params, params)           # user.py:87
        lo = self.pos
        hi = min(lo + self.batch_size, len(self.x))
        self.pos = 0 if hi == len(self.x) else hi                         # cycle(train_loader)
        self.net.zero_grad(set_to_none=True)
        loss = self.criterion(self.net(self.x[lo:hi]), self.y[lo:hi])
        loss.backward()                                                   # no optimiser step: the server steps (user.py:81)
        self.layout.flatten([p.grad for p in params], out=out_row)        # user.py:92, written into the matrix row
        self.grads = out_row


def backdoor_set(backdoor, x, y, seed=0, batch_size=200, sampled=False):
    """BackdoorTrainer's backdoor data (x, y) from the training set (x, y).  backdoor='pattern' (backdoor.py:37-42,
    47-50): rows r::u with u = max(len(x) // batch_size // 10, 1) and r = default_rng(seed).integers(u), the 5x5 corner
    of the 28x28 view (of every channel of a [3, 32, 32] image) set to 2.8, every label 0; backdoor = 1, 2 or 3
    (backdoor.py:30-35): training row backdoor - 1, labelled (y + 1) % 5.  sampled=True takes the rows the reference's
    DistributedSampler loader yields instead (data.backdoor_indices), with the same pattern and labels."""
    if sampled:
        i = _data.backdoor_indices(backdoor, len(x), seed, batch_size).to(x.device)
    elif backdoor == 'pattern':
        u = max(len(x) // batch_size // 10, 1)
        i = slice(int(np.random.default_rng(seed).integers(u)), None, u)
    else:
        i = slice(int(backdoor) - 1, int(backdoor))
    if backdoor != 'pattern':
        return x[i], (y[i] + 1) % 5
    x = x[i].clone()
    if x.dim() == 4:                                                      # add_pattern on a CHW image
        x[:, :, :5, :5] = 2.8
    else:
        x.view(-1, 28, 28)[:, :5, :5] = 2.8
    return x, torch.zeros_like(y[:len(x)])


class BackdoorTrainer:
    """backdoor.py:13-159 on the synthetic problem: the attacker's own network, trained from the starting point the
    crafting hands it towards the backdoor, and tested on the backdoor data.  backdoor='pattern': a shard of the
    training set with x[:, :5, :5] = 2.8 on the 28x28 view, all labelled 0; backdoor = 1, 2 or 3: the single training
    sample backdoor - 1, labelled (y + 1) % 5.  dataset='CIFAR10' trains a Cifar10Net, with the pattern on every channel.
    sampled=True: the rows of backdoor.py's DistributedSampler loader (backdoor_set)."""

    def __init__(self, backdoor, alpha, num_epochs, layout, x, y, device, my_print, seed=0, batch_size=200,
                 dataset='MNIST', sampled=False):
        self.backdoor, self.alpha, self.num_epochs, self.layout, self.my_print = backdoor, alpha, num_epochs, layout, my_print
        self.batch_size = batch_size
        self.net = model(dataset).to(device)
        self.x, self.y = backdoor_set(backdoor, x, y, seed, batch_size, sampled)

    def test(self, tag, to_print=True):                                   # backdoor.py:67-102
        loss, correct = 0.0, 0
        with torch.no_grad():
            for lo in range(0, len(self.x), self.batch_size):
                out = self.net(self.x[lo:lo + self.batch_size])
                loss += F.nll_loss(out, self.y[lo:lo + self.batch_size]).item()
                correct += int(out.max(1)[1].eq(self.y[lo:lo + self.batch_size]).sum())
        accuracy = 100. * correct / len(self.x)
        if to_print:
            self.my_print('##Test malicious net: [{}] Average loss: {:.4f}, Accuracy: {}/{} ({:.2f}%)'.format(
                tag, loss / len(self.x), correct, len(self.x), accuracy))
        return accuracy

    def train(self, initial):                                             # backdoor.py:108-159
        params = list(self.net.parameters())
        self.layout.row_into_parameters(initial, params)
        p0 = [p.detach().clone() for p in params]
        if self.test('BEFORE', to_print=False) >= 100.:
            return initial
        self.net.train()
        for _ in range(self.num_epochs):
            for lo in range(0, len(self.x), self.batch_size):
                opt = torch.optim.SGD(params, lr=0.1, momentum=0.9, weight_decay=0.0001)   # a new one every minibatch
                opt.zero_grad()
                loss = F.nll_loss(self.net(self.x[lo:lo + self.batch_size]), self.y[lo:lo + self.batch_size])
                if self.alpha > 0:
                    loss = loss + self.alpha * sum(F.mse_loss(p, q) for p, q in zip(params, p0))
                loss.backward()
                opt.step()
        self.test(self.num_epochs - 1)
        return self.layout.flatten(params)


def main(mal_prop, num_std, defense, users_count=10, epochs=150, learning_rate=0.1, fading_rate=10000, momentum=0.9,
         batch_size=83, output=None, device="cuda", out_dir=".", seed=0, train_size=None, test_size=None, test_step=5,
         backdoor=False, alpha=4, mal_epochs=5, dataset='MNIST', data_dir=None, trace=False):
    """main.py's experiment.  train_size and test_size (None: 20,000 and 4,000) size the synthetic problem; with
    data_dir the data are the real dataset's files there (see the module docstring) and the sizes, when given, must
    be the files' row counts.  Returns (accuracies, accuracies_epochs, csv).

    trace=True also records every epoch's attack figures after `defend` (sweep.run(trace=True)'s, from the existing
    calls): batched.attack_metrics on the [1, N, D] matrix against the applied aggregate and against row 0, Krum's
    index from a second `krum(..., return_index=True)` and Bulyan's selection from a second `bulyan(...,
    return_selection=True)`.  So a traced Krum or Bulyan epoch runs its rule twice and each traced epoch synchronises
    the host.  It writes the trace CSV beside the accuracy CSV (`..._trace.csv`, metrics.TRACE_HEADER) and returns the
    trace (metrics.trace_record's dict) as a fourth element."""
    synth = dataset_name(dataset, data_dir)
    if output:
        def my_print(s, end='\n'):
            with open(output, 'a+') as f:
                f.write(str(s) + end)
    else:
        my_print = print
    my_print(dict(mal_prop=mal_prop, num_std=num_std, defense=defense, users_count=users_count, epochs=epochs,
                  learning_rate=learning_rate, dataset=synth, backdoor=backdoor))
    corrupted_count = int(mal_prop * users_count)                         # main.py:21
    (xtr, ytr), (xte, yte), test_net = experiment_setup(seed, train_size, test_size, device, dataset, data_dir)
    layout = ParamLayout(test_net.parameters())
    srv = AggregationServer(users_count, layout.dim, mal_prop, learning_rate, momentum, device=device,
                            initial_weights=layout.flatten(list(test_net.parameters())))
    xs, ys = xtr, ytr
    if data_dir is not None:                                              # DistributedSampler's padded order (user.py:50)
        order = _data.sampler_order(len(xtr), users_count).to(xtr.device)
        xs, ys = xtr[order], ytr[order]
    users = [Client(u, u < corrupted_count, xs[u::users_count], ys[u::users_count], batch_size, layout, device,
                    dataset) for u in range(users_count)]                                 # DistributedSampler-style partition (user.py:50)
    if backdoor:                                                          # main.py:44-54
        trainer = BackdoorTrainer(backdoor, alpha, mal_epochs, layout, xtr, ytr, device, my_print, seed, dataset=dataset,
                                  sampled=data_dir is not None)
        attacker = malicious.BackdoorAttack(num_std, trainer.train)
    else:
        attacker = malicious.DriftAttack(num_std)
    my_print("\nStarting Training...")
    criterion = nn.NLLLoss()
    accuracies, accuracies_epochs = [], []
    figures = {k: [] for k in ('agg_deviation', 'malicious_deviation', 'krum_index', 'bulyan_malicious',
                               'bulyan_selected')}
    for epoch in range(epochs):
        lr_t = learning_rate * fading_rate / (epoch + fading_rate)       # server.py:50-52
        for u in users:                                                   # server.py:54-56 dispatch_weights
            u.step(srv.current_weights, lr_t, srv.users_grads[u.user_id])
        if backdoor:                                                      # main.py:66-68 + server.py:82-83, in place
            attacker.attack_rows(srv.users_grads, corrupted_count, users[0].original_params, users[0].learning_rate)
        else:
            attacker.attack_rows(srv.users_grads, corrupted_count)
        aggregate = srv.defend(defense, epoch)                            # main.py:71
        if trace:
            attack_figures(srv.users_grads, users_count, corrupted_count, defense, aggregate, figures)
        if epoch % test_step == 0 or epoch == epochs - 1:
            layout.row_into_parameters(srv.current_weights, list(test_net.parameters()))
            test_net.eval()
            test_loss, correct = 0.0, 0
            with torch.no_grad():
                for lo in range(0, len(xte), batch_size):                 # server.py:100-110
                    out = test_net(xte[lo:lo + batch_size])
                    test_loss += criterion(out, yte[lo:lo + batch_size]).item()
                    correct += int(out.max(1)[1].eq(yte[lo:lo + batch_size]).sum())
            test_loss /= len(xte)
            accuracy = 100. * float(correct) / len(xte)
            my_print('Test set: [{:3d}] Average loss: {:.4f}, Accuracy: {}/{} ({:.2f}%)'.format(epoch, test_loss, correct,
                                                                                             len(xte), accuracy))
            accuracies.append(accuracy)
            accuracies_epochs.append(epoch)
            if accuracy > 70.:                                            # main.py:84-89, server.py:40-46
                directory = os.path.join(out_dir, "runs", synth)
                os.makedirs(directory, exist_ok=True)
                torch.save({'epoch': epoch + 1, 'state_dict': test_net.state_dict(), 'acc': accuracy},
                           os.path.join(directory, 'checkpoint.pth.tar'))
            if backdoor:                                                  # main.py:91-95: the backdoor in the global model
                layout.row_into_parameters(srv.current_weights, list(trainer.net.parameters()))
                trainer.test('POST')
    my_print(datetime.datetime.now().time())
    my_print("Max accuracy: {}".format(max(accuracies)))
    os.makedirs(os.path.join(out_dir, "logs"), exist_ok=True)             # the reference needs a pre-made logs/ (readme.md:25)
    csv = os.path.join(out_dir, 'logs', csv_name(num_std, defense, backdoor, mal_prop, users_count, alpha, learning_rate,
                                                 dataset, data_dir))
    np.savetxt(csv, accuracies, delimiter=',')                            # main.py:100
    if not trace:
        return accuracies, accuracies_epochs, csv
    tr = metrics.trace_record(defense, corrupted_count, *figures.values())
    metrics.write_trace_csv(csv[:-len('.csv')] + '_trace.csv', tr)
    return accuracies, accuracies_epochs, csv, tr


def attack_figures(G, users_count, corrupted_count, defense, aggregate, figures):
    """One epoch's trace figures of main's server matrix G ([N, D]) and the aggregate `defend` applied, appended to
    figures' lists (metrics.trace_record's arguments)."""
    f, G3 = corrupted_count, G[None]
    sel = None
    if defense == 'Krum':
        figures['krum_index'].append(defences.krum(G, users_count, f, return_index=True))
    elif defense == 'Bulyan':
        sel = defences.bulyan(G, users_count, f, return_selection=True)[1].to(torch.int32)
        s = sel.cpu().numpy()
        figures['bulyan_malicious'].append(int(((s >= 0) & (s < f)).sum()))
        figures['bulyan_selected'].append(int((s >= 0).sum()))
    met = batched.attack_metrics(G3, f, aggregated=aggregate.float()[None], selection=None if sel is None else sel[None])
    figures['agg_deviation'].append(float(met['rel_deviation'][0]))
    mal = float('nan')
    if f > 0:
        row0 = torch.zeros(1, dtype=torch.int32, device=G.device)
        mal = float(batched.attack_metrics(G3, f, krum_index=row0)['rel_deviation'][0])
    figures['malicious_deviation'].append(mal)


def parser():
    """main.py's command line (the flags that apply here), plus --trace."""
    p = argparse.ArgumentParser()                                         # main.py:104-131 (the flags that apply here)
    p.add_argument('-m', '--mal-prop', default=0.24, type=float)
    p.add_argument('-z', '--num_std', default=1.5, type=float)
    p.add_argument('-d', '--defense', default='NoDefense', choices=['NoDefense', 'Bulyan', 'TrimmedMean', 'Krum'])
    p.add_argument('-n', '--users-count', default=10, type=int)
    p.add_argument('-c', '--batch_size', default=128, type=int)
    p.add_argument('-e', '--epochs', default=300, type=int)
    p.add_argument('-l', '--learning_rate', default=0.1, type=float)
    p.add_argument('-o', '--output', type=str)
    p.add_argument('-b', '--backdoor', default='No', choices=['No', 'pattern', '1', '2', '3'])
    p.add_argument('-s', '--dataset', default='MNIST', choices=list(DATASETS))
    p.add_argument('--data-dir', default=None, help="the directory holding torchvision's MNIST or CIFAR10 files "
                   "(the reference's ./mnist_data or ./cifar10_data); without it a synthetic stand-in is trained")
    p.add_argument('--trace', action='store_true', help="record every epoch's attack figures into a _trace.csv beside "
                   "the accuracy log (runs Krum and Bulyan twice per epoch)")
    return p


if __name__ == '__main__':
    a = parser().parse_args()
    bd = False if a.backdoor == 'No' else a.backdoor if a.backdoor == 'pattern' else int(a.backdoor)
    main(a.mal_prop, a.num_std, a.defense, users_count=a.users_count, epochs=a.epochs, learning_rate=a.learning_rate,
         batch_size=a.batch_size, output=a.output, backdoor=bd, dataset=a.dataset, data_dir=a.data_dir,
         fading_rate=2000 if a.dataset == 'CIFAR10' else 10000, trace=a.trace)   # main.py:144-147

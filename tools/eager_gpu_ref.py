"""Context number (SURVEY 8d): the reference learner iteration in PyTorch EAGER mode on one H100 - the only
pre-existing GPU implementation of this path (oracle/ref_port.py with its modules and batch moved to cuda).
Not part of bench.py's contract; prints one JSON line."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT]
import torch
from oracle import ref_port

if __name__ == "__main__":
    # PortLearner.iteration converts to numpy for the priorities (like the reference's .cpu()); reuse it as is:
    c = dict(obs=17, act=6, hidden=256, batch=256, burn_in=40, learning=80, n_step=5)
    pc = ref_port.PathConfig(**c)
    dev = torch.device("cuda:0")
    torch.set_default_device(dev)                    # modules, zero states and optim state are created on the GPU
    lr = ref_port.PortLearner(pc, seed=1)
    torch.set_default_device("cpu")
    for name in ("actor", "target_actor", "critic", "target_critic"):   # parameters built from numpy land on the CPU
        getattr(lr, name).to(dev)
    def _advance(self, x):
        z = torch.tanh(self.l1(x))
        if self.hx is None:
            self.hx = torch.zeros((z.size(0), self.hidden), device=z.device)
            self.cx = torch.zeros((z.size(0), self.hidden), device=z.device)
        self.hx, self.cx = self.l2(z, (self.hx, self.cx))
        return self.hx
    ref_port._RecurrentNet._advance = _advance
    batch_np = ref_port.synthetic_batch(pc, 0)
    # the reference moves the batch with .cuda() inside sample() and reads TD back with .cpu(): same here
    import numpy as np
    real_as_tensor = torch.as_tensor
    torch.as_tensor = lambda v, *a, **k: real_as_tensor(v, *a, **k).to(dev) if isinstance(v, np.ndarray) else real_as_tensor(v, *a, **k)
    _numpy = torch.Tensor.numpy
    torch.Tensor.numpy = lambda self, *a, **k: _numpy(self.cpu(), *a, **k)
    times = []
    for i in range(6):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        lr.iteration(batch_np, keep_tensors=False)
        torch.cuda.synchronize(); times.append(time.perf_counter() - t0)
    sec = sorted(times[2:])[len(times[2:]) // 2]
    print(json.dumps({"impl": "reference port, PyTorch eager on 1x H100 (fp32, TF32 off)", "config": c,
                      "sec_per_iteration": sec, "seq_steps_per_s": c["batch"] * c["learning"] / sec, "all": [round(t, 4) for t in times]}))

"""RMSprop of the reference trainer (``optim.RMSprop(policy_net.parameters(), lr=args.lrate, alpha=0.97,
eps=1e-6)``, trainer.py:21-22) as ONE kernel over flat buffers (csrc/optim.cu, ``ic3_rmsprop_step``).

The parameters of the policy are re-pointed to views of one contiguous fp32 buffer, their ``.grad`` to views of
a second one and the second-moment state to views of a third, so that

* ``zero_grad()`` is one memset,
* the data-parallel reduction all-reduces the flat gradient buffer in place (no gather / scatter copies,
  multi_processing.py:90-95),
* ``step(grad_div)`` -- gradient / global num_steps (trainer.py:251-253) and the update (trainer.py:254) -- is one
  launch.

``state_dict()`` / ``load_state_dict()`` speak ``torch.optim.RMSprop``'s format (``state[i] = {'step',
'square_avg'}``, one param group), so trainer checkpoints interchange with the reference
(trainer.py:258-262, main.py:260-272).  Parameters that never receive a gradient (``hidd_encoder``, which the
reference forward does not use) keep a zero gradient here: their update is exactly zero, as if skipped.
"""
import torch

from . import _lib


class FlatRMSprop(object):
    def __init__(self, params, lr, alpha=0.97, eps=1e-6):
        self.params = [p for p in params]
        if not self.params:
            raise ValueError("optimizer got an empty parameter list")
        dev = self.params[0].device
        for p in self.params:
            if not (p.is_cuda and p.dtype == torch.float32 and p.device == dev):
                raise RuntimeError("FlatRMSprop needs float32 CUDA parameters on one device (no CPU fallback)")
        _lib.require_cuda()
        self.lr, self.alpha, self.eps = float(lr), float(alpha), float(eps)
        self.steps = 0
        # every tensor starts on a 16-byte boundary (float4 kernel; also keeps views aligned for other kernels)
        self._off, n = [], 0
        for p in self.params:
            self._off.append(n)
            n += (p.numel() + 3) // 4 * 4
        self.numel = n
        self.flat_params = torch.zeros(n, device=dev)
        self.flat_grads = torch.zeros(n, device=dev)
        self.flat_square_avg = torch.zeros(n, device=dev)
        with torch.no_grad():
            for p, off in zip(self.params, self._off):
                view = self.flat_params[off:off + p.numel()].view_as(p)
                view.copy_(p.data)
                p.data = view                                   # the module now computes on the flat buffer
                p.grad = self.flat_grads[off:off + p.numel()].view_as(p)

    def _views(self, flat):
        return [flat[off:off + p.numel()].view_as(p) for p, off in zip(self.params, self._off)]

    # ---- torch.optim.Optimizer surface used by the trainer ------------------------------------------
    def zero_grad(self, set_to_none=False):
        if set_to_none:
            raise ValueError("FlatRMSprop keeps the gradients in one persistent buffer (set_to_none=False)")
        self.flat_grads.zero_()
        for p, g in zip(self.params, self._views(self.flat_grads)):
            if p.grad is None or p.grad.data_ptr() != g.data_ptr():
                p.grad = g                                      # someone dropped / replaced .grad: re-attach

    def _fold_grads(self):
        """Bring every parameter's gradient into the flat buffer the update kernels read."""
        self._check_attached()
        for p, g in zip(self.params, self._views(self.flat_grads)):
            if p.grad is None:
                raise RuntimeError("a parameter lost its flat gradient view; call zero_grad() before backward")
            if p.grad.data_ptr() != g.data_ptr():               # autograd replaced the tensor: fold it back in
                g.copy_(p.grad)
                p.grad = g

    def step(self, grad_div=1.0):
        """One update with ``grad / grad_div`` (the trainer passes the global number of env steps)."""
        self._fold_grads()
        _lib.check(_lib.load().ic3_rmsprop_step(self.numel, self.lr, self.alpha, self.eps, float(grad_div),
                                                self.flat_grads.data_ptr(), self.flat_params.data_ptr(),
                                                self.flat_square_avg.data_ptr(), _lib.stream()))
        self.mark_params_changed()
        self.steps += 1

    def step_dev(self, stat, err):
        """Enqueue the update of step() with grad_div = stat[1], the step count of the device float64 statistics vector
        stat (ic3_rmsprop_step_dev; nothing happens when stat[3] holds error flags, IC3_ERR_GRAD_DIV goes to the int32
        device word err when the count is not positive).  No host read, so a CUDA graph can hold it; the caller advances
        ``steps`` and calls mark_params_changed() once the update has run."""
        self._fold_grads()
        _lib.check(_lib.load().ic3_rmsprop_step_dev(self.numel, self.lr, self.alpha, self.eps, stat.data_ptr(),
                                                    self.flat_grads.data_ptr(), self.flat_params.data_ptr(),
                                                    self.flat_square_avg.data_ptr(), err.data_ptr(), _lib.stream()))

    def mark_params_changed(self):
        """The flat parameter buffer was written through raw pointers / collectives: bump the version counters so
        that caches keyed on (data_ptr, _version) -- CommNetMLP.packed() -- see the new weights."""
        bump = getattr(torch._C, "_increment_version", None)
        if bump is not None:
            bump(self.params)
        else:
            with torch.no_grad():
                for p in self.params:
                    p.add_(0)

    def _check_attached(self):
        """A second FlatRMSprop built on the same parameters re-points them to ITS buffers (the reference builds
        several Trainers on one policy_net, main.py:181-186): updating an orphaned buffer would be a silent no-op."""
        for p, v in zip(self.params, self._views(self.flat_params)):
            if p.data_ptr() != v.data_ptr():
                raise RuntimeError("a parameter no longer lives in this optimizer's flat buffer (another FlatRMSprop "
                                   "was built on the same policy_net); use ONE optimizer per policy_net")

    def state_dict(self):
        state = {}
        if self.steps > 0:
            for i, v in enumerate(self._views(self.flat_square_avg)):
                state[i] = {'step': torch.tensor(float(self.steps)), 'square_avg': v.clone()}
        group = dict(lr=self.lr, momentum=0, alpha=self.alpha, eps=self.eps, centered=False, weight_decay=0,
                     capturable=False, foreach=None, maximize=False, differentiable=False,
                     params=list(range(len(self.params))))
        return {'state': state, 'param_groups': [group]}

    def load_state_dict(self, sd):
        groups = sd['param_groups']
        if len(groups) != 1 or len(groups[0]['params']) != len(self.params):
            raise ValueError("optimizer state does not match the parameter list")
        g = groups[0]
        if g.get('momentum', 0) or g.get('centered', False) or g.get('weight_decay', 0):
            raise NotImplementedError("only the reference's plain RMSprop is implemented")
        self.lr, self.alpha, self.eps = float(g['lr']), float(g['alpha']), float(g['eps'])
        self.flat_square_avg.zero_()
        steps = 0
        views = self._views(self.flat_square_avg)
        for k, st in sd['state'].items():
            i = g['params'].index(k) if k in g['params'] else int(k)
            views[i].copy_(st['square_avg'].to(views[i].device, torch.float32))
            steps = max(steps, int(float(st.get('step', 0))))
        self.steps = steps

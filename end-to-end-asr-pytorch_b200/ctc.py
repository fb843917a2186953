"""CTC prefix scoring for joint CTC / attention beam search with the reference's interface
(/root/reference/src/ctc.py:12-116) on the GPU: `CTCPrefixScore(x).init_state()` / `.cheap_compute(g, r_prev, cands)`
return what the reference's numpy scorer returns, and `.cheap_compute_batch` scores every hypothesis of a beam-search
step in ONE kernel launch (the reference loops over hypotheses on the host, src/decode.py:103-131)."""
import numpy as np
import torch

from . import lib as L


class CTCPrefixScore:
    def __init__(self, x):
        """x: [1, T, V] CTC log-probs (CUDA tensor)."""
        self.logzero = -100000000.0
        self.blank = 0
        self.eos = 1
        if not x.is_cuda:
            raise L.B200AsrError("CTCPrefixScore needs a CUDA tensor; there is no CPU fallback")
        self.x = x[0].detach().to(torch.float32).contiguous()
        self.odim = x.shape[-1]
        self.input_length = self.x.shape[0]

    def init_state(self):
        """r[t] = (logzero, cumulative blank log-prob), src/ctc.py:27-35; device tensor [T, 2]."""
        r = torch.full((self.input_length, 2), self.logzero, device=self.x.device, dtype=torch.float32)
        r[:, 1] = torch.cumsum(self.x[:, self.blank].double(), 0).float()
        return r

    def cheap_compute_batch(self, prefixes, r_prevs, candidates):
        """prefixes: list of N token lists; r_prevs: [N, T, 2] device tensor (or list of [T,2]); candidates: [N, C]
        host int tensor / nested list.  Returns (psi [N, C], r [N, C, T, 2]) device tensors.  Token ids outside
        [0, V) raise ValueError before the launch (the kernel gathers log-probs at the candidate ids)."""
        lib = L.load()
        dev = self.x.device
        V = self.odim
        cand = torch.as_tensor(candidates, dtype=torch.int32).cpu()
        if cand.numel() and (int(cand.min()) < 0 or int(cand.max()) >= V):
            raise ValueError("CTCPrefixScore: candidate ids must lie in [0, %d)" % V)
        if any(not 0 <= int(tok) < V for g in prefixes for tok in g):
            raise ValueError("CTCPrefixScore: prefix tokens must lie in [0, %d)" % V)
        if not torch.is_tensor(r_prevs):
            r_prevs = torch.stack([torch.as_tensor(r, dtype=torch.float32).to(dev) for r in r_prevs])
        r_prevs = r_prevs.to(device=dev, dtype=torch.float32).contiguous()
        cand = cand.to(dev).contiguous()
        N, C = cand.shape
        T = self.input_length
        assert r_prevs.shape == (N, T, 2)
        last = torch.tensor([g[-1] if len(g) > 0 else 0 for g in prefixes], dtype=torch.int32, device=dev)
        plen = torch.tensor([len(g) for g in prefixes], dtype=torch.int32, device=dev)
        psi = torch.empty((N, C), device=dev, dtype=torch.float32)
        r = torch.empty((N, C, T, 2), device=dev, dtype=torch.float32)
        L.check(lib.b200asr_ctc_prefix_score(L.ptr(self.x), T, self.odim, L.ptr(r_prevs), L.ptr(last), L.ptr(plen),
                                             L.ptr(cand), N, C, self.blank, self.eos, L.ptr(psi), L.ptr(r), L.stream()),
                "ctc_prefix_score")
        return psi, r

    def cheap_compute(self, g, r_prev, candidates, as_numpy=True):
        """Same contract as src/ctc.py:81-116: (psi [C], r [C, T, 2]); numpy arrays by default like the reference."""
        rp = torch.as_tensor(r_prev, dtype=torch.float32)
        psi, r = self.cheap_compute_batch([list(g)], rp.reshape(1, self.input_length, 2), [list(candidates)])
        if as_numpy:
            return psi[0].cpu().numpy(), r[0].cpu().numpy()
        return psi[0], r[0]

"""Nested CSR containers with the reference's interface (torch_points3d/core/multimodal/csr.py).

`CSRData(pointers, *values)` stores a list of variable-length groups as one value tensor per
field plus int64 pointers (pointers[0] == 0).  Values may be tensors or CSRData (nesting).  All
bookkeeping is integer work; on CUDA tensors the two re-indexing primitives run as single-pass
kernels of libdva_b200.so (dva_csr_pointers_from_sorted, dva_csr_select_values) instead of the
reference's cat / where / cumsum / repeat_interleave chains (csr.py:158-264).
"""
import copy

import torch

from ... import _lib
from ...utils.multimodal import tensor_idx


def pointers_from_sorted(ids, num_groups):
    """Pointers [num_groups+1] of sorted dense group ids, zero-length groups included
    (= _sorted_indices_to_pointers + insert_empty_groups, csr.py:158-172, 197-229)."""
    ids = ids.long().contiguous()
    n = ids.numel()
    if ids.is_cuda:
        ptr = torch.empty(num_groups + 1, dtype=torch.long, device=ids.device)
        _lib.launch("dva_csr_pointers_from_sorted", ids.device, ids, ptr, n, num_groups)
        return ptr
    return torch.searchsorted(ids, torch.arange(num_groups + 1, dtype=torch.long))


def select_values(pointers, sel):
    """(pointers_new, val_idx) of the group selection `sel` (csr.py:235-264)."""
    sizes = pointers[sel + 1] - pointers[sel]
    pn = torch.cat([torch.zeros(1, dtype=torch.long, device=pointers.device), torch.cumsum(sizes, 0)])
    n_new = int(pn[-1].item())
    if pointers.is_cuda:
        val = torch.empty(n_new, dtype=torch.long, device=pointers.device)
        _lib.launch("dva_csr_select_values", pointers.device, pointers.contiguous(), sel.contiguous(), pn, val,
                    sel.numel(), n_new)
        return pn, val
    val = torch.arange(n_new) - pn[:-1].repeat_interleave(sizes) + pointers[sel].repeat_interleave(sizes)
    return pn, val


class CSRData(object):
    """csr.py:44-303."""

    def __init__(self, pointers, *args, dense=False, is_index_value=None):
        self.pointers = CSRData._sorted_indices_to_pointers(pointers) if dense else pointers
        self.values = [*args] if len(args) > 0 else None
        if is_index_value is None or len(is_index_value) == 0:
            self.is_index_value = torch.zeros(self.num_values, dtype=torch.bool)
        else:
            self.is_index_value = torch.as_tensor(is_index_value, dtype=torch.bool)

    def debug(self):
        assert self.pointers[0] == 0, "The first pointer element must always be 0."
        assert torch.all(self.pointers[1:] - self.pointers[:-1] >= 0), "pointer indices must be increasing."
        if self.values is not None:
            assert all(len(v) == self.num_items for v in self.values), \
                "All value objects must have the same size."
            for v in self.values:
                if isinstance(v, CSRData):
                    v.debug()

    def to(self, device):
        out = self.clone()
        out.pointers = out.pointers.to(device)
        for i in range(out.num_values):
            out.values[i] = out.values[i].to(device)
        return out

    def cpu(self):
        return self.to('cpu')

    def cuda(self):
        return self.to('cuda')

    @property
    def device(self):
        return self.pointers.device

    @property
    def num_groups(self):
        return self.pointers.shape[0] - 1

    @property
    def num_values(self):
        return len(self.values) if self.values is not None else 0

    @property
    def num_items(self):
        # the value tensors know their length on the host: no device read (csr.py:113 reads pointers[-1])
        if self.values:
            v = self.values[0]
            return int(v.num_groups) if isinstance(v, CSRData) else int(v.shape[0])
        return int(self.pointers[-1].item())

    @staticmethod
    def get_batch_type():
        return CSRBatch

    def clone(self):
        """Shallow copy (csr.py:147-156)."""
        out = copy.copy(self)
        out.pointers = copy.copy(self.pointers)
        out.values = copy.copy(self.values)
        return out

    @staticmethod
    def _sorted_indices_to_pointers(indices):
        """Pointers over the DISTINCT consecutive ids of a sorted tensor (csr.py:158-172)."""
        assert indices.dim() == 1 and indices.shape[0] >= 1, "At least one group index is required."
        change = torch.ones(indices.shape[0] + 1, dtype=torch.bool, device=indices.device)
        change[1:-1] = indices[1:] > indices[:-1]
        return torch.nonzero(change).view(-1)

    def reindex_groups(self, group_indices, num_groups=None):
        order = torch.argsort(group_indices)
        return self[order].insert_empty_groups(group_indices[order], num_groups=num_groups)

    def insert_empty_groups(self, group_indices, num_groups=None):
        """Existing group i moves to position group_indices[i] (sorted); missing positions become
        zero-length groups.  Mutates and returns self like the reference (csr.py:197-229)."""
        assert self.num_groups == group_indices.shape[0], \
            "New group indices must correspond to the existing number of groups"
        gi = group_indices.to(self.device).long()
        last = int(gi[-1].item()) + 1 if gi.numel() else 0
        num_groups = last if num_groups is None else max(last, int(num_groups))
        # new_ptr[g] = pointers[#groups with index < g]
        rank = torch.searchsorted(gi, torch.arange(num_groups + 1, device=self.device))
        self.pointers = self.pointers[rank]
        return self

    @staticmethod
    def _index_select_pointers(pointers, indices):
        return select_values(pointers, indices)

    def __getitem__(self, idx):
        idx = tensor_idx(idx).to(self.device)
        out = self.clone()
        if idx.shape[0] == 0:
            out.pointers = torch.zeros(1, dtype=torch.long, device=self.device)
            out.values = [v[[]] for v in self.values]
        else:
            out.pointers, val_idx = select_values(self.pointers, idx)
            out.values = [v[val_idx] for v in self.values]
        return out

    def __len__(self):
        return self.num_groups

    def __repr__(self):
        info = [f"{k}={getattr(self, k)}" for k in ['num_groups', 'num_items', 'device']]
        return f"{self.__class__.__name__}({', '.join(info)})"


class CSRBatch(CSRData):
    """Batch of CSRData with reversible stacking (csr.py:305-479)."""
    __csr_type__ = CSRData

    def __init__(self, pointers, *args, dense=False, is_index_value=None):
        super().__init__(pointers, *args, dense=dense, is_index_value=is_index_value)
        self.__sizes__ = None

    @property
    def batch_pointers(self):
        if self.__sizes__ is None:
            return None
        return torch.cumsum(torch.cat((torch.zeros(1, dtype=torch.long), self.__sizes__.cpu())), dim=0)

    @property
    def batch_items_sizes(self):
        return self.__sizes__

    @property
    def num_batch_items(self):
        return len(self.__sizes__) if self.__sizes__ is not None else 0

    def to(self, device):
        out = super().to(device)
        out.__sizes__ = self.__sizes__.to(device) if self.__sizes__ is not None else None
        return out

    @staticmethod
    def from_csr_list(csr_list):
        """csr.py:347-416: pointers shifted by the running item count, "index" values shifted by
        the running max+1 of the previous items."""
        assert isinstance(csr_list, list) and len(csr_list) > 0
        csr_type = type(csr_list[0])
        assert all(isinstance(c, csr_type) for c in csr_list), "All provided items must have the same class."
        device = csr_list[0].device
        num_values = csr_list[0].num_values
        is_index_value = csr_list[0].is_index_value
        item_counts = [c.num_items for c in csr_list]
        offsets = [0]
        for c in item_counts[:-1]:
            offsets.append(offsets[-1] + c)
        pointers = torch.cat([torch.zeros(1, dtype=torch.long, device=device)] +
                             [c.pointers[1:] + o for c, o in zip(csr_list, offsets)])
        values = []
        for i in range(num_values):
            vals = [c.values[i] for c in csr_list]
            if isinstance(vals[0], CSRData):
                val = CSRBatch.from_csr_list(vals)
            elif bool(is_index_value[i]):
                # running max + 1 of the previous items (csr.py:391-402), kept on the device: no .item()
                zero = torch.zeros((), dtype=vals[0].dtype, device=device)
                tops = torch.stack([(v.max() + 1) if v.shape[0] > 0 else zero for v in vals])
                shifts = torch.cumsum(tops, 0) - tops
                val = torch.cat([v + shifts[j] for j, v in enumerate(vals)], dim=0)
            else:
                val = torch.cat(vals, dim=0)
            values.append(val)
        batch = csr_type.get_batch_type()(pointers, *values, dense=False, is_index_value=is_index_value)
        batch.__sizes__ = torch.tensor([c.num_groups for c in csr_list], dtype=torch.long)
        batch.__csr_type__ = csr_type
        return batch

    def to_csr_list(self):
        """csr.py:418-456."""
        if self.__sizes__ is None:
            raise RuntimeError('Cannot reconstruct CSRData data list from batch because the batch '
                               'object was not created using `CSRBatch.from_csr_list()`.')
        gp = self.batch_pointers.to(self.device)
        ip = self.pointers[gp]
        n = self.num_batch_items
        pointers = [self.pointers[gp[i]:gp[i + 1] + 1] - ip[i] for i in range(n)]
        values = []
        for i in range(self.num_values):
            bv = self.values[i]
            if isinstance(bv, CSRData):
                val = bv.to_csr_list()
            elif bool(self.is_index_value[i]):
                val = [bv[ip[j]:ip[j + 1]] - (bv[:ip[j]].max() + 1 if (j > 0 and ip[j] > 0) else 0)
                       for j in range(n)]
            else:
                val = [bv[ip[j]:ip[j + 1]] for j in range(n)]
            values.append(val)
        values = [list(x) for x in zip(*values)]
        return [self.__csr_type__(p, *v, dense=False, is_index_value=self.is_index_value)
                for p, v in zip(pointers, values)]

    def __getitem__(self, idx):
        b = super().__getitem__(idx)
        return self.__csr_type__(b.pointers, *b.values, dense=False, is_index_value=b.is_index_value)

    def __repr__(self):
        info = [f"{k}={getattr(self, k)}" for k in ['num_batch_items', 'num_groups', 'num_items', 'device']]
        return f"{self.__class__.__name__}({', '.join(info)})"

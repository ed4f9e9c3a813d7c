"""ScatterConnection -- drop-in for /root/reference/hpc_rll/torch_utils/network/scatter_connection.py
(class ScatterConnection, ScatterConnectionFunction).

Same constructor ``ScatterConnection(B, M, N, H, W, scatter_type)`` and ``forward(x, location)`` as the reference.
``x`` (B, M, N) fp32 and ``location`` (B, M, 2) int64 ``(y, x)`` give the map (B, N, H, W): a cell holds the row of the
entity with the largest m that lands on it (``'cover'``), the in-order fp32 sum of those rows (``'add'``), or 0.
Differences, all deliberate (DESIGN.md "Deviations"):
  * ``cover`` and ``add`` are deterministic and bit-identical to hpc_rll/origin/scatter_connection.py on the CPU
    (the reference's ``cover`` kernel races when entities share a cell, its ``add`` uses float atomics);
  * an entity whose ``y`` is outside [0, H) or ``x`` outside [0, W) is dropped: it writes nothing and gets a zero
    gradient (the reference and origin write into a neighbouring row or sample);
  * the result is a fresh tensor sized from the inputs, not a module-owned ``output`` buffer -- B, M and N of the
    constructor are kept only for API compatibility, H and W give the map size;
  * kernels run on PyTorch's current stream, with argument checks.
"""
import torch

from ... import _ext


@_ext.reference_function
def ScatterConnectionFunction(input, location, output, grad_in, scatter_type):
    """The reference's argument order.  ``output`` supplies the map size only: either an (H, W) pair or a tensor whose
    last two dimensions are (H, W), such as the reference module's (B, N, H, W) buffer, which is not written.
    ``grad_in`` is accepted and ignored; the result and the gradient are fresh tensors."""
    H, W = (int(s) for s in (output.shape[-2:] if isinstance(output, torch.Tensor) else output))
    return _ext.require().scatter_connection(input, location, H, W, scatter_type)


class ScatterConnection(torch.nn.Module):
    r"""
    Overview:
        Scatter feature to its corresponding location
        In alphastar, each entity is embedded into a tensor, these tensors are scattered into a feature map
        with map size

    Interface:
        __init__, forward
    """

    def __init__(self, B, M, N, H, W, scatter_type) -> None:
        r"""
        Arguments:
            - B (:obj:`int`): batch size
            - M (:obj:`int`): the number of entity
            - N (:obj:`int`): the dimension of entity attributes
            - H (:obj:`int`): height of spatial feature
            - W (:obj:`int`): width of spatial feature
            - scatter_type (:obj:`str`): 'add' or 'cover': what a cell holds when several entities land on it
        """
        super().__init__()
        self.B, self.M, self.N, self.H, self.W = B, M, N, H, W
        self.scatter_type = scatter_type
        assert self.scatter_type in ['cover', 'add']

    def forward(self, x: torch.Tensor, location: torch.Tensor) -> torch.Tensor:
        """
        Arguments:
            - x (:obj:`torch.FloatTensor`): :math:`(B, M, N)`, the entity embeddings
            - location (:obj:`torch.LongTensor`): :math:`(B, M, 2)`, each location is (y, x)
        Returns:
            - output (:obj:`torch.FloatTensor`): :math:`(B, N, H, W)`, the scattered feature map
        """
        assert (x.is_cuda)
        assert (location.is_cuda)
        return ScatterConnectionFunction.apply(x, location, (self.H, self.W), None, self.scatter_type)

"""Sign-bit packing backend (reference ``runtime/compression/cupy.py:CupyBackend``), without cupy: the packing is the
``pack_signs`` / ``unpack_signs`` pair of ``runtime/comm/compressed.py`` (sm_90a kernel on device, torch on host)."""
import torch

from deepspeed_b200.runtime.comm.compressed import pack_signs, unpack_signs


class CupyBackend:

    def torch2cupy(self, tensor):
        return tensor  # no foreign array type: everything stays a torch tensor

    def cupy2torch(self, tensor):
        return tensor

    def compress_by_chunk(self, bool_tensor, num_chunks):
        """Pack a boolean (sign) tensor 8:1 and split the bytes into ``num_chunks`` equal pieces."""
        packed = pack_signs(torch.where(bool_tensor.bool(), 1.0, -1.0).to(torch.float32))
        return list(packed.chunk(num_chunks))

    def decompress(self, packed, dtype=torch.float32):
        return unpack_signs(packed, dtype)

from .ops import bsr_bsc_matmul

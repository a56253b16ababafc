"""nvbio_b200 -- H100-native (sm_90a) implementation of nvbio's two data-parallel hot paths:
FM-index rank/match/locate (nvbio/fmindex) and batched banded Gotoh scoring (nvbio/alignment),
behind a C ABI (include/nvbio_b200.h).  This package is the host-side mirror of the reference's
interface for those paths; torch is used only for device memory, streams and torch.distributed."""
from ._lib import NvbError, lib, LIB_PATH                                        # noqa: F401
from .strings import PackedStringSet, pack_symbols, unpack_symbols               # noqa: F401
from .fmindex import (FMIndexDevice, FMIndexFilterDevice, rank, rank4, match, match_approx, locate, map_seeds, locate_init, locate_lookup, locate_sorted,  # noqa: F401
                      MAP_EXACT, MAP_APPROX, dict_rank, dict_build_occ,
                      MATCH_FORWARD_ORDER, MATCH_COMPLEMENT)
from . import aln                                                                # noqa: F401
from .pipeline import SeedExtendParams, seed_extend, StreamingSeedExtend, StreamingBam, PairParams, seed_extend_paired, MapqParams, seed_extend_all, AllAlignments, ReseedParams, seed_extend_reseed, seed_extend_paired_reseed     # noqa: F401
from .pipeline import PAIR_UNPAIRED, PAIR_CONCORDANT, PAIR_RESCUED_MATE1, PAIR_RESCUED_MATE2, PAIR_DISCORDANT    # noqa: F401
from .finish import finish_alignments, FinishedAlignments                        # noqa: F401
from .bam import ContigTable, BamRecords, bam_records, bam_records_all, bam_header, write_bam, numbered_names, BamBatch, pack_names    # noqa: F401
from .bgzf import BgzfBlocks, BgzfCall, bgzf_compress                           # noqa: F401
from .bam_sort import SortedBamRecords, sort_bam_records, bam_index, write_sorted_bam    # noqa: F401
from .sam import SamText, SamCall, sam_header, sam_text, write_sam                  # noqa: F401

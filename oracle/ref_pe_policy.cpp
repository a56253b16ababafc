// oracle/ref_pe_policy.cpp -- TEST INFRASTRUCTURE (oracle/_ref/libnvbio_ref_pe_policy.so, built by oracle/ref_pe_policy.mk):
// nvBowtie's OWN frame_opposite_mate (nvBowtie/bowtie2/cuda/alignment_utils.h:61-98), compiled from an nvbio source tree where it lies,
// so that the paired-end framing of pipeline_core.cuh (pe_frame) is pinned against the reference's code on all 16 inputs.
#include <nvbio/basic/types.h>
#include <nvBowtie/bowtie2/cuda/alignment_utils.h>

using namespace nvbio;

extern "C" {

// frame_opposite_mate(policy[i], anchor[i], anchor_fw[i]) -> (left[i], fw[i]) for n inputs; policy in io::PE_POLICY_* numbering
// (FF 0, FR 1, RF 2, RR 3, nvbio/io/sequence/sequence.h:192-195)
void ref_frame_opposite_mate(const int32_t* policy, const uint32_t* anchor, const uint8_t* anchor_fw, uint32_t n, uint8_t* left, uint8_t* fw)
{
    for (uint32_t i = 0; i < n; ++i) {
        bool l = false, f = false;
        bowtie2::cuda::detail::frame_opposite_mate(policy[i], anchor[i], anchor_fw[i] != 0, l, f);
        left[i] = l ? 1 : 0; fw[i] = f ? 1 : 0;
    }
}

} // extern "C"

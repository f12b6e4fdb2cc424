"""torch.rand on a CUDA generator restated in Python (torch's ATen/native/cuda/DistributionTemplates.h): the launch policy of a draw of
N float32 values, the offset it advances the generator by, and which Philox call produces each element.  The perturbed one-launch step
(neuralsim_b200/torch_rng.py, csrc/torch_uniform.cuh) computes the same things on the device."""
BLOCK = 256
CURAND_OFFSETS = 4        # max_generator_offsets_per_curand_call
UNROLL = 4                # float4 / float: one curand_uniform4 per loop iteration


def calc_execution_policy(numel, sms, max_threads_per_sm):
    """-> (counter_offset, grid, block) as torch computes them"""
    grid = (numel + BLOCK - 1) // BLOCK
    grid = min(sms * (max_threads_per_sm // BLOCK), grid)
    counter_offset = ((numel - 1) // (BLOCK * grid * UNROLL) + 1) * CURAND_OFFSETS
    return counter_offset, grid, BLOCK


def element_calls(numel, sms, max_threads_per_sm):
    """the grid-stride loop of distribution_elementwise_grid_stride_kernel, run serially: {li: (thread idx, call k, component c)}"""
    _, grid, block = calc_execution_policy(numel, sms, max_threads_per_sm)
    stride = block * grid
    rounded = ((numel - 1) // (stride * UNROLL) + 1) * stride * UNROLL
    out = {}
    for idx in range(stride):
        for k, linear in enumerate(range(idx, rounded, stride * UNROLL)):
            for c in range(UNROLL):
                li = linear + stride * c
                if li < numel:
                    assert li not in out
                    out[li] = (idx, k, c)
    return out


def element_call(li, numel, cap):
    """the closed form of element_calls at grid cap `cap` = SMs * (maxThreadsPerSM / 256)"""
    stride = BLOCK * min((numel + BLOCK - 1) // BLOCK, cap)
    return li % stride, li // (UNROLL * stride), (li // stride) % UNROLL

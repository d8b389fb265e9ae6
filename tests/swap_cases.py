"""Cases of conv_swap_kernel (SSDK_PLAN_GEMM_SWAP: a forward convolution of at most 64 output channels on a large map, with
the weights on the wgmma M side and 192-pixel tiles), and the plan builder's rule for choosing it (model.cu, conv_kernel),
mirrored here so that a CPU test can check which case tables reach the variant.

Every case has at least 2 * 132 * 192 output pixels (two 192-pixel tiles per SM of an H100 SXM), and the images of the
multi-image cases end inside a 192-row tile."""
from conv_cases import SM_COUNT_H100, conv_case


def selects_swap(cin, cout, stride, pixels, head=False, sm_count=SM_COUNT_H100):
    """model.cu, conv_kernel: the plan's choice of conv_swap_kernel for a forward convolution (inference or training plan)."""
    return not head and stride == 1 and 64 <= cin and cout <= 64 and pixels >= 2 * sm_count * 192


def S(split):
    return dict(kernel='gemm_swap', bn=64, bm=192, split=split, epilogue='split', k_split=1, n_tiles_n=1)


SWAP_CASES = [
    conv_case('swap_64_relu_shared', 1, 264, 264, 64, 64, 3, S(1)),
    conv_case('swap_64_linear_unshared', 1, 264, 264, 64, 64, 3, S(1), act=None, env={'SSDK_SHARED_BORDER': '0'}),
    conv_case('swap_cout40_elu_3img', 3, 151, 151, 64, 40, 3, S(1), act='elu'),
    conv_case('swap_cin128_relu_2img', 2, 187, 185, 128, 64, 3, S(1)),
    conv_case('swap_64_nobias_folded_bn', 2, 190, 183, 64, 64, 3, S(1), bias=False, bn=True),
    conv_case('bf16_swap_64_relu_shared', 1, 264, 264, 64, 64, 3, S(0), prec='bf16'),
    conv_case('bf16_swap_cout24_elu_unshared', 3, 151, 151, 72, 24, 3, S(0), prec='bf16', act='elu', env={'SSDK_SHARED_BORDER': '0'}),
    conv_case('bf16_swap_cin128_linear_2img', 2, 187, 185, 128, 56, 3, S(0), prec='bf16', act=None),
]

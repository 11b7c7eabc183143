// TEST INFRASTRUCTURE: host execution of the depthwise-stencil body of csrc/td_demofusion.cu (tap order, fmaf
// accumulation and circular indexing of td_depthwise_conv2d / td_depthwise_conv2d_wrap), so that it can be checked on a
// machine without a GPU.  Built by tests/test_demofusion_wrap.py into tests/_build/; never part of libtd_b200.so.
#define TD_DEMOFUSION_HOST_EMULATION 1
#include "td_demofusion.cu"

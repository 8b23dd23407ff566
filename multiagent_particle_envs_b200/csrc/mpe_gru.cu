// mpe_gru.cu -- the 14 kernels of MAPPO's recurrent actor (mpe_policy_gru[_episode]_kernel, see mpe_kernels.cu),
// compiled as a translation unit of their own so that the build runs them alongside the rest of the library.
#define MPE_KERNEL_TEMPLATES_ONLY
#include "mpe_kernels.cu"

namespace mpe {

template <class P>
const void *gru_kernel(int episodes) {
    return episodes ? reinterpret_cast<const void *>(mpe_policy_gru_episode_kernel<P>)
                    : reinterpret_cast<const void *>(mpe_policy_gru_kernel<P>);
}

// the programs of GruBuilt
template const void *gru_kernel<Simple<1, 1>>(int);
template const void *gru_kernel<Spread<2>>(int);
template const void *gru_kernel<Spread<3>>(int);
template const void *gru_kernel<Spread<4>>(int);
template const void *gru_kernel<Spread<5>>(int);
template const void *gru_kernel<Spread<6>>(int);
template const void *gru_kernel<Reference>(int);

}  // namespace mpe

// mpe_critic.cu -- the 30 kernels of MAPPO's actor with its centralized critic (mpe_policy_mappo_critic[_episode]_kernel,
// see mpe_kernels.cu), compiled as a translation unit of their own so that the build runs them alongside the rest of the
// library.
#define MPE_KERNEL_TEMPLATES_ONLY
#include "mpe_kernels.cu"

namespace mpe {

template <class P>
const void *critic_kernel(int episodes) {
    static_assert(critic_built<P>(), "a program with a critic kernel");
    return episodes ? reinterpret_cast<const void *>(mpe_policy_mappo_critic_episode_kernel<P>)
                    : reinterpret_cast<const void *>(mpe_policy_mappo_critic_kernel<P>);
}

// the programs of critic_built: every MAPPO program but spread N=6 and tag 6+2
template const void *critic_kernel<Simple<1, 1>>(int);
template const void *critic_kernel<Spread<2>>(int);
template const void *critic_kernel<Spread<3>>(int);
template const void *critic_kernel<Spread<4>>(int);
template const void *critic_kernel<Spread<5>>(int);
template const void *critic_kernel<Tag<3, 1, 2>>(int);
template const void *critic_kernel<Tag<1, 1, 2>>(int);
template const void *critic_kernel<Tag<2, 1, 2>>(int);
template const void *critic_kernel<Tag<4, 2, 2>>(int);
template const void *critic_kernel<Adversary<1, 2, 2>>(int);
template const void *critic_kernel<Adversary<1, 3, 3>>(int);
template const void *critic_kernel<Push<1, 1, 2>>(int);
template const void *critic_kernel<SpeakerListener>(int);
template const void *critic_kernel<Reference>(int);
template const void *critic_kernel<Crypto>(int);

}  // namespace mpe

/* dfx_testing.h — entry points of libdfx_b200.so that exist for the project's tests and cost tools, not for applications: they are not
 * part of the C-ABI of include/dfx_b200.h and may change with any release. They are exported so that the tests can reach them through
 * ctypes. */
#ifndef DFX_TESTING_H
#define DFX_TESTING_H

#include "../../include/dfx_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* dfx_shadow_convert_to_filterable through its two-pass path at every range (the intermediate is then always required), where the
 * public entry picks the fused path for ranges up to 16. Both paths give the same bits; this lets the tests hold them to each other
 * and the cost tool time them on the same inputs. */
DFX_API dfx_status dfx_testing_shadow_convert_two_pass(void* stream, int32_t mode, const dfx_shadow_map_attribs* attribs,
                                                       const dfx_plane* shadow_map, int32_t n, const dfx_plane* filterable,
                                                       const dfx_plane* intermediate);

#ifdef __cplusplus
} /* extern "C" */
#endif
#endif /* DFX_TESTING_H */

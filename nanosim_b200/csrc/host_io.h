// What nanosim_api.cu calls in host_io.cu: the host-side expansion of the 2-bit bases that ns_fetch packs on the device.
#pragma once
#include <stdint.h>

// expands seq_bytes 2-bit bases (pack_bases_kernel: base k in bits [2(k&3)+1 : 2(k&3)] of byte k >> 2) into ASCII with
// `nt` host threads
void unpack_bases(const uint8_t* packed, uint8_t* seq, uint64_t seq_bytes, bool uracil, int nt);
// threads that expand the bases of one ns_fetch; 0: the bases are copied as ASCII, without packing
int unpack_threads();

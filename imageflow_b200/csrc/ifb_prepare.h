// ifb_prepare.h -- the order in which a batched call rejects a descriptor, shared by the host planners' <op>_prepare functions.  Plain
// C++ without CUDA calls (tests/cpu_emu links the planners unchanged).
#pragma once
#include <cstddef>
#include <string>

#include "../../include/ifb200.h"

namespace ifb {

// Runs check(d[i], code) over d[0..n) in order.  Empty when every descriptor passes (*code = IFB200_OK); else "<op> job i: <why>" for
// the first one rejected, with *code its status.  The <op>_prepare functions plan nothing until this has passed.
template <class Desc>
std::string check_each(const char* op, const Desc* d, size_t n, std::string (*check)(const Desc&, int*), int* code) {
    for (size_t i = 0; i < n; ++i) {
        const std::string why = check(d[i], code);
        if (!why.empty()) return std::string(op) + " job " + std::to_string(i) + ": " + why;
    }
    *code = IFB200_OK;
    return "";
}

}  // namespace ifb

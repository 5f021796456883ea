// Light path expressions: compiler from a subset of OSL's LPE grammar to the transition table FILM_MODE_LPE walks
// (host only, no CUDA call). See DESIGN.md §3 "Light path expressions".
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace mcrt
{
    // The compiled union of n <= MCRT_LPE_MAX_EXPRESSIONS expressions. State 0 is the state after the camera event C;
    // next[s * n_symbols + symbol] is the state after the event (MCRT_LPE_DEAD once no expression can match any more);
    // accept[s] has bit i set when expression i matches the events read so far (accept[MCRT_LPE_DEAD] = 0). Symbols are
    // the MCRT_LPE_SYM_* events, then one per label: symbol MCRT_LPE_SYM_LABEL0 + k is the lights of group labels[k]
    // (ascending); the lights of every other group read MCRT_LPE_SYM_L.
    struct LpeTable
    {
        uint32_t n_states = 0, n_symbols = 0;
        std::vector<uint8_t> next;
        std::vector<uint32_t> accept;   // [256]
        std::vector<uint32_t> labels;
    };

    // Parses, builds the Thompson NFA of each expression and the subset-construction DFA of their union, collapses the
    // states from which nothing is accepted into MCRT_LPE_DEAD and numbers the others breadth-first from state 0.
    // Labels must be below n_groups. Returns MCRT_OK, MCRT_ERR_INVALID (syntax, counts, labels) or
    // MCRT_ERR_UNSUPPORTED (more than MCRT_LPE_MAX_STATES live states), with the reason in error.
    int lpeCompile(const char* const* exprs, uint32_t n, uint32_t n_groups, LpeTable& out, std::string& error);
}

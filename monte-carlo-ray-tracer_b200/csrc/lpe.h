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
        // The photon mapper's side. A photon's events are read in emission order, its light's symbol first, by the DFA
        // of the reversed expressions: rev_next[r * n_symbols + symbol] (MCRT_LPE_DEAD once no camera prefix can make
        // the history match), starting at rev_start (MCRT_LPE_DEAD when nothing can match). A contribution whose camera
        // prefix ends in forward state s and whose photon history ends in reverse state r matches the expressions of
        // join[s * rev_n_states + r]; join_any[s] (256 entries) is 1 when some history completes s. photon_error is
        // non-empty, and the rest empty, when the reversed expressions exceed the limits: the photon mapper refuses the
        // table, the path tracer still takes it.
        uint32_t rev_n_states = 0, rev_start = 0;
        std::vector<uint8_t> rev_next;
        std::vector<uint32_t> join;
        std::vector<uint8_t> join_any;
        std::string photon_error;
    };

    // Parses, builds the Thompson NFA of each expression and the subset-construction DFA of their union, collapses the
    // states from which nothing is accepted into MCRT_LPE_DEAD and numbers the others breadth-first from state 0; then
    // the same for the reversed expressions and the join of the two (photon side, above). Labels must be below
    // n_groups. Returns MCRT_OK, MCRT_ERR_INVALID (syntax, counts, labels) or MCRT_ERR_UNSUPPORTED (more than
    // MCRT_LPE_MAX_STATES live forward states), with the reason in error.
    int lpeCompile(const char* const* exprs, uint32_t n, uint32_t n_groups, LpeTable& out, std::string& error);
}
